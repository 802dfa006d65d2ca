/* The whole PIPs forward from plain C: weight pack + raw frames + queries -> trajectories and visibility logits.
 *
 *   pips_encode                  frames -> channels-last feature maps        (BasicEncoder, nets/pips.py:436-445)
 *   pips_pyramid_build_nhwc      -> 4-level correlation pyramid              (CorrBlock.__init__, :346-352)
 *   pips_init_gather             -> the queries' features, broadcast over S  (:463-466)
 *   pips_refine_iter x iters     -> coords*stride of every iteration         (:499-539)
 *   pips_vis_head                -> visibility logits                        (:559)
 *
 * The weight pack is the file pips_b200/pack.py writes (pips_b200.saverloader.load writes <checkpoint>.pack next to the
 * checkpoint), read as examples/pack_read.c reads it.  Arithmetic: bf16x3 mixer, fp32 pyramid -- Pips(precision='bf16x3',
 * feat_dtype='fp32'), whose Pips.forward returns the same bits.
 *
 *   gcc -std=c99 -O2 -Wall -Wextra -Werror examples/track.c -Iinclude -I/usr/local/cuda/include \
 *       -Lpips_b200/lib -lpips_b200 -L/usr/local/cuda/lib64 -lcudart -lm -Wl,-rpath,$PWD/pips_b200/lib -o track
 *   ./track model.pack frames.f32 queries.f32 B S H W N stride iters trajs.f32 vis.f32
 *
 * frames.f32: (B, S, 3, H, W) fp32 raw, values 0..255 (RGB).  queries.f32: (B, N, 2) fp32 (x, y) in frame-0 pixels.
 * trajs.f32 receives (iters, B, S, N, 2) fp32 pixel coordinates, one set per refinement iteration (the last is the
 * result); vis.f32 (B, S, N) fp32 visibility logits.
 */
#include <math.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <cuda_runtime_api.h>

#include "pips_b200.h"

/* ---- the weight pack (see examples/pack_read.c for the layout) ---- */
typedef struct {
    const unsigned char* file;
    uint64_t size, origin;
    char* manifest;
} pack_file;

static int pack_open(const char* path, pack_file* p) {
    static const unsigned char magic[16] = {'P', 'I', 'P', 'S', 'B', '2', '0', '0', 'P', 'A', 'C', 'K', 0, 0, 0, 1};
    FILE* f = fopen(path, "rb");
    if (!f) return -1;
    fseek(f, 0, SEEK_END);
    const long size = ftell(f);
    fseek(f, 0, SEEK_SET);
    unsigned char* buf = (unsigned char*)malloc((size_t)size);
    const int ok = buf && fread(buf, 1, (size_t)size, f) == (size_t)size;
    fclose(f);
    uint64_t mlen = 0;
    if (!ok || size < 32 || memcmp(buf, magic, 16) != 0) { free(buf); return -1; }
    memcpy(&mlen, buf + 16, 8);
    memcpy(&p->origin, buf + 24, 8);
    if (32 + mlen > (uint64_t)size) { free(buf); return -1; }
    p->manifest = (char*)malloc(mlen + 1);
    memcpy(p->manifest, buf + 32, mlen);
    p->manifest[mlen] = 0;
    p->file = buf;
    p->size = (uint64_t)size;
    return 0;
}

/* the tensor `name` copied to a new device allocation; NULL if the pack has no such tensor */
static void* pack_upload(const pack_file* p, const char* name, uint64_t* nbytes_out) {
    char key[160];
    snprintf(key, sizeof key, "{\"name\":\"%s\",", name);
    const char* e = strstr(p->manifest, key);
    if (!e) return NULL;
    const char* of = strstr(e, "\"offset\":");
    const char* nb = strstr(e, "\"nbytes\":");
    if (!of || !nb) return NULL;
    const uint64_t off = strtoull(of + 9, NULL, 10), nbytes = strtoull(nb + 9, NULL, 10);
    if (p->origin + off + nbytes > p->size) return NULL;
    void* d = NULL;
    if (cudaMalloc(&d, nbytes) != cudaSuccess || cudaMemcpy(d, p->file + p->origin + off, nbytes, cudaMemcpyHostToDevice) != cudaSuccess)
        return NULL;
    if (nbytes_out) *nbytes_out = nbytes;
    return d;
}

static const void* need(const pack_file* p, const char* name) {
    const void* d = pack_upload(p, name, NULL);
    if (!d) {
        fprintf(stderr, "weight pack: no tensor %s\n", name);
        exit(1);
    }
    return d;
}

static void* dev_zeros(size_t bytes) {
    void* d = NULL;
    if (cudaMalloc(&d, bytes) != cudaSuccess || cudaMemset(d, 0, bytes) != cudaSuccess) {
        fprintf(stderr, "cudaMalloc of %zu bytes failed\n", bytes);
        exit(1);
    }
    return d;
}

static void check(int rc, const char* what) {
    if (rc != 0) {
        fprintf(stderr, "%s failed: %s\n", what, pips_last_error());
        exit(1);
    }
}

static void* read_file(const char* path, size_t bytes) {
    FILE* f = fopen(path, "rb");
    void* h = malloc(bytes);
    if (!f || !h || fread(h, 1, bytes, f) != bytes) {
        fprintf(stderr, "%s: cannot read %zu bytes\n", path, bytes);
        exit(1);
    }
    fclose(f);
    return h;
}

static void write_file(const char* path, const void* h, size_t bytes) {
    FILE* f = fopen(path, "wb");
    if (!f || fwrite(h, 1, bytes, f) != bytes) {
        fprintf(stderr, "%s: cannot write\n", path);
        exit(1);
    }
    fclose(f);
}

static size_t round_up(size_t v, size_t m) { return (v + m - 1) / m * m; }

int main(int argc, char** argv) {
    if (argc != 13) {
        fprintf(stderr, "usage: %s model.pack frames.f32 queries.f32 B S H W N stride iters trajs.f32 vis.f32\n", argv[0]);
        return 2;
    }
    const int B = atoi(argv[4]), S = atoi(argv[5]), H = atoi(argv[6]), W = atoi(argv[7]), N = atoi(argv[8]);
    const int stride = atoi(argv[9]), iters = atoi(argv[10]);
    if (B < 1 || S < 2 || S > PIPS_S_MAX || N < 1 || iters < 1 || (stride != 4 && stride != 8)) {
        fprintf(stderr, "need B, N, iters >= 1, 2 <= S <= %d, stride 4 or 8\n", PIPS_S_MAX);
        return 2;
    }
    const int H8 = H / stride, W8 = W / stride, F = B * S;
    if (pips_abi_version() != PIPS_B200_ABI_VERSION) {
        fprintf(stderr, "libpips_b200 ABI %d, header %d\n", pips_abi_version(), PIPS_B200_ABI_VERSION);
        return 1;
    }
    pack_file pk;
    if (pack_open(argv[1], &pk) != 0) {
        fprintf(stderr, "%s: not a pips_b200 weight pack\n", argv[1]);
        return 1;
    }
    char name[160];

    /* ---- weights: encoder filters "fnet.<conv>.w_hi/.w_lo/.b", mixer and heads "mixer.<pips_weights field>" ---- */
    pips_encoder_weights ew;
    memset(&ew, 0, sizeof ew);
    static const char* convs[] = {
        "conv1", "layer1.0.conv1", "layer1.0.conv2", "layer1.1.conv1", "layer1.1.conv2",
        "layer2.0.conv1", "layer2.0.conv2", "layer2.0.downsample.0", "layer2.1.conv1", "layer2.1.conv2",
        "layer3.0.conv1", "layer3.0.conv2", "layer3.0.downsample.0", "layer3.1.conv1", "layer3.1.conv2",
        "layer4.0.conv1", "layer4.0.conv2", "layer4.0.downsample.0", "layer4.1.conv1", "layer4.1.conv2", "conv2", "conv3"};
    pips_conv_weights* cw = &ew.conv1;                 /* the fields in the order of convs[] */
    for (size_t i = 0; i < sizeof convs / sizeof convs[0]; ++i) {
        snprintf(name, sizeof name, "fnet.%s.w_hi", convs[i]);
        cw[i].w_hi = need(&pk, name);
        snprintf(name, sizeof name, "fnet.%s.w_lo", convs[i]);
        cw[i].w_lo = need(&pk, name);
        snprintf(name, sizeof name, "fnet.%s.b", convs[i]);
        cw[i].b = (const float*)need(&pk, name);
    }
    pips_weights mw;
    memset(&mw, 0, sizeof mw);
#define TOP(f) mw.f = need(&pk, "mixer." #f)
    TOP(in_w_hi); TOP(in_w_lo); TOP(in_w_f32); TOP(in_b); TOP(out_ln_w); TOP(out_ln_b); TOP(head_w_hi); TOP(head_w_lo);
    TOP(head_w_f32); TOP(head_b); TOP(gn_w); TOP(gn_b); TOP(upd_w); TOP(upd_b); TOP(vis_w); TOP(vis_b);
#undef TOP
    for (int l = 0; l < PIPS_DEPTH; ++l) {
        pips_layer_weights* lw = &mw.layer[l];
#define LAYER(f) snprintf(name, sizeof name, "mixer.layer%d." #f, l), lw->f = need(&pk, name)
        LAYER(ln1_w); LAYER(ln1_b); LAYER(tok_w1); LAYER(tok_b1); LAYER(tok_w2); LAYER(tok_b2); LAYER(ln2_w); LAYER(ln2_b);
        LAYER(fc1_b); LAYER(fc2_b); LAYER(fc1_w_hi); LAYER(fc1_w_lo); LAYER(fc2_w_hi); LAYER(fc2_w_lo); LAYER(fc1_w_f32);
        LAYER(fc2_w_f32);
#undef LAYER
    }
    uint64_t tok_b2_bytes = 0;
    pack_upload(&pk, "mixer.layer0.tok_b2", &tok_b2_bytes);
    if (tok_b2_bytes != (uint64_t)S * 4) {
        fprintf(stderr, "the weight pack is for windows of %d frames, not %d\n", (int)(tok_b2_bytes / 4), S);
        return 1;
    }

    /* ---- inputs ---- */
    const size_t frame_bytes = (size_t)F * 3 * H * W * sizeof(float);
    float* h_rgb = (float*)read_file(argv[2], frame_bytes);
    float* h_xys = (float*)read_file(argv[3], (size_t)B * N * 2 * sizeof(float));
    void* rgb = dev_zeros(frame_bytes);
    cudaMemcpy(rgb, h_rgb, frame_bytes, cudaMemcpyHostToDevice);
    /* coords (B,S,N,2) in feature-map pixels: the queries over all S frames (nets/pips.py:450-453) */
    const size_t nc = (size_t)B * S * N * 2;
    float* h_coords = (float*)malloc(nc * sizeof(float));
    for (int b = 0; b < B; ++b)
        for (int s = 0; s < S; ++s)
            for (int n = 0; n < N * 2; ++n) h_coords[((size_t)b * S + s) * N * 2 + n] = h_xys[(size_t)b * N * 2 + n] / (float)stride;
    float* coords = (float*)dev_zeros(nc * sizeof(float));
    float* coords0 = (float*)dev_zeros(nc * sizeof(float));
    cudaMemcpy(coords, h_coords, nc * sizeof(float), cudaMemcpyHostToDevice);
    cudaMemcpy(coords0, h_coords, nc * sizeof(float), cudaMemcpyHostToDevice);
    /* times = linspace(0, S, S) as torch evaluates it in fp32 (nets/pips.py:519): from both ends towards the middle */
    float h_times[PIPS_S_MAX];
    const float step = (float)S / (float)(S - 1);
    for (int i = 0; i < S; ++i) h_times[i] = i < S / 2 ? fmaf(step, (float)i, 0.f) : fmaf(-step, (float)(S - i - 1), (float)S);
    float* times = (float*)dev_zeros(sizeof h_times);
    cudaMemcpy(times, h_times, S * sizeof(float), cudaMemcpyHostToDevice);

    /* ---- feature maps and pyramid ---- */
    const size_t ws_bytes = pips_encode_workspace_bytes(F, H, W, stride);
    if (ws_bytes == 0) check(pips_encode(&ew, rgb, 0, F, H, W, stride, NULL, 0, NULL, NULL, NULL), "pips_encode");
    void* enc_ws = dev_zeros(ws_bytes);
    float* fmaps = (float*)dev_zeros((size_t)F * H8 * W8 * PIPS_C * sizeof(float));
    check(pips_encode(&ew, rgb, 0, F, H, W, stride, enc_ws, ws_bytes, fmaps, NULL, NULL), "pips_encode");
    float* lvl[PIPS_LEVELS];
    for (int l = 0; l < PIPS_LEVELS; ++l) lvl[l] = (float*)dev_zeros((size_t)F * (H8 >> l) * (W8 >> l) * PIPS_C * sizeof(float));
    check(pips_pyramid_build_nhwc(fmaps, F, H8, W8, lvl, NULL, NULL), "pips_pyramid_build_nhwc");

    /* ---- refinement: the mixer workspace of B*N tracks in whole 256-row tiles, bf16x3 ---- */
    const int seqs = B * N;
    pips_workspace ws;
    memset(&ws, 0, sizeof ws);
    ws.rows_alloc = (int)round_up((size_t)seqs * S, 256);
    ws.seqs_alloc = (int)round_up((size_t)seqs, 256);
    const size_t rows = (size_t)ws.rows_alloc, sq = (size_t)ws.seqs_alloc;
    ws.x = (float*)dev_zeros(rows * PIPS_DIM * 4);
    ws.delta = (float*)dev_zeros(sq * PIPS_DELTA_LD(S) * 4);
    ws.x0_hi = dev_zeros(rows * PIPS_KITCHEN_PAD * 2); ws.x0_lo = dev_zeros(rows * PIPS_KITCHEN_PAD * 2);
    ws.y_hi = dev_zeros(rows * PIPS_DIM * 2);          ws.y_lo = dev_zeros(rows * PIPS_DIM * 2);
    ws.h_hi = dev_zeros(rows * PIPS_HIDDEN * 2);       ws.h_lo = dev_zeros(rows * PIPS_HIDDEN * 2);
    ws.p_hi = dev_zeros(sq * PIPS_DIM * 2);            ws.p_lo = dev_zeros(sq * PIPS_DIM * 2);
    float* ffeat = (float*)dev_zeros((size_t)seqs * PIPS_C * 4);
    float* ffeats = (float*)dev_zeros((size_t)seqs * S * PIPS_C * 4);
    check(pips_init_gather(lvl[0], B, S, N, H8, W8, coords, NULL, S, ffeat, ffeats, NULL), "pips_init_gather");

    pips_problem prob;
    memset(&prob, 0, sizeof prob);
    prob.B = B; prob.S = S; prob.N = N; prob.H = H8; prob.W = W8;
    prob.feat_dtype = PIPS_FEAT_F32;
    prob.precision = PIPS_PREC_BF16X3;
    for (int l = 0; l < PIPS_LEVELS; ++l) prob.lvl[l] = lvl[l];
    prob.times = times; prob.coords = coords; prob.coords0 = coords0; prob.ffeats = ffeats;
    prob.stride = (float)stride;
    prob.frames_per_batch = S;
    float* trajs = (float*)dev_zeros((size_t)iters * nc * sizeof(float));
    for (int it = 0; it < iters; ++it)
        check(pips_refine_iter(&prob, &mw, &ws, trajs + (size_t)it * nc, NULL), "pips_refine_iter");
    float* vis = (float*)dev_zeros((size_t)B * S * N * sizeof(float));
    check(pips_vis_head(ffeats, mw.vis_w, mw.vis_b, vis, B, S, N, NULL), "pips_vis_head");

    /* ---- results ---- */
    float* h_trajs = (float*)malloc((size_t)iters * nc * sizeof(float));
    float* h_vis = (float*)malloc((size_t)B * S * N * sizeof(float));
    if (cudaMemcpy(h_trajs, trajs, (size_t)iters * nc * sizeof(float), cudaMemcpyDeviceToHost) != cudaSuccess ||
        cudaMemcpy(h_vis, vis, (size_t)B * S * N * sizeof(float), cudaMemcpyDeviceToHost) != cudaSuccess) {
        fprintf(stderr, "the forward failed: %s\n", cudaGetErrorString(cudaGetLastError()));
        return 1;
    }
    write_file(argv[11], h_trajs, (size_t)iters * nc * sizeof(float));
    write_file(argv[12], h_vis, (size_t)B * S * N * sizeof(float));
    printf("tracked %d queries over %d frames of %dx%d in %d iterations\n", B * N, S, H, W, iters);
    return 0;
}
