// The whole feature encoder (BasicEncoder.forward, nets/pips.py:247-281) as one C call: host code only.  pips_encode
// enqueues the library's existing encoder kernels -- stem pack, wgmma convolutions with their InstanceNorm statistics,
// fused normalise/ReLU/residual passes, the resizes into the concatenation and the head -- in the order the Python
// sequence used to, into one caller-provided workspace.  It allocates nothing and never synchronises, so a stream
// capture records it as it is.
#include <stdio.h>
#include <stdlib.h>

#include "common.cuh"

using pips::fail;

namespace {

constexpr size_t kAlign = 256;                 // every workspace region starts on a 256-byte boundary
constexpr int kCat = 64 + 96 + 128 + 128;      // channels of the concatenation the head reads
constexpr int kCatP = (kCat + 63) / 64 * 64;   // ... padded to whole 64-channel K blocks

size_t round_up(size_t v) { return (v + kAlign - 1) / kAlign * kAlign; }
int pad64(int c) { return (c + 63) / 64 * 64; }
int half_up(int v) { return (v - 1) / 2 + 1; }            // output size of the stride-2 convolutions

struct Map { int H, W, C; };

// Shapes of one call and the byte offsets of its workspace regions.
struct Plan {
    int N, H, W, stride, H8, W8;
    Map stem, level[4];                        // the stem's output and each layer's output
    size_t unf_hi, unf_lo;                     // the stem operand (N, Ho+3, Wo, 64) bf16 pair
    size_t x[2];                               // block outputs, fp32, ping-pong
    size_t xp_hi[2], xp_lo[2];                 // ... and their bf16 pairs
    size_t a_hi, a_lo;                         // the pair between a block's two convolutions / the head's two
    size_t y, d;                               // convolution outputs before their InstanceNorm; the downsample's
    size_t part;                               // partial statistics of one convolution
    size_t s[2];                               // InstanceNorm statistics (N, 2, C)
    size_t cat_hi, cat_lo;                     // the head's input (N, H8, W8, 448) bf16 pair
    size_t total;
};

size_t px(int N, const Map& m) { return static_cast<size_t>(N) * m.H * m.W; }

bool conv_rows_fits(int W) {
    // the row-ring kernel's CTA pair covers 256 pixels of a row: widths that fill less than 3/4 of the last pair are
    // faster on the tap-by-tap kernel
    return W / static_cast<double>(((W + 255) / 256) * 256) >= 0.75;
}

int inorm_stats_chunks(int hw) {
    // partial sums per image by image size only (never by N), 64 chunks at most
    const int c = hw / 256;
    return c < 1 ? 1 : (c > 64 ? 64 : c);
}

// rows of partial statistics per image the convolution over `in` may write, whichever kernel computes them
size_t partial_rows(const Map& in, int R, int st, int pad, bool layer1) {
    int c = pips_conv_tc_chunks(in.H, in.W, R, R, st, st, pad, pad);
    const Map out = {(in.H + 2 * pad - R) / st + 1, (in.W + 2 * pad - R) / st + 1, 0};
    const int cs = inorm_stats_chunks(out.H * out.W);
    if (cs > c) c = cs;
    if (layer1) {
        const int cr = pips_conv_rows_chunks(in.H, in.W);
        if (cr > c) c = cr;
    }
    return static_cast<size_t>(c);
}

bool make_plan(int N, int H, int W, int stride, Plan& p) {
    if (N <= 0 || N > 65535 || (stride != 4 && stride != 8) || H < stride || W < stride) return false;
    if (static_cast<long long>(H) * W > (1ll << 26)) return false;
    p.N = N; p.H = H; p.W = W; p.stride = stride; p.H8 = H / stride; p.W8 = W / stride;
    p.stem = {half_up(H), half_up(W), 64};
    const int widths[4] = {64, 96, 128, 128};
    Map m = p.stem;
    for (int l = 0; l < 4; ++l) {
        if (l > 0) { m.H = half_up(m.H); m.W = half_up(m.W); }
        m.C = widths[l];
        p.level[l] = m;
    }
    const Map head = {p.H8, p.W8, 256};
    size_t x_elems = px(N, p.stem) * 64, pair_elems = px(N, p.stem) * 64, d_elems = 0;
    size_t part_floats = static_cast<size_t>(pips_conv_tc_chunks(p.stem.H + 3, p.stem.W, 4, 1, 1, 1, 0, 0)) * 64;   // stem
    Map in = p.stem;
    for (int l = 0; l < 4; ++l) {
        const Map& o = p.level[l];
        const size_t n = px(N, o);
        if (n * o.C > x_elems) x_elems = n * o.C;
        if (n * pad64(o.C) > pair_elems) pair_elems = n * pad64(o.C);
        if (l > 0 && n * o.C > d_elems) d_elems = n * o.C;
        const int st = l > 0 ? 2 : 1;
        size_t r = partial_rows(in, 3, st, 1, l == 0);                   // block 0's conv1
        if (l > 0) {
            const size_t rd = partial_rows(in, 1, 2, 0, false);          // its downsample
            if (rd > r) r = rd;
        }
        const size_t r2 = partial_rows(o, 3, 1, 1, l == 0);              // every other convolution of the layer
        if (r2 > r) r = r2;
        if (r * o.C > part_floats) part_floats = r * o.C;
        in = o;
    }
    const size_t head_part = partial_rows({p.H8, p.W8, kCat}, 3, 1, 1, false) * 256;
    if (head_part > part_floats) part_floats = head_part;
    const size_t head_elems = px(N, head) * 256;
    const size_t y_elems = x_elems > head_elems ? x_elems : head_elems;
    const size_t a_elems = pair_elems > head_elems ? pair_elems : head_elems;

    size_t off = 0;
    auto take = [&off](size_t bytes) { const size_t o = off; off += round_up(bytes); return o; };
    const size_t unf = static_cast<size_t>(N) * (p.stem.H + 3) * p.stem.W * 64 * 2;
    p.unf_hi = take(unf); p.unf_lo = take(unf);
    for (int i = 0; i < 2; ++i) p.x[i] = take(x_elems * 4);
    for (int i = 0; i < 2; ++i) { p.xp_hi[i] = take(pair_elems * 2); p.xp_lo[i] = take(pair_elems * 2); }
    p.a_hi = take(a_elems * 2); p.a_lo = take(a_elems * 2);
    p.y = take(y_elems * 4);
    p.d = take(d_elems * 4);
    p.part = take(static_cast<size_t>(N) * part_floats * 3 * 4);
    for (int i = 0; i < 2; ++i) p.s[i] = take(static_cast<size_t>(N) * 2 * 256 * 4);
    const size_t cat = px(N, head) * kCatP * 2;
    p.cat_hi = take(cat); p.cat_lo = take(cat);
    p.total = off;
    return true;
}

bool env_off(const char* name) {
    const char* e = getenv(name);
    return e && e[0] == '0' && e[1] == 0;
}

// A bf16 (hi, lo) activation of the workspace: (N, H, W, pad64(C)).
struct Pair { void* hi; void* lo; Map m; };

struct Run {
    const Plan& p;
    char* ws;
    void* stream;
    bool rows_on, stats_fused;
    int launches;
    bool dry;                                  // count the launches only

    float* f32(size_t off) { return reinterpret_cast<float*>(ws + off); }

    int step(int rc, int n) { launches += n; return rc; }

    // a convolution feeding an InstanceNorm: out (N, Ho, Wo, Cout) fp32 and its statistics
    int conv_stats(const Pair& x, const pips_conv_weights& w, int Cout, int R, int st, int pad, float* out, float* stats) {
        const int N = p.N, H = x.m.H, W = x.m.W, Cp = pad64(x.m.C);
        const int Ho = (H + 2 * pad - R) / st + 1, Wo = (W + 2 * pad - R) / st + 1;
        float* part = f32(p.part);
        if (x.m.C == 64 && Cout == 64 && R == 3 && st == 1 && pad == 1 && conv_rows_fits(W) && rows_on) {
            if (dry) return step(0, 2);
            const int chunks = pips_conv_rows_chunks(H, W);
            int rc = pips_conv_rows(x.hi, x.lo, N, H, W, w.w_hi, w.w_lo, out, part, stream);
            if (rc == 0) rc = pips_inorm_finalize(part, N, chunks, H * W, 64, stats, stream);
            return step(rc, 2);
        }
        if (!stats_fused) {                    // separate statistics pass
            if (dry) return step(0, 3);
            int rc = pips_conv_tc(x.hi, x.lo, N, H, W, Cp, w.w_hi, w.w_lo, Cout, R, R, st, pad, nullptr, out, stream);
            if (rc == 0) rc = pips_inorm_stats(out, N, Ho * Wo, Cout, part, inorm_stats_chunks(Ho * Wo), stats, stream);
            return step(rc, 3);
        }
        if (dry) return step(0, 2);
        const int chunks = pips_conv_tc_chunks(H, W, R, R, st, st, pad, pad);
        int rc = pips_conv_tc_stats(x.hi, x.lo, N, H, W, Cp, w.w_hi, w.w_lo, Cout, R, R, st, st, pad, pad, nullptr, out, part,
                                    stream);
        if (rc == 0) rc = pips_inorm_finalize(part, N, chunks, Ho * Wo, Cout, stats, stream);
        return step(rc, 2);
    }

    int apply(const float* y, const float* stats, const float* r, const float* stats_r, int relu_out, float* plain,
              const Pair& out) {
        if (dry) return step(0, 1);
        return step(pips_inorm_apply_pair(y, stats, r, stats_r, 1, relu_out, plain, out.hi, out.lo, pad64(out.m.C), p.N,
                                          out.m.H * out.m.W, out.m.C, stream), 1);
    }
};

// The sequence of the encoder.  keep: NULL or the 9 block boundaries' destinations.
int encode(Run& run, const pips_encoder_weights* w, const void* rgb, int dtype, float* fmaps, float* const* keep) {
    const Plan& p = run.p;
    const int N = p.N;
    char* ws = run.ws;
    void* st = run.stream;
    int rc = 0;
#define PIPS_TRY(expr) do { if ((rc = (expr)) != 0) return rc; } while (0)

    // stem: normalisation + 7x7/2 unfolded into a 4x1 stride-1 convolution over row pairs, its InstanceNorm, ReLU
    const Map unf = {p.stem.H + 3, p.stem.W, 64};
    const Pair u = {ws + p.unf_hi, ws + p.unf_lo, unf};
    float* y = run.f32(p.y);
    float* s0 = run.f32(p.s[0]);
    float* s1 = run.f32(p.s[1]);
    if (!run.dry) {
        PIPS_TRY(run.step(pips_stem_pack(rgb, dtype, N, p.H, p.W, u.hi, u.lo, st), 1));
        const int chunks = pips_conv_tc_chunks(unf.H, unf.W, 4, 1, 1, 1, 0, 0);
        PIPS_TRY(run.step(pips_conv_tc_stats(u.hi, u.lo, N, unf.H, unf.W, 64, w->conv1.w_hi, w->conv1.w_lo, 64, 4, 1, 1, 1, 0, 0,
                                             nullptr, y, run.f32(p.part), st), 1));
        PIPS_TRY(run.step(pips_inorm_finalize(run.f32(p.part), N, chunks, p.stem.H * p.stem.W, 64, s0, st), 1));
    } else {
        run.launches += 3;
    }
    int cur = 0, k = 0;
    float* X = keep ? keep[0] : run.f32(p.x[0]);
    Pair XP = {ws + p.xp_hi[0], ws + p.xp_lo[0], p.stem};
    PIPS_TRY(run.apply(y, s0, nullptr, nullptr, 0, X, XP));

    // the 8 residual blocks; after each layer its output is resized into the head's concatenation
    const pips_conv_weights* blocks[8][3] = {
        {&w->layer1_0_conv1, &w->layer1_0_conv2, nullptr}, {&w->layer1_1_conv1, &w->layer1_1_conv2, nullptr},
        {&w->layer2_0_conv1, &w->layer2_0_conv2, &w->layer2_0_downsample_0}, {&w->layer2_1_conv1, &w->layer2_1_conv2, nullptr},
        {&w->layer3_0_conv1, &w->layer3_0_conv2, &w->layer3_0_downsample_0}, {&w->layer3_1_conv1, &w->layer3_1_conv2, nullptr},
        {&w->layer4_0_conv1, &w->layer4_0_conv2, &w->layer4_0_downsample_0}, {&w->layer4_1_conv1, &w->layer4_1_conv2, nullptr}};
    const Map head = {p.H8, p.W8, kCat};
    const Pair cat = {ws + p.cat_hi, ws + p.cat_lo, head};
    int c_off = 0;
    for (int b = 0; b < 8; ++b) {
        const Map& o = p.level[b / 2];
        const int stride = blocks[b][2] ? 2 : 1;
        const Pair A = {ws + p.a_hi, ws + p.a_lo, o};
        PIPS_TRY(run.conv_stats(XP, *blocks[b][0], o.C, 3, stride, 1, y, s0));
        PIPS_TRY(run.apply(y, s0, nullptr, nullptr, 0, nullptr, A));
        PIPS_TRY(run.conv_stats(A, *blocks[b][1], o.C, 3, 1, 1, y, s0));
        float* Xn = keep ? keep[++k] : run.f32(p.x[cur ^ 1]);
        const Pair XPn = {ws + p.xp_hi[cur ^ 1], ws + p.xp_lo[cur ^ 1], o};
        if (blocks[b][2]) {
            float* d = run.f32(p.d);
            PIPS_TRY(run.conv_stats(XP, *blocks[b][2], o.C, 1, 2, 0, d, s1));
            PIPS_TRY(run.apply(y, s0, d, s1, 1, Xn, XPn));
        } else {
            PIPS_TRY(run.apply(y, s0, X, nullptr, 1, Xn, XPn));
        }
        X = Xn;
        XP = XPn;
        cur ^= 1;
        if (b % 2 == 1) {
            if (!run.dry) PIPS_TRY(pips_resize_pair(X, N, o.H, o.W, o.C, cat.hi, cat.lo, p.H8, p.W8, kCatP, c_off, st));
            run.launches += 1;
            c_off += o.C;
        }
    }

    // head: conv2 (416 -> 256, 3x3) with its InstanceNorm and ReLU, then conv3 (256 -> 128, 1x1) with its bias
    const Pair A = {ws + p.a_hi, ws + p.a_lo, {p.H8, p.W8, 256}};
    PIPS_TRY(run.conv_stats(cat, w->conv2, 256, 3, 1, 1, y, s0));
    PIPS_TRY(run.apply(y, s0, nullptr, nullptr, 0, nullptr, A));
    if (!run.dry)
        PIPS_TRY(pips_conv_tc(A.hi, A.lo, N, p.H8, p.W8, 256, w->conv3.w_hi, w->conv3.w_lo, 128, 1, 1, 1, 0, w->conv3.b, fmaps, st));
    run.launches += 1;
#undef PIPS_TRY
    return 0;
}

int shape_error(const char* who, int N, int H, int W, int stride) {
    char msg[256];
    if (stride != 4 && stride != 8)
        snprintf(msg, sizeof msg, "%s: stride must be 4 or 8 (got %d)", who, stride);
    else if (N <= 0 || N > 65535)
        snprintf(msg, sizeof msg, "%s: need 1 <= N <= 65535 frames (got %d)", who, N);
    else if (H < stride || W < stride)
        snprintf(msg, sizeof msg, "%s: a %dx%d frame is too small: the feature map (H/stride x W/stride) would be empty", who, H, W);
    else
        snprintf(msg, sizeof msg, "%s: a %dx%d frame is too large (at most 2^26 pixels)", who, H, W);
    return fail(msg);
}

}  // namespace

extern "C" size_t pips_encode_workspace_bytes(int N, int H, int W, int stride) {
    Plan p;
    return make_plan(N, H, W, stride, p) ? p.total : 0;
}

extern "C" int pips_encode_launches(int N, int H, int W, int stride) {
    Plan p;
    if (!make_plan(N, H, W, stride, p)) return 0;
    static const pips_encoder_weights none = {};
    Run run = {p, nullptr, nullptr, !env_off("PIPS_B200_CONV_ROWS"), !env_off("PIPS_B200_CONV_STATS"), 0, true};
    encode(run, &none, nullptr, 0, nullptr, nullptr);
    return run.launches;
}

extern "C" int pips_encode(const pips_encoder_weights* w, const void* rgb, int dtype, int N, int H, int W, int stride,
                           void* workspace, size_t workspace_bytes, float* fmaps_nhwc, float* const* keep, void* stream) {
    char msg[256];
    if (!w || !rgb || !fmaps_nhwc) return fail("pips_encode: null pointer (weights, rgb or fmaps_nhwc)");
    const pips_conv_weights* convs = &w->conv1;
    const int n_convs = static_cast<int>(sizeof(pips_encoder_weights) / sizeof(pips_conv_weights));
    for (int i = 0; i < n_convs; ++i) {
        if (!convs[i].w_hi || !convs[i].w_lo) {
            snprintf(msg, sizeof msg, "pips_encode: null filter pointer in convolution %d of pips_encoder_weights", i);
            return fail(msg);
        }
    }
    if (dtype != 0 && dtype != 1) return fail("pips_encode: dtype must be 0 (fp32) or 1 (bf16)");
    Plan p;
    if (!make_plan(N, H, W, stride, p)) return shape_error("pips_encode", N, H, W, stride);
    if (!workspace) return fail("pips_encode: null workspace");
    if (workspace_bytes < p.total) {
        snprintf(msg, sizeof msg, "pips_encode: workspace too small: %zu bytes given, %zu needed (pips_encode_workspace_bytes)",
                 workspace_bytes, p.total);
        return fail(msg);
    }
    if (reinterpret_cast<uintptr_t>(workspace) % kAlign) return fail("pips_encode: workspace must be 256-byte aligned");
    if (reinterpret_cast<uintptr_t>(rgb) % (dtype == 0 ? 4 : 2)) return fail("pips_encode: rgb is not aligned to its element size");
    if (reinterpret_cast<uintptr_t>(fmaps_nhwc) % 16) return fail("pips_encode: fmaps_nhwc must be 16-byte aligned");
    if (keep) {
        for (int i = 0; i < 9; ++i) {
            if (!keep[i] || reinterpret_cast<uintptr_t>(keep[i]) % 16) {
                snprintf(msg, sizeof msg, "pips_encode: keep[%d] is null or not 16-byte aligned", i);
                return fail(msg);
            }
        }
    }
    Run run = {p, static_cast<char*>(workspace), stream, !env_off("PIPS_B200_CONV_ROWS"), !env_off("PIPS_B200_CONV_STATS"), 0,
               false};
    return encode(run, w, rgb, dtype, fmaps_nhwc, keep);
}
