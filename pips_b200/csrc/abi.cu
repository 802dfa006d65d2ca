// C-ABI glue: error state, driver entry points, weight packing and the whole-iteration operators
// (pips_mixer_forward / pips_refine_iter) that chain the kernels of this library on one stream.
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "common.cuh"

namespace pips {

static thread_local char g_err[512] = "";

int fail(const char* msg) {
    snprintf(g_err, sizeof(g_err), "%s", msg);
    return 1;
}
int fail_cuda(const char* where, cudaError_t e) {
    snprintf(g_err, sizeof(g_err), "%s: %s", where, cudaGetErrorString(e));
    return 2;
}

bool pdl_enabled() {
    static int on = -1;
    if (on < 0) {
        const char* e = getenv("PIPS_B200_PDL");
        on = (e && e[0] == '0') ? 0 : 1;
    }
    return on != 0;
}

int current_device() {
    int dev = 0;
    return cudaGetDevice(&dev) == cudaSuccess ? dev : -1;
}

int sm_count() {
    static int n[kMaxDevices] = {};
    const int dev = current_device();
    if (dev < 0 || dev >= kMaxDevices) return 132;
    if (n[dev] == 0) {
        int v = 0;
        if (cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || v <= 0) v = 132;
        n[dev] = v;
    }
    return n[dev];
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

bool encode_tiled(CUtensorMap* map, CUtensorMapDataType dtype, uint32_t rank, void* base, const cuuint64_t* gdim,
                  const cuuint64_t* gstride_bytes, const cuuint32_t* box, const cuuint32_t* estride,
                  CUtensorMapSwizzle swizzle) {
    static EncodeTiledFn fn = nullptr;
    if (!fn) {
        void* p = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) != cudaSuccess || !p) return false;
        fn = reinterpret_cast<EncodeTiledFn>(p);
    }
    CUresult r = fn(map, dtype, rank, base, gdim, gstride_bytes, box, estride, CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle,
                    CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    return r == CUDA_SUCCESS;
}

__global__ void split_bf16_kernel(const float* __restrict__ src, __nv_bfloat16* __restrict__ hi, __nv_bfloat16* __restrict__ lo, size_t n) {
    for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < n; i += static_cast<size_t>(gridDim.x) * blockDim.x) {
        __nv_bfloat16 h, l;
        split_bf16(src[i], h, l);
        hi[i] = h;
        if (lo) lo[i] = l;
    }
}

}  // namespace pips

using namespace pips;

extern "C" int pips_abi_version(void) { return PIPS_B200_ABI_VERSION; }
extern "C" const char* pips_last_error(void) { return g_err; }

extern "C" int pips_split_bf16(const float* src, void* hi, void* lo, size_t n, void* stream) {
    if (!src || !hi) return fail("pips_split_bf16: null pointer");
    if (n == 0) return 0;
    size_t blocks = (n + 255) / 256;
    if (blocks > sm_count() * 16) blocks = sm_count() * 16;
    split_bf16_kernel<<<static_cast<unsigned>(blocks), 256, 0, static_cast<cudaStream_t>(stream)>>>(
        src, static_cast<__nv_bfloat16*>(hi), static_cast<__nv_bfloat16*>(lo), n);
    cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? 0 : fail_cuda("pips_split_bf16", e);
}

// Dense layer dispatch on the precision knob.  A is (rows, K) in the workspace, W (N, K) in pips_weights.
static int dense(int precision, const void* a_hi, const void* a_lo, const float* a_f32, int lda, int a_rows,
                 const void* w_hi, const void* w_lo, const float* w_f32, int ldw, int w_rows,
                 int M, int N, int K, const float* bias, int epi,
                 float* out_f32, int ldo, void* out_hi, void* out_lo, float* out_gelu_f32, int ldh, void* stream) {
    if (precision == PIPS_PREC_F32) {
        float* out = epi == PIPS_EPI_BIAS_GELU ? out_gelu_f32 : out_f32;
        int ld = epi == PIPS_EPI_BIAS_GELU ? ldh : ldo;
        if (!a_f32 || !w_f32 || !out) return fail("pips dense: fp32 precision needs the fp32 buffers");
        return pips_gemm_f32(a_f32, lda, w_f32, ldw, M, N, K, bias, epi, out, ld, stream);
    }
    const bool x3 = precision == PIPS_PREC_BF16X3;
    if (!a_hi || !w_hi || (x3 && (!a_lo || !w_lo))) return fail("pips dense: missing bf16 operand buffers for this precision");
    return pips_gemm_tc(a_hi, x3 ? a_lo : nullptr, lda, a_rows, w_hi, x3 ? w_lo : nullptr, ldw, w_rows, M, N, K, bias, epi,
                        out_f32, ldo, out_hi, x3 ? out_lo : nullptr, ldh, stream);
}

extern "C" int pips_mixer_forward_s(const pips_weights* w, const pips_workspace* ws, int seqs, int S, int precision,
                                    void* stream) {
    if (!w || !ws) return fail("pips_mixer_forward: null argument");
    if (seqs <= 0) return fail("pips_mixer_forward: no sequences");
    if (S < 2 || S > PIPS_S_MAX) return fail("pips_mixer_forward: S must be in 2..16");
    const int M = seqs * S;
    if (M > ws->rows_alloc || seqs > ws->seqs_alloc) return fail("pips_mixer_forward: workspace too small");
    const bool f32 = precision == PIPS_PREC_F32;
    const bool x3 = precision == PIPS_PREC_BF16X3;
    int rc;
    // nets/pips.py:115  Linear(519 -> 512)
    rc = dense(precision, ws->x0_hi, ws->x0_lo, ws->x0_f32, PIPS_KITCHEN_PAD, ws->rows_alloc,
               w->in_w_hi, w->in_w_lo, w->in_w_f32, PIPS_KITCHEN_PAD, PIPS_DIM,
               M, PIPS_DIM, PIPS_KITCHEN_PAD, w->in_b, PIPS_EPI_BIAS, ws->x, PIPS_DIM, nullptr, nullptr, nullptr, 0, stream);
    if (rc) return rc;
    for (int l = 0; l < PIPS_DEPTH; ++l) {
        const pips_layer_weights* L = &w->layer[l];
        // :117 token mixing (+ the LayerNorm of :118)
        rc = pips_tokenmix_s(ws->x, seqs, S, L->ln1_w, L->ln1_b, L->tok_w1, L->tok_b1, L->tok_w2, L->tok_b2, L->ln2_w, L->ln2_b,
                           f32 ? nullptr : ws->y_hi, x3 ? ws->y_lo : nullptr, f32 ? ws->y_f32 : nullptr, stream);
        if (rc) return rc;
        // :118 channel mixing: Linear(512,2048) -> GELU -> Linear(2048,512) -> + x
        rc = dense(precision, ws->y_hi, ws->y_lo, ws->y_f32, PIPS_DIM, ws->rows_alloc,
                   L->fc1_w_hi, L->fc1_w_lo, L->fc1_w_f32, PIPS_DIM, PIPS_HIDDEN,
                   M, PIPS_HIDDEN, PIPS_DIM, L->fc1_b, PIPS_EPI_BIAS_GELU, nullptr, 0, ws->h_hi, ws->h_lo, ws->h_f32, PIPS_HIDDEN, stream);
        if (rc) return rc;
        rc = dense(precision, ws->h_hi, ws->h_lo, ws->h_f32, PIPS_HIDDEN, ws->rows_alloc,
                   L->fc2_w_hi, L->fc2_w_lo, L->fc2_w_f32, PIPS_HIDDEN, PIPS_DIM,
                   M, PIPS_DIM, PIPS_HIDDEN, L->fc2_b, PIPS_EPI_BIAS_RESID, ws->x, PIPS_DIM, nullptr, nullptr, nullptr, 0, stream);
        if (rc) return rc;
    }
    // :120-121 LayerNorm + mean over S
    rc = pips_ln_pool_s(ws->x, seqs, S, w->out_ln_w, w->out_ln_b, f32 ? nullptr : ws->p_hi, x3 ? ws->p_lo : nullptr,
                      f32 ? ws->p_f32 : nullptr, stream);
    if (rc) return rc;
    // :122 Linear(512 -> 130 S)
    rc = dense(precision, ws->p_hi, ws->p_lo, ws->p_f32, PIPS_DIM, ws->seqs_alloc,
               w->head_w_hi, w->head_w_lo, w->head_w_f32, PIPS_DIM, PIPS_HEAD_PAD(S),
               seqs, PIPS_HEAD_N(S), PIPS_DIM, w->head_b, PIPS_EPI_BIAS, ws->delta, PIPS_DELTA_LD(S), nullptr, nullptr, nullptr, 0, stream);
    return rc;
}

extern "C" int pips_mixer_forward(const pips_weights* w, const pips_workspace* ws, int seqs, int precision, void* stream) {
    return pips_mixer_forward_s(w, ws, seqs, PIPS_S, precision, stream);
}

// pips_refine_iter, _clips and _groups: `groups` (with clip as its [B*N][4] table) selects pips_corr_gather_groups
static int refine_iter_entry(const char* who, const pips_problem* p, const int* clip, const pips_weights* w,
                             const pips_workspace* ws, float* out_px, void* stream, const pips_groups* groups = nullptr) {
    if (!p || !w || !ws || !out_px) {
        snprintf(g_err, sizeof(g_err), "%s: null argument", who);
        return 1;
    }
    if (clip ? p->S != PIPS_S : (p->S < 2 || p->S > PIPS_S_MAX)) {
        snprintf(g_err, sizeof(g_err), clip ? "%s: S must be 8" : "%s: S must be in 2..16", who);
        return 1;
    }
    if (clip && !p->frame_base) {
        snprintf(g_err, sizeof(g_err), "%s: a clip table needs frame_base", who);
        return 1;
    }
    const int seqs = p->B * p->N;
    const bool f32 = p->precision == PIPS_PREC_F32;
    const bool x3 = p->precision == PIPS_PREC_BF16X3;
    int rc = groups ? pips_corr_gather_groups(groups, p->feat_dtype, p->B, p->S, p->N, p->coords, p->ffeats, p->times,
                                              p->frame_base, clip,
                                              f32 ? nullptr : ws->x0_hi, x3 ? ws->x0_lo : nullptr, f32 ? ws->x0_f32 : nullptr,
                                              PIPS_KITCHEN_PAD, stream)
           : clip ? pips_corr_gather_clips(p->lvl, p->feat_dtype, p->B, p->S, p->N, p->H, p->W, p->coords, p->ffeats, p->times,
                                           p->frame_base, p->frames_per_batch, clip,
                                           f32 ? nullptr : ws->x0_hi, x3 ? ws->x0_lo : nullptr, f32 ? ws->x0_f32 : nullptr,
                                           PIPS_KITCHEN_PAD, stream)
                  : pips_corr_gather(p->lvl, p->feat_dtype, p->B, p->S, p->N, p->H, p->W, p->coords, p->ffeats, p->times,
                                     p->frame_base, p->frames_per_batch,
                                     f32 ? nullptr : ws->x0_hi, x3 ? ws->x0_lo : nullptr, f32 ? ws->x0_f32 : nullptr,
                                     PIPS_KITCHEN_PAD, stream);
    if (rc) return rc;
    rc = pips_mixer_forward_s(w, ws, seqs, p->S, p->precision, stream);
    if (rc) return rc;
    return pips_update_peer(ws->delta, p->coords, p->coords0, p->ffeats, w->gn_w, w->gn_b, w->upd_w, w->upd_b, out_px,
                            p->stride, p->B, p->S, p->N, &p->peer, stream);
}

extern "C" int pips_refine_iter(const pips_problem* p, const pips_weights* w, const pips_workspace* ws,
                                float* out_px, void* stream) {
    return refine_iter_entry("pips_refine_iter", p, nullptr, w, ws, out_px, stream);
}

extern "C" int pips_refine_iter_clips(const pips_problem* p, const int* clip, const pips_weights* w,
                                      const pips_workspace* ws, float* out_px, void* stream) {
    return refine_iter_entry("pips_refine_iter_clips", p, clip, w, ws, out_px, stream);
}

extern "C" int pips_refine_iter_groups(const pips_problem* p, const pips_groups* groups, const int* table,
                                       const pips_weights* w, const pips_workspace* ws, float* out_px, void* stream) {
    if (!groups || !table) {
        snprintf(g_err, sizeof(g_err), "pips_refine_iter_groups: the grouped mode needs groups and a table");
        return 1;
    }
    return refine_iter_entry("pips_refine_iter_groups", p, table, w, ws, out_px, stream, groups);
}
