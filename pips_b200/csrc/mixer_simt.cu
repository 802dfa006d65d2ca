// CUDA-core parts of the DeltaBlock mixer and the state update:
//   pips_gemm_f32   exact fp32 dense layer (PIPS_PREC_F32; also the on-device cross-check of the wgmma path)
//   pips_tokenmix   LN -> token-mixing MLP over the S frames -> +x -> LN   (K = S/4S: not a tensor-core shape)
//   pips_ln_pool    final LN + mean over S
//   pips_update     GroupNorm/Linear/GELU feature update + coord update + frame-0 lock
//   pips_vis_head   Linear(128,1)
#include <stdlib.h>

#include "mixer_common.cuh"

namespace pips {

// ------------------------------------------------------------------------------------------ fp32 GEMM
constexpr int SG_BM = 64, SG_BN = 64, SG_BK = 16;

__global__ void __launch_bounds__(256)
gemm_f32_kernel(const float* __restrict__ a, int lda, const float* __restrict__ w, int ldw, int M, int N, int K,
                const float* __restrict__ bias, int epilogue, float* out, int ldo) {
    __shared__ float sa[SG_BK][SG_BM + 4];
    __shared__ float sw[SG_BK][SG_BN + 4];
    const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
    const int m0 = blockIdx.y * SG_BM, n0 = blockIdx.x * SG_BN;
    float acc[4][4] = {};
    const int lr = threadIdx.x >> 2;          // 0..63: tile row loaded by this thread
    const int lk = (threadIdx.x & 3) * 4;     // 0,4,8,12
    for (int k0 = 0; k0 < K; k0 += SG_BK) {
        float4 va = make_float4(0.f, 0.f, 0.f, 0.f), vw = va;
        if (m0 + lr < M) va = *reinterpret_cast<const float4*>(a + static_cast<size_t>(m0 + lr) * lda + k0 + lk);
        if (n0 + lr < N) vw = *reinterpret_cast<const float4*>(w + static_cast<size_t>(n0 + lr) * ldw + k0 + lk);
        sa[lk + 0][lr] = va.x; sa[lk + 1][lr] = va.y; sa[lk + 2][lr] = va.z; sa[lk + 3][lr] = va.w;
        sw[lk + 0][lr] = vw.x; sw[lk + 1][lr] = vw.y; sw[lk + 2][lr] = vw.z; sw[lk + 3][lr] = vw.w;
        __syncthreads();
#pragma unroll
        for (int k = 0; k < SG_BK; ++k) {
            float ra[4], rw[4];
#pragma unroll
            for (int i = 0; i < 4; ++i) { ra[i] = sa[k][ty * 4 + i]; rw[i] = sw[k][tx * 4 + i]; }
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
                for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(ra[i], rw[j], acc[i][j]);
        }
        __syncthreads();
    }
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int m = m0 + ty * 4 + i;
        if (m >= M) continue;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int n = n0 + tx * 4 + j;
            if (n >= N) continue;
            float v = acc[i][j] + bias[n];
            float* o = out + static_cast<size_t>(m) * ldo + n;
            if (epilogue == PIPS_EPI_BIAS_GELU) v = gelu_exact(v);
            else if (epilogue == PIPS_EPI_BIAS_RESID) v += *o;
            *o = v;
        }
    }
}

// ------------------------------------------------------------------------------------------ token mixing
// S <= 8 frames per track, padded to 8 with zero weights (padded frames are neither loaded nor stored: x = 0 there).
// kFull: S == 8, compiled without the per-frame guards (which need more than 128 registers).
template <bool kFull>
__global__ void __launch_bounds__(TM_THREADS, kFull ? 4 : 3)
tokenmix_kernel(float* __restrict__ x, int s_arg, const float* __restrict__ ln1_w, const float* __restrict__ ln1_b,
                const float* __restrict__ w1, const float* __restrict__ b1, const float* __restrict__ w2,
                const float* __restrict__ b2, const float* __restrict__ ln2_w, const float* __restrict__ ln2_b,
                __nv_bfloat16* y_hi, __nv_bfloat16* y_lo, float* y_f32) {
    __shared__ float red[4][8];
    // weights duplicated into (w, w) pairs so that one LDS.128 yields two packed FFMA2 operands
    __shared__ __align__(16) float2 s_w1[32 * 8], s_w2t[32 * 8];  // w1[j][s] and w2 transposed to [j][s]
    __shared__ float s_b1[32], s_b2[8];
    const int S = kFull ? 8 : s_arg;
    pdl_trigger();
    for (int i = threadIdx.x; i < 256; i += TM_THREADS) {
        const int j = i >> 3, s = i & 7;
        const bool in = j < 4 * S && s < S;
        s_w1[i] = bcast2(in ? w1[j * S + s] : 0.f);        // w1 is (4S j, S s)
        s_w2t[i] = bcast2(in ? w2[s * 4 * S + j] : 0.f);   // w2 is (S s, 4S j)
    }
    if (threadIdx.x < 32) s_b1[threadIdx.x] = static_cast<int>(threadIdx.x) < 4 * S ? b1[threadIdx.x] : 0.f;
    if (threadIdx.x < 8) s_b2[threadIdx.x] = static_cast<int>(threadIdx.x) < S ? b2[threadIdx.x] : 0.f;

    const size_t base = static_cast<size_t>(blockIdx.x) * S * 512 + threadIdx.x * 4;
    float xv[8][4], yv[8][4];
    pdl_wait();                                // x comes from the previous kernel; the weights staged above are constants
#pragma unroll
    for (int s = 0; s < 8; ++s) {
        const float4 t = s < S ? *reinterpret_cast<const float4*>(x + base + s * 512) : make_float4(0.f, 0.f, 0.f, 0.f);
        xv[s][0] = t.x; xv[s][1] = t.y; xv[s][2] = t.z; xv[s][3] = t.w;
    }
    const float4 g1 = *reinterpret_cast<const float4*>(ln1_w + threadIdx.x * 4);
    const float4 c1 = *reinterpret_cast<const float4*>(ln1_b + threadIdx.x * 4);
    layernorm8(xv, yv, g1, c1, red);          // also orders the smem weight writes before their use

    // Conv1d(8->32,k=1) -> GELU -> Conv1d(32->8,k=1) across the frame axis, independently per channel;
    // channels are processed as two packed pairs (FFMA2).
    float2 y2[8][2], z2[8][2];
#pragma unroll
    for (int s = 0; s < 8; ++s) {
        y2[s][0] = make_float2(yv[s][0], yv[s][1]);
        y2[s][1] = make_float2(yv[s][2], yv[s][3]);
        z2[s][0] = z2[s][1] = bcast2(s_b2[s]);
    }
#pragma unroll 4
    for (int j = 0; j < 32; ++j) {
        float2 wa[8], wb[8];
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const float4 a = *reinterpret_cast<const float4*>(s_w1 + j * 8 + 2 * k);
            const float4 b = *reinterpret_cast<const float4*>(s_w2t + j * 8 + 2 * k);
            wa[2 * k] = make_float2(a.x, a.y); wa[2 * k + 1] = make_float2(a.z, a.w);
            wb[2 * k] = make_float2(b.x, b.y); wb[2 * k + 1] = make_float2(b.z, b.w);
        }
        float2 h0 = bcast2(s_b1[j]), h1 = h0;
#pragma unroll
        for (int s = 0; s < 8; ++s) {
            h0 = fma2(wa[s], y2[s][0], h0);
            h1 = fma2(wa[s], y2[s][1], h1);
        }
        h0 = gelu_fast2(h0);
        h1 = gelu_fast2(h1);
#pragma unroll
        for (int s = 0; s < 8; ++s) {
            z2[s][0] = fma2(wb[s], h0, z2[s][0]);
            z2[s][1] = fma2(wb[s], h1, z2[s][1]);
        }
    }
    float z[8][4];
#pragma unroll
    for (int s = 0; s < 8; ++s) { z[s][0] = z2[s][0].x; z[s][1] = z2[s][0].y; z[s][2] = z2[s][1].x; z[s][3] = z2[s][1].y; }
#pragma unroll
    for (int s = 0; s < 8; ++s) {
#pragma unroll
        for (int c = 0; c < 4; ++c) xv[s][c] += z[s][c];
        if (s < S) *reinterpret_cast<float4*>(x + base + s * 512) = make_float4(xv[s][0], xv[s][1], xv[s][2], xv[s][3]);
    }
    const float4 g2 = *reinterpret_cast<const float4*>(ln2_w + threadIdx.x * 4);
    const float4 c2 = *reinterpret_cast<const float4*>(ln2_b + threadIdx.x * 4);
    layernorm8(xv, yv, g2, c2, red);
#pragma unroll
    for (int s = 0; s < 8; ++s)
        if (s < S) store_row4(yv[s], base + s * 512, y_hi, y_lo, y_f32);
}

// 9 <= S <= 16 frames per track, padded to 16: 256 threads, warpgroup w holds frames 8w..8w+7 for both LayerNorms
// (thread t: channels 4t..4t+3); the token-mixing MLP runs with every thread on 2 channels of all 16 frames, exchanged
// through shared memory.
__global__ void __launch_bounds__(2 * TM_THREADS)
tokenmix16_kernel(float* __restrict__ x, int S, const float* __restrict__ ln1_w, const float* __restrict__ ln1_b,
                  const float* __restrict__ w1, const float* __restrict__ b1, const float* __restrict__ w2,
                  const float* __restrict__ b2, const float* __restrict__ ln2_w, const float* __restrict__ ln2_b,
                  __nv_bfloat16* y_hi, __nv_bfloat16* y_lo, float* y_f32) {
    __shared__ float red[8][8];
    __shared__ __align__(16) float s_w1[64 * 16], s_w2t[64 * 16];      // w1[j][s] and w2 transposed to [j][s], zero-padded
    __shared__ float s_b1[64], s_b2[16];
    __shared__ __align__(16) float xs[16][512];                        // LN1(x), then z, of the whole track
    pdl_trigger();
    for (int i = threadIdx.x; i < 64 * 16; i += 2 * TM_THREADS) {
        const int j = i >> 4, s = i & 15;
        const bool in = j < 4 * S && s < S;
        s_w1[i] = in ? w1[j * S + s] : 0.f;
        s_w2t[i] = in ? w2[s * 4 * S + j] : 0.f;
    }
    if (threadIdx.x < 64) s_b1[threadIdx.x] = static_cast<int>(threadIdx.x) < 4 * S ? b1[threadIdx.x] : 0.f;
    if (threadIdx.x < 16) s_b2[threadIdx.x] = static_cast<int>(threadIdx.x) < S ? b2[threadIdx.x] : 0.f;

    const int t = threadIdx.x & 127, f0 = 8 * (threadIdx.x >> 7);
    const size_t base = static_cast<size_t>(blockIdx.x) * S * 512 + t * 4;
    float xv[8][4], yv[8][4];
    pdl_wait();
#pragma unroll
    for (int s = 0; s < 8; ++s) {
        const float4 v = f0 + s < S ? *reinterpret_cast<const float4*>(x + base + (f0 + s) * 512) : make_float4(0.f, 0.f, 0.f, 0.f);
        xv[s][0] = v.x; xv[s][1] = v.y; xv[s][2] = v.z; xv[s][3] = v.w;
    }
    const float4 g1 = *reinterpret_cast<const float4*>(ln1_w + t * 4);
    const float4 c1 = *reinterpret_cast<const float4*>(ln1_b + t * 4);
    layernorm8_wg(xv, yv, g1, c1, red);
#pragma unroll
    for (int s = 0; s < 8; ++s) *reinterpret_cast<float4*>(&xs[f0 + s][t * 4]) = make_float4(yv[s][0], yv[s][1], yv[s][2], yv[s][3]);
    __syncthreads();
    {
        const int c = 2 * threadIdx.x;
        float2 y2[16], z2[16];
#pragma unroll
        for (int s = 0; s < 16; ++s) {
            y2[s] = *reinterpret_cast<const float2*>(&xs[s][c]);
            z2[s] = bcast2(s_b2[s]);
        }
#pragma unroll 2
        for (int j = 0; j < 64; ++j) {
            float2 h = bcast2(s_b1[j]);
#pragma unroll
            for (int s = 0; s < 16; ++s) h = fma2(bcast2(s_w1[j * 16 + s]), y2[s], h);
            h = gelu_fast2(h);
#pragma unroll
            for (int s = 0; s < 16; ++s) z2[s] = fma2(bcast2(s_w2t[j * 16 + s]), h, z2[s]);
        }
        __syncthreads();                                               // every thread has read its y
#pragma unroll
        for (int s = 0; s < 16; ++s) *reinterpret_cast<float2*>(&xs[s][c]) = z2[s];
    }
    __syncthreads();
#pragma unroll
    for (int s = 0; s < 8; ++s) {
        const float4 z = *reinterpret_cast<const float4*>(&xs[f0 + s][t * 4]);
        xv[s][0] += z.x; xv[s][1] += z.y; xv[s][2] += z.z; xv[s][3] += z.w;
        if (f0 + s < S) *reinterpret_cast<float4*>(x + base + (f0 + s) * 512) = make_float4(xv[s][0], xv[s][1], xv[s][2], xv[s][3]);
    }
    const float4 g2 = *reinterpret_cast<const float4*>(ln2_w + t * 4);
    const float4 c2 = *reinterpret_cast<const float4*>(ln2_b + t * 4);
    layernorm8_wg(xv, yv, g2, c2, red);
#pragma unroll
    for (int s = 0; s < 8; ++s)
        if (f0 + s < S) store_row4(yv[s], base + (f0 + s) * 512, y_hi, y_lo, y_f32);
}

// ------------------------------------------------------------------------------------------ final LN + mean over S
// the S rows of a track are normalised 8 at a time and summed in frame order; the mean is that sum / S
__global__ void __launch_bounds__(TM_THREADS)
ln_pool_kernel(const float* __restrict__ x, int S, const float* __restrict__ ln_w, const float* __restrict__ ln_b,
               __nv_bfloat16* p_hi, __nv_bfloat16* p_lo, float* p_f32) {
    __shared__ float red[4][8];
    const size_t base = static_cast<size_t>(blockIdx.x) * S * 512 + threadIdx.x * 4;
    float xv[8][4], yv[8][4];
    pdl_trigger();
    pdl_wait();
    const float4 g = *reinterpret_cast<const float4*>(ln_w + threadIdx.x * 4);
    const float4 c = *reinterpret_cast<const float4*>(ln_b + threadIdx.x * 4);
    float a[4] = {0.f, 0.f, 0.f, 0.f};
    for (int f0 = 0; f0 < S; f0 += 8) {
#pragma unroll
        for (int s = 0; s < 8; ++s) {
            const float4 t = f0 + s < S ? *reinterpret_cast<const float4*>(x + base + (f0 + s) * 512) : make_float4(0.f, 0.f, 0.f, 0.f);
            xv[s][0] = t.x; xv[s][1] = t.y; xv[s][2] = t.z; xv[s][3] = t.w;
        }
        layernorm8(xv, yv, g, c, red);
#pragma unroll
        for (int k = 0; k < 4; ++k)
#pragma unroll
            for (int s = 0; s < 8; ++s)
                if (f0 + s < S) a[k] += yv[s][k];
    }
    float m[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) m[k] = __fdiv_rn(a[k], static_cast<float>(S));
    store_row4(m, static_cast<size_t>(blockIdx.x) * 512 + threadIdx.x * 4, p_hi, p_lo, p_f32);
}

// ------------------------------------------------------------------------------------------ state update
// CTA = 256 threads handles 64 mixer rows.  Phase 1: GroupNorm(1,128) of the 128 delta-feature channels
// (4 threads per row), normalised rows to smem.  Phase 2: (64x128).(128x128)^T fp32 with the weight in
// smem (transposed, padded), +bias, GELU, += ffeats.  Threads with col==0 also advance the coordinates.
constexpr int UP_ROWS = 64;

__global__ void __launch_bounds__(256)
update_kernel(const float* __restrict__ delta, float* __restrict__ coords, const float* __restrict__ coords0,
              float* __restrict__ ffeats, const float* __restrict__ gn_w, const float* __restrict__ gn_b,
              const float* __restrict__ wu, const float* __restrict__ bu, float* __restrict__ out_px, float stride,
              int B, int S, int N, const pips_peer_out peer) {
    extern __shared__ float sm[];
    float* s_wt = sm;                         // [128 k][129]  wt[k][j] = wu[j][k]
    float* s_g = sm + 128 * 129;              // [64 rows][132]
    const int rows_total = B * N * S;
    const int r0 = blockIdx.x * UP_ROWS;
    pdl_trigger();
    for (int i = threadIdx.x; i < 128 * 128; i += 256) {      // constant weights: staged while the head GEMM drains
        const int j = i >> 7, k = i & 127;
        s_wt[k * 129 + j] = wu[i];
    }
    pdl_wait();
    {
        const int lr = threadIdx.x >> 2, part = threadIdx.x & 3;      // 4 threads x 32 channels per row
        const int r = r0 + lr;
        float v[32];
        float sum = 0.f;
        if (r < rows_total) {
            const int seq = r / S, s = r % S;
            const float* d = delta + static_cast<size_t>(seq) * PIPS_DELTA_LD(S) + s * 130 + 2 + part * 32;
#pragma unroll
            for (int i = 0; i < 32; ++i) { v[i] = d[i]; sum += v[i]; }
        } else {
#pragma unroll
            for (int i = 0; i < 32; ++i) v[i] = 0.f;
        }
        sum += __shfl_xor_sync(0xffffffffu, sum, 1);
        sum += __shfl_xor_sync(0xffffffffu, sum, 2);
        const float mean = sum * (1.0f / 128.0f);
        float sq = 0.f;
#pragma unroll
        for (int i = 0; i < 32; ++i) { const float dlt = v[i] - mean; sq += dlt * dlt; }
        sq += __shfl_xor_sync(0xffffffffu, sq, 1);
        sq += __shfl_xor_sync(0xffffffffu, sq, 2);
        const float rstd = rsqrtf(sq * (1.0f / 128.0f) + 1e-5f);
#pragma unroll
        for (int i = 0; i < 32; ++i) {
            const int c = part * 32 + i;
            s_g[lr * 132 + c] = (v[i] - mean) * rstd * gn_w[c] + gn_b[c];
        }
        // coordinate update (one thread per row)
        if (part == 0 && r < rows_total) {
            const int seq = r / S, s = r % S;
            const int b = seq / N, n = seq % N;
            const float* d = delta + static_cast<size_t>(seq) * PIPS_DELTA_LD(S) + s * 130;
            const size_t ci = ((static_cast<size_t>(b) * S + s) * N + n) * 2;
            float cx, cy;
            if (s == 0) { cx = coords0[ci]; cy = coords0[ci + 1]; }        // nets/pips.py:535-536
            else { cx = coords[ci] + d[0]; cy = coords[ci + 1] + d[1]; }    // :533
            coords[ci] = cx; coords[ci + 1] = cy;
            out_px[ci] = cx * stride; out_px[ci + 1] = cy * stride;         // :538
            if (peer.n_peers > 0) {
                // the all-gather of the prediction, fused: this rank's slice goes straight into every rank's
                // full (B,S,n_total,2) result over NVLink (peer-mapped stores; visibility: pips_peer_barrier)
                const size_t gi = ((static_cast<size_t>(b) * S + s) * peer.n_total + peer.n_offset + n) * 2;
                const float2 v = make_float2(cx * stride, cy * stride);
                for (int p = 0; p < peer.n_peers; ++p) *reinterpret_cast<float2*>(peer.out[p] + gi) = v;
            }
        }
    }
    __syncthreads();
    // phase 2: thread (ty 0..15, tx 0..15) -> rows ty*4..+3, cols tx + 16*j (j<8)
    const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
    float acc[4][8] = {};
#pragma unroll 4
    for (int k = 0; k < 128; ++k) {
        float a[4], wv[8];
#pragma unroll
        for (int i = 0; i < 4; ++i) a[i] = s_g[(ty * 4 + i) * 132 + k];
#pragma unroll
        for (int j = 0; j < 8; ++j) wv[j] = s_wt[k * 129 + tx + 16 * j];
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
            for (int j = 0; j < 8; ++j) acc[i][j] = fmaf(a[i], wv[j], acc[i][j]);
    }
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int r = r0 + ty * 4 + i;
        if (r >= rows_total) continue;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const int c = tx + 16 * j;
            float* f = ffeats + static_cast<size_t>(r) * 128 + c;
            *f = gelu_exact(acc[i][j] + bu[c]) + *f;                      // :530
        }
    }
}

__global__ void vis_head_kernel(const float* __restrict__ ffeats, const float* __restrict__ w, const float* __restrict__ b,
                                float* __restrict__ vis, int B, int S, int N) {
    const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (warp >= B * N * S) return;
    const float4 f = *reinterpret_cast<const float4*>(ffeats + static_cast<size_t>(warp) * 128 + lane * 4);
    const float4 wv = *reinterpret_cast<const float4*>(w + lane * 4);
    float d = warp_sum(f.x * wv.x + f.y * wv.y + f.z * wv.z + f.w * wv.w);
    if (lane == 0) {
        const int seq = warp / S, s = warp % S, bb = seq / N, n = seq % N;
        vis[(static_cast<size_t>(bb) * S + s) * N + n] = d + b[0];
    }
}

}  // namespace pips

int tokenmix_tc_launch(float* x, int seqs, int S, const float* ln1_w, const float* ln1_b, const float* w1, const float* b1,
                       const float* w2, const float* b2, const float* ln2_w, const float* ln2_b, void* y_hi, void* y_lo,
                       cudaStream_t st);   // tokenmix_tc.cu

using namespace pips;

#define LAUNCH_CHECK(name)                                        \
    do {                                                          \
        cudaError_t e__ = cudaGetLastError();                     \
        if (e__ != cudaSuccess) return fail_cuda(name, e__);      \
    } while (0)

extern "C" int pips_gemm_f32(const float* a, int lda, const float* w, int ldw, int M, int N, int K,
                             const float* bias, int epilogue, float* out, int ldo, void* stream) {
    if (!a || !w || !bias || !out) return fail("pips_gemm_f32: null pointer");
    if (M <= 0 || N <= 0 || K <= 0 || (K % SG_BK) || (lda % 4) || (ldw % 4)) return fail("pips_gemm_f32: bad shape (K%16, ld%4)");
    dim3 grid((N + SG_BN - 1) / SG_BN, (M + SG_BM - 1) / SG_BM);
    gemm_f32_kernel<<<grid, 256, 0, static_cast<cudaStream_t>(stream)>>>(a, lda, w, ldw, M, N, K, bias, epilogue, out, ldo);
    LAUNCH_CHECK("pips_gemm_f32");
    return 0;
}

extern "C" int pips_tokenmix_s(float* x, int seqs, int S, const float* ln1_w, const float* ln1_b, const float* w1,
                               const float* b1, const float* w2, const float* b2, const float* ln2_w, const float* ln2_b,
                               void* y_hi, void* y_lo, float* y_f32, void* stream) {
    if (!x || !ln1_w || !ln1_b || !w1 || !b1 || !w2 || !b2 || !ln2_w || !ln2_b) return fail("pips_tokenmix: null pointer");
    if (seqs <= 0) return fail("pips_tokenmix: no sequences");
    if (!y_hi && !y_f32) return fail("pips_tokenmix: no output buffer");
    if (S < 2 || S > PIPS_S_MAX) return fail("pips_tokenmix: S must be in 2..16");
    {
        // bf16 / bf16x3 precisions run the tensor-core kernel (tokenmix_tc.cu: both contractions as wgmma MMAs,
        // pipelined over the four channel tiles); PIPS_B200_TOKENMIX=simt keeps the CUDA-core kernels below, which are
        // also the fp32-precision path.
        static int use_tc = -1;
        if (use_tc < 0) {
            const char* e = getenv("PIPS_B200_TOKENMIX");
            use_tc = (e && e[0] == 's') ? 0 : 1;
        }
        if (use_tc && y_hi && !y_f32)
            return tokenmix_tc_launch(x, seqs, S, ln1_w, ln1_b, w1, b1, w2, b2, ln2_w, ln2_b, y_hi, y_lo, static_cast<cudaStream_t>(stream));
    }
    {
        cudaError_t e = S == 8 ? launch_pdl(tokenmix_kernel<true>, dim3(seqs), dim3(TM_THREADS), 0, static_cast<cudaStream_t>(stream), x, S,
                                             ln1_w, ln1_b, w1, b1, w2, b2, ln2_w, ln2_b, static_cast<__nv_bfloat16*>(y_hi),
                                             static_cast<__nv_bfloat16*>(y_lo), y_f32)
                      : S < 8 ? launch_pdl(tokenmix_kernel<false>, dim3(seqs), dim3(TM_THREADS), 0, static_cast<cudaStream_t>(stream), x, S,
                                            ln1_w, ln1_b, w1, b1, w2, b2, ln2_w, ln2_b, static_cast<__nv_bfloat16*>(y_hi),
                                            static_cast<__nv_bfloat16*>(y_lo), y_f32)
                               : launch_pdl(tokenmix16_kernel, dim3(seqs), dim3(2 * TM_THREADS), 0, static_cast<cudaStream_t>(stream), x,
                                            S, ln1_w, ln1_b, w1, b1, w2, b2, ln2_w, ln2_b, static_cast<__nv_bfloat16*>(y_hi),
                                            static_cast<__nv_bfloat16*>(y_lo), y_f32);
        if (e != cudaSuccess) return fail_cuda("pips_tokenmix", e);
    }
    LAUNCH_CHECK("pips_tokenmix");
    return 0;
}

extern "C" int pips_tokenmix(float* x, int seqs, const float* ln1_w, const float* ln1_b, const float* w1, const float* b1,
                             const float* w2, const float* b2, const float* ln2_w, const float* ln2_b,
                             void* y_hi, void* y_lo, float* y_f32, void* stream) {
    return pips_tokenmix_s(x, seqs, PIPS_S, ln1_w, ln1_b, w1, b1, w2, b2, ln2_w, ln2_b, y_hi, y_lo, y_f32, stream);
}

extern "C" int pips_ln_pool_s(const float* x, int seqs, int S, const float* ln_w, const float* ln_b, void* p_hi, void* p_lo,
                              float* p_f32, void* stream) {
    if (!x || !ln_w || !ln_b) return fail("pips_ln_pool: null pointer");
    if (seqs <= 0) return fail("pips_ln_pool: no sequences");
    if (!p_hi && !p_f32) return fail("pips_ln_pool: no output buffer");
    if (S < 2 || S > PIPS_S_MAX) return fail("pips_ln_pool: S must be in 2..16");
    {
        cudaError_t e = launch_pdl(ln_pool_kernel, dim3(seqs), dim3(TM_THREADS), 0, static_cast<cudaStream_t>(stream), x, S, ln_w, ln_b,
                                   static_cast<__nv_bfloat16*>(p_hi), static_cast<__nv_bfloat16*>(p_lo), p_f32);
        if (e != cudaSuccess) return fail_cuda("pips_ln_pool", e);
    }
    LAUNCH_CHECK("pips_ln_pool");
    return 0;
}

extern "C" int pips_ln_pool(const float* x, int seqs, const float* ln_w, const float* ln_b, void* p_hi, void* p_lo,
                            float* p_f32, void* stream) {
    return pips_ln_pool_s(x, seqs, PIPS_S, ln_w, ln_b, p_hi, p_lo, p_f32, stream);
}

extern "C" int pips_update(const float* delta, float* coords, const float* coords0, float* ffeats, const float* gn_w,
                           const float* gn_b, const float* wu, const float* bu, float* out_px, float stride, int B, int S,
                           int N, void* stream) {
    return pips_update_peer(delta, coords, coords0, ffeats, gn_w, gn_b, wu, bu, out_px, stride, B, S, N, nullptr, stream);
}

extern "C" int pips_update_peer(const float* delta, float* coords, const float* coords0, float* ffeats, const float* gn_w,
                                const float* gn_b, const float* wu, const float* bu, float* out_px, float stride, int B,
                                int S, int N, const pips_peer_out* peer, void* stream) {
    pips_peer_out po;
    po.n_peers = 0;
    po.n_offset = 0;
    po.n_total = N;
    if (peer && peer->n_peers > 0) {
        po = *peer;
        if (po.n_peers > PIPS_MAX_PEERS) return fail("pips_update: more than PIPS_MAX_PEERS ranks");
        if (po.n_offset < 0 || po.n_offset + N > po.n_total) return fail("pips_update: particle slice outside n_total");
        for (int r = 0; r < po.n_peers; ++r)
            if (!po.out[r] || (reinterpret_cast<uintptr_t>(po.out[r]) & 7)) return fail("pips_update: null or misaligned peer result");
    }
    if (!delta || !coords || !coords0 || !ffeats || !gn_w || !gn_b || !wu || !bu || !out_px) return fail("pips_update: null pointer");
    if (S < 2 || S > PIPS_S_MAX) return fail("pips_update: S must be in 2..16");
    if (B <= 0 || N <= 0) return fail("pips_update: empty problem");
    const int rows = B * N * S;
    const size_t smem = (128 * 129 + UP_ROWS * 132) * sizeof(float);
    static bool attr[kMaxDevices] = {};
    {
        cudaError_t e = ensure_dyn_smem(update_kernel, attr, static_cast<int>(smem));
        if (e != cudaSuccess) return fail_cuda("pips_update: smem attribute", e);
    }
    {
        cudaError_t e = launch_pdl(update_kernel, dim3((rows + UP_ROWS - 1) / UP_ROWS), dim3(256), smem, static_cast<cudaStream_t>(stream),
                                   delta, coords, coords0, ffeats, gn_w, gn_b, wu, bu, out_px, stride, B, S, N, po);
        if (e != cudaSuccess) return fail_cuda("pips_update", e);
    }
    LAUNCH_CHECK("pips_update");
    return 0;
}

extern "C" int pips_vis_head(const float* ffeats, const float* w, const float* b, float* vis, int B, int S, int N, void* stream) {
    if (!ffeats || !w || !b || !vis) return fail("pips_vis_head: null pointer");
    if (B <= 0 || N <= 0 || S <= 0) return fail("pips_vis_head: empty problem");
    const int rows = B * N * S;
    vis_head_kernel<<<(rows * 32 + 255) / 256, 256, 0, static_cast<cudaStream_t>(stream)>>>(ffeats, w, b, vis, B, S, N);
    LAUNCH_CHECK("pips_vis_head");
    return 0;
}
