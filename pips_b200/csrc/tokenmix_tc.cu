// Token mixing with the two small contractions on the tensor cores.
//
//   x (8 frames x 512 channels per track)
//   y = LN1(x);  h[c, j] = gelu(sum_s y[s, c] W1[j, s] + b1[j]);  z[c, s'] = sum_j h[c, j] W2[s', j] + b2[s'];
//   x += z;  out = LN2(x)                                                    (nets/pips.py:117, :93-109, :100)
//
// K = 8 and K = 32 are far too small for a conventional tensor-core GEMM, but with the CHANNELS as the MMA's M
// dimension each track is four 128-row tiles (two wgmma M = 64 blocks each) and the per-channel MLP becomes
//   GEMM1  H (128 x 32) = A1 (128 x 16) . B^T      A1 row c = [y_hi[0..8) | y_lo[0..8)]   (bf16, K-major, no swizzle)
//   GEMM2  Z (128 x 8)  = G  (128 x 64) . B^T      G  row c = [g_hi[0..32) | g_lo[0..32)]
// where the bf16x3 split is folded into K: B = [w_hi | w_hi] gives hi*hi + lo*hi in one MMA and B' = [w_lo | 0]
// adds hi*lo.  A handful of wgmma per tile replace 512 FMAs per channel; LayerNorm, GELU, the hi/lo splits and all
// global traffic stay on the CUDA cores (thread t owns channels 4t..4t+3 == row t of tile 0..3, so loads and
// stores are 16-byte vectors).  One CTA = 128 threads = one warpgroup; accumulators are wgmma register fragments:
// GELU is applied on the H fragment and written to the G operand in shared memory, GEMM2 of tile i runs while GEMM1
// of tile i+1 is issued, and the Z fragments return to the thread-per-row layout through shared memory (in G's place).
// 55 KB of shared memory per CTA -> 4 CTAs (16 warps) per SM.
#include "mixer_common.cuh"
#include "ptx.cuh"

namespace pips {

constexpr int TT_THREADS = 128;
constexpr int TT_CTAS_PER_SM = 4;
constexpr uint32_t TT_A1_TILE = 128 * 32;            // 4 KB: 128 rows x K=16 bf16
constexpr uint32_t TT_G_TILE = 128 * 128;            // 16 KB: 128 rows x K=64 bf16; later Z: 4 tiles x 128 rows x 8 fp32
constexpr uint32_t TT_OFF_A1 = 0;
constexpr uint32_t TT_OFF_X = TT_OFF_A1 + 4 * TT_A1_TILE;          // copy of the track's x for the residual (8 x 2 KB)
constexpr uint32_t TT_OFF_G = TT_OFF_X + 8 * 2048;
constexpr uint32_t TT_OFF_B1A = TT_OFF_G + TT_G_TILE;              // [w1_hi | w1_hi]  32 rows x 32 B
constexpr uint32_t TT_OFF_B1B = TT_OFF_B1A + 1024;                 // [w1_lo | 0]
constexpr uint32_t TT_OFF_B2A = TT_OFF_B1B + 1024;                 // [w2_hi | w2_hi]  8 rows x 128 B
constexpr uint32_t TT_OFF_B2B = TT_OFF_B2A + 1024;                 // [w2_lo | 0]
constexpr uint32_t TT_OFF_MISC = TT_OFF_B2B + 1024;                // reductions, biases
constexpr uint32_t TT_SMEM = TT_OFF_MISC + 512 + 128;              // + alignment slack; 4 CTAs: 4 x (52.6 + 1) KB <= 227 KB

// K-major operand without swizzle: 8-row x 16-byte core matrices; element (r, k) lives at
// (r / 8) * sbo + (k / 8) * 128 + (r % 8) * 16 + (k % 8) * 2.
__device__ __forceinline__ uint64_t wgmma_desc_nosw(uint32_t smem_addr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
    uint64_t d = 0;
    d |= static_cast<uint64_t>((smem_addr & 0x3FFFF) >> 4);
    d |= static_cast<uint64_t>(lbo_bytes >> 4) << 16;       // between core matrices along K
    d |= static_cast<uint64_t>(sbo_bytes >> 4) << 32;       // between 8-row groups; layout type 0 = no swizzle
    return d;
}
__device__ __forceinline__ uint32_t core_off(int r, int kcore, uint32_t sbo) {
    return static_cast<uint32_t>(r >> 3) * sbo + static_cast<uint32_t>(kcore) * 128 + static_cast<uint32_t>(r & 7) * 16;
}

// ---- 8-row statistics with a transposing butterfly: every lane contributes 8 partial sums (one per frame); three
// exchange steps halve the number of live values while doubling the lanes summed, two more finish the warp:
// 9 shuffles instead of 8 x 5.  Lane l ends with the warp total of row  4*bit4(l) + 2*bit3(l) + bit2(l).
__device__ __forceinline__ float warp_rowsum8(const float (&v)[8]) {
    const int lane = threadIdx.x & 31;
    float a[4], b[2];
    {
        const bool up = lane & 16;
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const float send = up ? v[i] : v[i + 4], keep = up ? v[i + 4] : v[i];
            a[i] = keep + __shfl_xor_sync(0xffffffffu, send, 16);
        }
    }
    {
        const bool up = lane & 8;
#pragma unroll
        for (int i = 0; i < 2; ++i) {
            const float send = up ? a[i] : a[i + 2], keep = up ? a[i + 2] : a[i];
            b[i] = keep + __shfl_xor_sync(0xffffffffu, send, 8);
        }
    }
    const bool up = lane & 4;
    float c = (up ? b[1] : b[0]) + __shfl_xor_sync(0xffffffffu, up ? b[0] : b[1], 4);
    c += __shfl_xor_sync(0xffffffffu, c, 2);
    c += __shfl_xor_sync(0xffffffffu, c, 1);
    return c;
}

// CTA-wide sums of 8 per-thread values (128 threads): v[s] <- total over the CTA.  `red` is [4 warps][8 rows].
__device__ __forceinline__ void cta_rowsum8(float (&v)[8], float (*red)[8]) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const float c = warp_rowsum8(v);
    __syncthreads();                                        // previous readers of `red` are done
    if ((lane & 3) == 0) red[warp][(lane >> 2) & 7] = c;
    __syncthreads();
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        const float4 r0 = *reinterpret_cast<const float4*>(&red[0][4 * h]), r1 = *reinterpret_cast<const float4*>(&red[1][4 * h]);
        const float4 r2 = *reinterpret_cast<const float4*>(&red[2][4 * h]), r3 = *reinterpret_cast<const float4*>(&red[3][4 * h]);
        v[4 * h + 0] = (r0.x + r1.x) + (r2.x + r3.x);
        v[4 * h + 1] = (r0.y + r1.y) + (r2.y + r3.y);
        v[4 * h + 2] = (r0.z + r1.z) + (r2.z + r3.z);
        v[4 * h + 3] = (r0.w + r1.w) + (r2.w + r3.w);
    }
}

// two-pass LayerNorm over the 512 channels of the 8 rows held as x[s][0..3] (biased variance, eps 1e-5); the
// per-element arithmetic is written on fp32 pairs
__device__ __forceinline__ void layernorm8_fast(const float (&x)[8][4], float (&y)[8][4], const float4 g, const float4 b, float (*red)[8]) {
    float m[8], q[8];
#pragma unroll
    for (int s = 0; s < 8; ++s) {
        const float2 t = add2(make_float2(x[s][0], x[s][1]), make_float2(x[s][2], x[s][3]));
        m[s] = t.x + t.y;
    }
    cta_rowsum8(m, red);
#pragma unroll
    for (int s = 0; s < 8; ++s) {
        m[s] *= (1.0f / 512.0f);
        const float2 nm = bcast2(-m[s]);
        const float2 d0 = add2(make_float2(x[s][0], x[s][1]), nm), d1 = add2(make_float2(x[s][2], x[s][3]), nm);
        const float2 t = fma2(d1, d1, mul2(d0, d0));
        q[s] = t.x + t.y;
    }
    cta_rowsum8(q, red);
    const float2 g0 = make_float2(g.x, g.y), g1 = make_float2(g.z, g.w), b0 = make_float2(b.x, b.y), b1 = make_float2(b.z, b.w);
#pragma unroll
    for (int s = 0; s < 8; ++s) {
        const float r = rsqrtf(q[s] * (1.0f / 512.0f) + 1e-5f);
        const float2 nm = bcast2(-m[s]), r2 = bcast2(r);
        const float2 o0 = fma2(mul2(add2(make_float2(x[s][0], x[s][1]), nm), r2), g0, b0);
        const float2 o1 = fma2(mul2(add2(make_float2(x[s][2], x[s][3]), nm), r2), g1, b1);
        y[s][0] = o0.x; y[s][1] = o0.y; y[s][2] = o1.x; y[s][3] = o1.y;
    }
}

__global__ void __launch_bounds__(TT_THREADS, TT_CTAS_PER_SM)
tokenmix_tc_kernel(float* __restrict__ x, int seqs, const float* __restrict__ ln1_w, const float* __restrict__ ln1_b,
                   const float* __restrict__ w1, const float* __restrict__ b1, const float* __restrict__ w2,
                   const float* __restrict__ b2, const float* __restrict__ ln2_w, const float* __restrict__ ln2_b,
                   __nv_bfloat16* __restrict__ y_hi, __nv_bfloat16* __restrict__ y_lo) {
    pdl_trigger();
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 127) & ~static_cast<uintptr_t>(127));
    const uint32_t sbase = smem_u32(smem);
    float (*red)[8] = reinterpret_cast<float (*)[8]>(smem + TT_OFF_MISC);
    float* s_b1 = reinterpret_cast<float*>(smem + TT_OFF_MISC + 128);
    float* s_b2 = s_b1 + 32;

    const int t = threadIdx.x, warp = t >> 5, lane = t & 31;
    const int frow = warp * 16 + (lane >> 2), fq = lane & 3;        // fragment row (+8, +64 m) and column pair of this thread

    // ---- one-time setup: weight operands
    for (int i = t; i < 32 * 16; i += TT_THREADS) {                 // GEMM1 B operands: row j, k in [0,16)
        const int j = i >> 4, k = i & 15;
        __nv_bfloat16 h, l;
        split_bf16(w1[j * 8 + (k & 7)], h, l);
        const uint32_t off = core_off(j, k >> 3, 256) + (k & 7) * 2;
        *reinterpret_cast<__nv_bfloat16*>(smem + TT_OFF_B1A + off) = h;                                   // [hi | hi]
        *reinterpret_cast<__nv_bfloat16*>(smem + TT_OFF_B1B + off) = k < 8 ? l : __float2bfloat16_rn(0.f); // [lo | 0]
    }
    for (int i = t; i < 8 * 64; i += TT_THREADS) {                  // GEMM2 B operands: row s', k in [0,64)
        const int r = i >> 6, k = i & 63;
        __nv_bfloat16 h, l;
        split_bf16(w2[r * 32 + (k & 31)], h, l);
        const uint32_t off = core_off(r, k >> 3, 1024) + (k & 7) * 2;
        *reinterpret_cast<__nv_bfloat16*>(smem + TT_OFF_B2A + off) = h;
        *reinterpret_cast<__nv_bfloat16*>(smem + TT_OFF_B2B + off) = k < 32 ? l : __float2bfloat16_rn(0.f);
    }
    if (t < 32) s_b1[t] = b1[t];
    if (t < 8) s_b2[t] = b2[t];
    fence_proxy_async_smem();
    __syncthreads();
    const uint64_t d_b1a = wgmma_desc_nosw(sbase + TT_OFF_B1A, 128, 256), d_b1b = wgmma_desc_nosw(sbase + TT_OFF_B1B, 128, 256);

    pdl_wait();                                             // x is written by the previous kernel (weights above are constants)
    // x of the track after the current one is fetched into registers while the current track's GELU phase runs; the
    // current x is dropped after LayerNorm 1 and parked in shared memory for the residual, so that both fit 128 registers
    float4 nx[8];
    if (static_cast<int>(blockIdx.x) < seqs) {
        const float* src = x + static_cast<size_t>(blockIdx.x) * 8 * 512 + t * 4;
#pragma unroll
        for (int s = 0; s < 8; ++s) nx[s] = *reinterpret_cast<const float4*>(src + s * 512);
    }
    const float4 g1 = __ldg(reinterpret_cast<const float4*>(ln1_w + t * 4)), c1 = __ldg(reinterpret_cast<const float4*>(ln1_b + t * 4));

    for (int seq = blockIdx.x; seq < seqs; seq += gridDim.x) {
        const size_t base = static_cast<size_t>(seq) * 8 * 512 + t * 4;
        {
            // a copy of this track's x for the residual at the end (cp.async, no registers held) -- re-reading it from L2
            // there exposed ~500 cycles of latency per track
            const uint32_t dst = sbase + TT_OFF_X + t * 16;
            const float* src = x + base;
#pragma unroll
            for (int sr = 0; sr < 8; ++sr)
                asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst + sr * 2048), "l"(src + sr * 512) : "memory");
            asm volatile("cp.async.commit_group;" ::: "memory");
        }
        {
            float xv[8][4], yv[8][4];
#pragma unroll
            for (int s = 0; s < 8; ++s) { xv[s][0] = nx[s].x; xv[s][1] = nx[s].y; xv[s][2] = nx[s].z; xv[s][3] = nx[s].w; }
            layernorm8_fast(xv, yv, g1, c1, red);

            // ---- A1: row t of tile i = [y_hi over the 8 frames | y_lo over the 8 frames] of channel 4t+i
            // (the previous track's MMAs were waited for before its Z was read)
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                uint32_t hw[4], lw[4];
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                    const float a = yv[2 * e][i], b = yv[2 * e + 1][i];
                    hw[e] = cvt_bf16x2(a, b);
                    lw[e] = cvt_bf16x2(a - __uint_as_float(hw[e] << 16), b - __uint_as_float(hw[e] & 0xffff0000u));
                }
                uint8_t* row = smem + TT_OFF_A1 + i * TT_A1_TILE;
                *reinterpret_cast<uint4*>(row + core_off(t, 0, 256)) = make_uint4(hw[0], hw[1], hw[2], hw[3]);
                *reinterpret_cast<uint4*>(row + core_off(t, 1, 256)) = make_uint4(lw[0], lw[1], lw[2], lw[3]);
            }
        }
        fence_proxy_async_smem();
        __syncthreads();
        if (seq + static_cast<int>(gridDim.x) < seqs) {      // next track's x: in flight during the GELU phase
            const float* src = x + static_cast<size_t>(seq + gridDim.x) * 8 * 512 + t * 4;
#pragma unroll
            for (int s = 0; s < 8; ++s) nx[s] = *reinterpret_cast<const float4*>(src + s * 512);
        }

        // ---- per tile: GEMM1 -> GELU(H_i) on the fragment -> G -> GEMM2_i (asynchronous: it runs while GEMM1 of tile
        // i+1 is issued; the wait after that GEMM1 also retires it, which frees G)
        float z[4][2][4];
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            float h[2][16];
            wgmma_fence();
#pragma unroll
            for (int m = 0; m < 2; ++m) {
                const uint64_t a = wgmma_desc_nosw(sbase + TT_OFF_A1 + i * TT_A1_TILE + m * 2048, 128, 256);
                wgmma_n32(h[m], a, d_b1a, 0);
                wgmma_n32(h[m], a, d_b1b, 1);
            }
            wgmma_commit();
            wgmma_wait<0>();
            wgmma_acc_ready(h[0]);
            wgmma_acc_ready(h[1]);
#pragma unroll
            for (int m = 0; m < 2; ++m) {
#pragma unroll
                for (int hh = 0; hh < 2; ++hh) {
                    uint8_t* row = smem + TT_OFF_G + core_off(64 * m + frow + 8 * hh, 0, 1024) + fq * 4;
#pragma unroll
                    for (int j = 0; j < 4; ++j) {
                        const float2 bj = *reinterpret_cast<const float2*>(s_b1 + 8 * j + 2 * fq);
                        const float2 g = gelu_fast2_abs(add2(make_float2(h[m][4 * j + 2 * hh], h[m][4 * j + 2 * hh + 1]), bj));
                        const uint32_t hw = cvt_bf16x2(g.x, g.y);
                        const float2 lo = fma2(make_float2(__uint_as_float(hw << 16), __uint_as_float(hw & 0xffff0000u)), bcast2(-1.0f), g);
                        *reinterpret_cast<uint32_t*>(row + j * 128) = hw;
                        *reinterpret_cast<uint32_t*>(row + (j + 4) * 128) = cvt_bf16x2(lo.x, lo.y);
                    }
                }
            }
            fence_proxy_async_smem();
            __syncthreads();
            wgmma_fence();
#pragma unroll
            for (int m = 0; m < 2; ++m) {
                const uint32_t ga = sbase + TT_OFF_G + m * 8192;
#pragma unroll
                for (int k = 0; k < 4; ++k)                      // [g_hi | g_lo] . [w2_hi | w2_hi]
                    wgmma_n8(z[i][m], wgmma_desc_nosw(ga + k * 256, 128, 1024), wgmma_desc_nosw(sbase + TT_OFF_B2A + k * 256, 128, 1024), k != 0);
#pragma unroll
                for (int k = 0; k < 2; ++k)                      // g_hi . w2_lo
                    wgmma_n8(z[i][m], wgmma_desc_nosw(ga + k * 256, 128, 1024), wgmma_desc_nosw(sbase + TT_OFF_B2B + k * 256, 128, 1024), 1);
            }
            wgmma_commit();
        }
        wgmma_wait<0>();
#pragma unroll
        for (int i = 0; i < 4; ++i) { wgmma_acc_ready(z[i][0]); wgmma_acc_ready(z[i][1]); }
        __syncthreads();                                     // every warp's GEMM2 has read G: Z takes its place
        {
            float* zs = reinterpret_cast<float*>(smem + TT_OFF_G);         // [tile][row][frame]
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
                for (int m = 0; m < 2; ++m)
#pragma unroll
                    for (int hh = 0; hh < 2; ++hh)
                        *reinterpret_cast<float2*>(zs + (i * 128 + 64 * m + frow + 8 * hh) * 8 + 2 * fq) =
                            make_float2(z[i][m][2 * hh], z[i][m][2 * hh + 1]);
        }
        __syncthreads();
        // ---- residual, LN2, outputs
        float xv[8][4];
        asm volatile("cp.async.wait_group 0;" ::: "memory");
#pragma unroll
        for (int sr = 0; sr < 8; ++sr) {                     // this thread's own copies: no CTA-wide barrier needed
            const float4 v = *reinterpret_cast<const float4*>(smem + TT_OFF_X + sr * 2048 + t * 16);
            xv[sr][0] = v.x; xv[sr][1] = v.y; xv[sr][2] = v.z; xv[sr][3] = v.w;
        }
        {
            const float* zs = reinterpret_cast<const float*>(smem + TT_OFF_G);
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const float4 z0 = *reinterpret_cast<const float4*>(zs + (i * 128 + t) * 8), z1 = *reinterpret_cast<const float4*>(zs + (i * 128 + t) * 8 + 4);
                const float zz[8] = {z0.x, z0.y, z0.z, z0.w, z1.x, z1.y, z1.z, z1.w};
#pragma unroll
                for (int s = 0; s < 8; ++s) xv[s][i] += zz[s] + s_b2[s];
            }
        }
#pragma unroll
        for (int s = 0; s < 8; ++s)
            *reinterpret_cast<float4*>(x + base + s * 512) = make_float4(xv[s][0], xv[s][1], xv[s][2], xv[s][3]);
        {
            float yv[8][4];
            const float4 g2 = __ldg(reinterpret_cast<const float4*>(ln2_w + t * 4)), c2 = __ldg(reinterpret_cast<const float4*>(ln2_b + t * 4));
            layernorm8_fast(xv, yv, g2, c2, red);            // its __syncthreads also order the Z reads before the next track's G
#pragma unroll
            for (int s = 0; s < 8; ++s) store_row4(yv[s], base + s * 512, y_hi, y_lo, nullptr);
        }
    }
}

}  // namespace pips

using namespace pips;

// called by pips_tokenmix (mixer_simt.cu) for the bf16 / bf16x3 precisions
int tokenmix_tc_launch(float* x, int seqs, const float* ln1_w, const float* ln1_b, const float* w1, const float* b1, const float* w2,
                       const float* b2, const float* ln2_w, const float* ln2_b, void* y_hi, void* y_lo, cudaStream_t st) {
    static bool attr[kMaxDevices] = {};
    {
        cudaError_t e = ensure_dyn_smem(tokenmix_tc_kernel, attr, static_cast<int>(TT_SMEM));
        if (e != cudaSuccess) return fail_cuda("pips_tokenmix (tc): smem attribute", e);
    }
    const int cap = TT_CTAS_PER_SM * sm_count();
    const int grid = seqs < cap ? seqs : cap;
    cudaError_t e = launch_pdl(tokenmix_tc_kernel, dim3(grid), dim3(TT_THREADS), TT_SMEM, st, x, seqs, ln1_w, ln1_b, w1, b1, w2, b2, ln2_w,
                               ln2_b, static_cast<__nv_bfloat16*>(y_hi), static_cast<__nv_bfloat16*>(y_lo));
    if (e == cudaSuccess) e = cudaGetLastError();
    return e == cudaSuccess ? 0 : fail_cuda("pips_tokenmix (tc): launch", e);
}

// explicit entry point of the tensor-core variant (same contract as pips_tokenmix with bf16 outputs)
extern "C" int pips_tokenmix_tc(float* x, int seqs, const float* ln1_w, const float* ln1_b, const float* w1, const float* b1,
                                const float* w2, const float* b2, const float* ln2_w, const float* ln2_b, void* y_hi, void* y_lo,
                                void* stream) {
    if (!x || !ln1_w || !ln1_b || !w1 || !b1 || !w2 || !b2 || !ln2_w || !ln2_b || !y_hi) return fail("pips_tokenmix_tc: null pointer");
    if (seqs <= 0) return fail("pips_tokenmix_tc: no sequences");
    return tokenmix_tc_launch(x, seqs, ln1_w, ln1_b, w1, b1, w2, b2, ln2_w, ln2_b, y_hi, y_lo, static_cast<cudaStream_t>(stream));
}
