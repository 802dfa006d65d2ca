// Token mixing with the two small contractions on the tensor cores.
//
//   x (S frames x 512 channels per track, 2 <= S <= 16)
//   y = LN1(x);  h[c, j] = gelu(sum_s y[s, c] W1[j, s] + b1[j]);  z[c, s'] = sum_j h[c, j] W2[s', j] + b2[s'];
//   x += z;  out = LN2(x)                                                    (nets/pips.py:117, :93-109, :100)
//
// K = S and K = 4S are far too small for a conventional tensor-core GEMM, but with the CHANNELS as the MMA's M
// dimension each track is four 128-row tiles (two wgmma M = 64 blocks each) and the per-channel MLP becomes
//   GEMM1  H (128 x 4P) = A1 (128 x 2P) . B^T      A1 row c = [y_hi[0..P) | y_lo[0..P)]   (bf16, K-major, no swizzle)
//   GEMM2  Z (128 x P)  = G  (128 x 8P) . B^T      G  row c = [g_hi[0..4P) | g_lo[0..4P)]
// over P = 8 padded frames (S = 2..8) or P = 16 (S = 9..16): the frame axis is padded with zero token-mixing weights and
// the hidden axis 4S with zero weights and biases up to 4P (GELU(0) = 0, so the padding adds exact zeros).  Padded
// frames are never loaded or stored -- their rows in x belong to the next track -- and hold x = 0 in registers.
// The bf16x3 split is folded into K: B = [w_hi | w_hi] gives hi*hi + lo*hi in one pass and B' = [w_lo | 0] adds hi*lo.
// A handful of wgmma per tile replace 8P^2 FMAs per channel; LayerNorm, GELU, the hi/lo splits and all global traffic
// stay on the CUDA cores.  One warpgroup per 8 padded frames (kWG = P / 8): thread t of warpgroup w owns channels
// 4t..4t+3 (row t of tiles 0..3) of frames 8w..8w+7, so loads and stores are 16-byte vectors and LayerNorm sums stay
// inside a warpgroup.  Every warpgroup writes its frames into the shared A1 tiles; warpgroup w then runs tiles
// w*4/kWG .. of both GEMMs on its own G buffer.  Accumulators are wgmma register fragments: GELU is applied on the H
// fragment and written to the G operand in shared memory, GEMM2 of tile i runs while GEMM1 of tile i+1 is issued, and
// the Z fragments return to the thread-per-row layout through shared memory (in G's place).
// P = 8: 55 KB of shared memory per 128-thread CTA -> 4 CTAs (16 warps) per SM at S = 8; 3 at S < 8, whose per-frame
// guards need more than 128 registers.
// P = 16: 145 KB per 256-thread CTA -> 1 CTA (8 warps) per SM.
#include "mixer_common.cuh"
#include "ptx.cuh"

namespace pips {

template <int kWG>
struct TtCfg {
    static constexpr int kThreads = 128 * kWG;
    static constexpr int kCtasPerSm = kWG == 1 ? 4 : 1;
    static constexpr int kCtasPerSmPadded = kWG == 1 ? 3 : 1;     // S < 8: the frame guards need > 128 registers
    static constexpr int kP = 8 * kWG;                             // padded frames
    static constexpr int kHid = 4 * kP;                            // padded hidden width
    static constexpr int kTiles = 4 / kWG;                         // channel tiles per warpgroup
    static constexpr uint32_t kSboA = 256 * kWG;                   // A1 / B1 rows: K = 2P bf16
    static constexpr uint32_t kSboG = 1024 * kWG;                  // G / B2 rows: K = 8P bf16
    static constexpr uint32_t kA1Tile = 128 * kSboA / 8;           // 128 rows
    static constexpr uint32_t kGTile = 128 * kSboG / 8;            // 128 rows, one per warpgroup; later Z: 4 tiles x 128 rows x P fp32
    static constexpr uint32_t kB1 = kHid * kSboA / 8;              // [w1_hi | w1_hi]: 4P rows
    static constexpr uint32_t kB2 = kP * kSboG / 8;                // [w2_hi | w2_hi]: P rows
    static constexpr uint32_t kOffA1 = 0;
    static constexpr uint32_t kOffX = kOffA1 + 4 * kA1Tile;        // copy of the track's x for the residual (P x 2 KB)
    static constexpr uint32_t kOffG = kOffX + kP * 2048;
    static constexpr uint32_t kOffB1A = kOffG + kWG * kGTile;
    static constexpr uint32_t kOffB1B = kOffB1A + kB1;             // [w1_lo | 0]
    static constexpr uint32_t kOffB2A = kOffB1B + kB1;
    static constexpr uint32_t kOffB2B = kOffB2A + kB2;             // [w2_lo | 0]
    static constexpr uint32_t kOffMisc = kOffB2B + kB2;            // reductions [4 kWG warps][8], b1 [4P], b2 [P]
    static constexpr uint32_t kSmem = kOffMisc + 512 * kWG + 128;  // + alignment slack
    static_assert(4 * 128 * kP * 4 <= kWG * kGTile, "Z must fit in G's place");
};
static_assert(TtCfg<1>::kSmem * 4 <= 227 * 1024, "4 CTAs of the 8-frame kernel per SM");
static_assert(TtCfg<2>::kSmem <= 227 * 1024, "16-frame kernel exceeds the shared memory of an SM");

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

// Warpgroup-wide sums of 8 per-thread values: v[s] <- total over the thread's warpgroup (128 threads), every
// warpgroup of the CTA at once.  `red` is [warps of the CTA][8 rows].
template <int kWG>
__device__ __forceinline__ void cta_rowsum8(float (&v)[8], float (*red)[8]) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, w0 = kWG == 1 ? 0 : warp & ~3;
    const float c = warp_rowsum8(v);
    __syncthreads();                                        // previous readers of `red` are done
    if ((lane & 3) == 0) red[warp][(lane >> 2) & 7] = c;
    __syncthreads();
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        const float4 r0 = *reinterpret_cast<const float4*>(&red[w0 + 0][4 * h]), r1 = *reinterpret_cast<const float4*>(&red[w0 + 1][4 * h]);
        const float4 r2 = *reinterpret_cast<const float4*>(&red[w0 + 2][4 * h]), r3 = *reinterpret_cast<const float4*>(&red[w0 + 3][4 * h]);
        v[4 * h + 0] = (r0.x + r1.x) + (r2.x + r3.x);
        v[4 * h + 1] = (r0.y + r1.y) + (r2.y + r3.y);
        v[4 * h + 2] = (r0.z + r1.z) + (r2.z + r3.z);
        v[4 * h + 3] = (r0.w + r1.w) + (r2.w + r3.w);
    }
}

// two-pass LayerNorm over the 512 channels of the 8 rows held as x[s][0..3] (biased variance, eps 1e-5); the
// per-element arithmetic is written on fp32 pairs
template <int kWG>
__device__ __forceinline__ void layernorm8_fast(const float (&x)[8][4], float (&y)[8][4], const float4 g, const float4 b, float (*red)[8]) {
    float m[8], q[8];
#pragma unroll
    for (int s = 0; s < 8; ++s) {
        const float2 t = add2(make_float2(x[s][0], x[s][1]), make_float2(x[s][2], x[s][3]));
        m[s] = t.x + t.y;
    }
    cta_rowsum8<kWG>(m, red);
#pragma unroll
    for (int s = 0; s < 8; ++s) {
        m[s] *= (1.0f / 512.0f);
        const float2 nm = bcast2(-m[s]);
        const float2 d0 = add2(make_float2(x[s][0], x[s][1]), nm), d1 = add2(make_float2(x[s][2], x[s][3]), nm);
        const float2 t = fma2(d1, d1, mul2(d0, d0));
        q[s] = t.x + t.y;
    }
    cta_rowsum8<kWG>(q, red);
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

// the two GEMMs' MMA shapes: N = 4P for GEMM1, N = P for GEMM2
template <int kWG>
__device__ __forceinline__ void mma_h(float (&d)[16 * kWG], uint64_t a, uint64_t b, uint32_t acc) {
    if constexpr (kWG == 1) wgmma_n32(d, a, b, acc);
    else wgmma_n64(d, a, b, acc);
}
template <int kWG>
__device__ __forceinline__ void mma_z(float (&d)[4 * kWG], uint64_t a, uint64_t b, uint32_t acc) {
    if constexpr (kWG == 1) wgmma_n8(d, a, b, acc);
    else wgmma_n16(d, a, b, acc);
}
// barrier of one warpgroup (the whole CTA when it has one)
template <int kWG>
__device__ __forceinline__ void wg_sync(int wg) {
    if constexpr (kWG == 1) __syncthreads();
    else named_bar_sync(1 + wg, 128);
}

// kFull: S == P, no padded frames (S = 8 and S = 16 compile without the per-frame guards)
template <int kWG, bool kFull>
__global__ void __launch_bounds__(TtCfg<kWG>::kThreads, kFull ? TtCfg<kWG>::kCtasPerSm : TtCfg<kWG>::kCtasPerSmPadded)
tokenmix_tc_kernel(float* __restrict__ x, int seqs, int s_arg, const float* __restrict__ ln1_w, const float* __restrict__ ln1_b,
                   const float* __restrict__ w1, const float* __restrict__ b1, const float* __restrict__ w2,
                   const float* __restrict__ b2, const float* __restrict__ ln2_w, const float* __restrict__ ln2_b,
                   __nv_bfloat16* __restrict__ y_hi, __nv_bfloat16* __restrict__ y_lo) {
    using Cfg = TtCfg<kWG>;
    constexpr int P = Cfg::kP, HID = Cfg::kHid;
    const int S = kFull ? P : s_arg;
    pdl_trigger();
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 127) & ~static_cast<uintptr_t>(127));
    const uint32_t sbase = smem_u32(smem);
    float (*red)[8] = reinterpret_cast<float (*)[8]>(smem + Cfg::kOffMisc);
    float* s_b1 = reinterpret_cast<float*>(smem + Cfg::kOffMisc + 128 * kWG);
    float* s_b2 = s_b1 + HID;

    const int wg = kWG == 1 ? 0 : threadIdx.x >> 7, t = threadIdx.x & 127, warp = t >> 5, lane = t & 31;
    const int frow = warp * 16 + (lane >> 2), fq = lane & 3;        // fragment row (+8, +64 m) and column pair of this thread
    const int f0 = 8 * wg;                                          // this thread's frames f0 .. f0+7 (f < S are real)

    // ---- one-time setup: weight operands, zero outside the S x 4S weights
    for (int i = threadIdx.x; i < HID * 2 * P; i += Cfg::kThreads) {      // GEMM1 B operands: row j, k in [0,2P)
        const int j = i / (2 * P), k = i % (2 * P), s = k % P;
        __nv_bfloat16 h, l;
        split_bf16(j < 4 * S && s < S ? w1[j * S + s] : 0.f, h, l);
        const uint32_t off = core_off(j, k >> 3, Cfg::kSboA) + (k & 7) * 2;
        *reinterpret_cast<__nv_bfloat16*>(smem + Cfg::kOffB1A + off) = h;                                   // [hi | hi]
        *reinterpret_cast<__nv_bfloat16*>(smem + Cfg::kOffB1B + off) = k < P ? l : __float2bfloat16_rn(0.f); // [lo | 0]
    }
    for (int i = threadIdx.x; i < P * 8 * P; i += Cfg::kThreads) {        // GEMM2 B operands: row s', k in [0,8P)
        const int r = i / (8 * P), k = i % (8 * P), j = k % HID;
        __nv_bfloat16 h, l;
        split_bf16(r < S && j < 4 * S ? w2[r * 4 * S + j] : 0.f, h, l);
        const uint32_t off = core_off(r, k >> 3, Cfg::kSboG) + (k & 7) * 2;
        *reinterpret_cast<__nv_bfloat16*>(smem + Cfg::kOffB2A + off) = h;
        *reinterpret_cast<__nv_bfloat16*>(smem + Cfg::kOffB2B + off) = k < HID ? l : __float2bfloat16_rn(0.f);
    }
    if (threadIdx.x < HID) s_b1[threadIdx.x] = static_cast<int>(threadIdx.x) < 4 * S ? b1[threadIdx.x] : 0.f;
    if (threadIdx.x < P) s_b2[threadIdx.x] = static_cast<int>(threadIdx.x) < S ? b2[threadIdx.x] : 0.f;
    fence_proxy_async_smem();
    __syncthreads();

    pdl_wait();                                             // x is written by the previous kernel (weights above are constants)
    // x of the track after the current one is fetched into registers while the current track's GELU phase runs; the
    // current x is dropped after LayerNorm 1 and parked in shared memory for the residual, so that both fit the
    // register budget.  Padded frames hold zeros and are never loaded.
    float4 nx[8];
#pragma unroll
    for (int s = 0; s < 8; ++s) nx[s] = make_float4(0.f, 0.f, 0.f, 0.f);
    if (static_cast<int>(blockIdx.x) < seqs) {
        const float* src = x + static_cast<size_t>(blockIdx.x) * S * 512 + t * 4;
#pragma unroll
        for (int s = 0; s < 8; ++s)
            if (f0 + s < S) nx[s] = *reinterpret_cast<const float4*>(src + (f0 + s) * 512);
    }
    const float4 g1 = __ldg(reinterpret_cast<const float4*>(ln1_w + t * 4)), c1 = __ldg(reinterpret_cast<const float4*>(ln1_b + t * 4));

    for (int seq = blockIdx.x; seq < seqs; seq += gridDim.x) {
        const size_t base = static_cast<size_t>(seq) * S * 512 + t * 4;
        {
            // a copy of this track's x for the residual at the end (cp.async, no registers held) -- re-reading it from L2
            // there exposed ~500 cycles of latency per track
            const uint32_t dst = sbase + Cfg::kOffX + t * 16;
            const float* src = x + base;
#pragma unroll
            for (int sr = 0; sr < 8; ++sr)
                if (f0 + sr < S)
                    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst + (f0 + sr) * 2048), "l"(src + (f0 + sr) * 512) : "memory");
            asm volatile("cp.async.commit_group;" ::: "memory");
        }
        {
            float xv[8][4], yv[8][4];
#pragma unroll
            for (int s = 0; s < 8; ++s) { xv[s][0] = nx[s].x; xv[s][1] = nx[s].y; xv[s][2] = nx[s].z; xv[s][3] = nx[s].w; }
            layernorm8_fast<kWG>(xv, yv, g1, c1, red);

            // ---- A1: row t of tile i = [y_hi over the P frames | y_lo over the P frames] of channel 4t+i; this
            // warpgroup's 8 frames are core matrix wg of each half
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
                uint8_t* row = smem + Cfg::kOffA1 + i * Cfg::kA1Tile;
                *reinterpret_cast<uint4*>(row + core_off(t, wg, Cfg::kSboA)) = make_uint4(hw[0], hw[1], hw[2], hw[3]);
                *reinterpret_cast<uint4*>(row + core_off(t, kWG + wg, Cfg::kSboA)) = make_uint4(lw[0], lw[1], lw[2], lw[3]);
            }
        }
        fence_proxy_async_smem();
        __syncthreads();
        if (seq + static_cast<int>(gridDim.x) < seqs) {      // next track's x: in flight during the GELU phase
            const float* src = x + static_cast<size_t>(seq + gridDim.x) * S * 512 + t * 4;
#pragma unroll
            for (int s = 0; s < 8; ++s)
                if (f0 + s < S) nx[s] = *reinterpret_cast<const float4*>(src + (f0 + s) * 512);
        }

        // ---- per tile of this warpgroup: GEMM1 -> GELU(H_i) on the fragment -> G -> GEMM2_i (asynchronous: it runs
        // while GEMM1 of tile i+1 is issued; the wait after that GEMM1 also retires it, which frees G)
        const uint32_t g_off = Cfg::kOffG + wg * Cfg::kGTile;
        float z[Cfg::kTiles][2][P / 2];
#pragma unroll
        for (int ii = 0; ii < Cfg::kTiles; ++ii) {
            const int i = wg * Cfg::kTiles + ii;
            float h[2][HID / 2];
            wgmma_fence();
#pragma unroll
            for (int m = 0; m < 2; ++m) {
#pragma unroll
                for (int k = 0; k < kWG; ++k) {                // K = 2P in steps of 16: [y_hi | y_lo]
                    const uint64_t a = wgmma_desc_nosw(sbase + Cfg::kOffA1 + i * Cfg::kA1Tile + m * 8 * Cfg::kSboA + k * 256, 128, Cfg::kSboA);
                    mma_h<kWG>(h[m], a, wgmma_desc_nosw(sbase + Cfg::kOffB1A + k * 256, 128, Cfg::kSboA), k != 0);
                    if (2 * k < kWG)                           // [w_lo | 0] is zero over the y_lo half
                        mma_h<kWG>(h[m], a, wgmma_desc_nosw(sbase + Cfg::kOffB1B + k * 256, 128, Cfg::kSboA), 1);
                }
            }
            wgmma_commit();
            wgmma_wait<0>();
            wgmma_acc_ready(h[0]);
            wgmma_acc_ready(h[1]);
#pragma unroll
            for (int m = 0; m < 2; ++m) {
#pragma unroll
                for (int hh = 0; hh < 2; ++hh) {
                    uint8_t* row = smem + g_off + core_off(64 * m + frow + 8 * hh, 0, Cfg::kSboG) + fq * 4;
#pragma unroll
                    for (int j = 0; j < HID / 8; ++j) {
                        const float2 bj = *reinterpret_cast<const float2*>(s_b1 + 8 * j + 2 * fq);
                        const float2 g = gelu_fast2_abs(add2(make_float2(h[m][4 * j + 2 * hh], h[m][4 * j + 2 * hh + 1]), bj));
                        const uint32_t hw = cvt_bf16x2(g.x, g.y);
                        const float2 lo = fma2(make_float2(__uint_as_float(hw << 16), __uint_as_float(hw & 0xffff0000u)), bcast2(-1.0f), g);
                        *reinterpret_cast<uint32_t*>(row + j * 128) = hw;
                        *reinterpret_cast<uint32_t*>(row + (j + HID / 8) * 128) = cvt_bf16x2(lo.x, lo.y);
                    }
                }
            }
            fence_proxy_async_smem();
            wg_sync<kWG>(wg);
            wgmma_fence();
#pragma unroll
            for (int m = 0; m < 2; ++m) {
                const uint32_t ga = sbase + g_off + m * 8 * Cfg::kSboG;
#pragma unroll
                for (int k = 0; k < P / 2; ++k)                // [g_hi | g_lo] . [w2_hi | w2_hi]
                    mma_z<kWG>(z[ii][m], wgmma_desc_nosw(ga + k * 256, 128, Cfg::kSboG), wgmma_desc_nosw(sbase + Cfg::kOffB2A + k * 256, 128, Cfg::kSboG), k != 0);
#pragma unroll
                for (int k = 0; k < P / 4; ++k)                // g_hi . w2_lo
                    mma_z<kWG>(z[ii][m], wgmma_desc_nosw(ga + k * 256, 128, Cfg::kSboG), wgmma_desc_nosw(sbase + Cfg::kOffB2B + k * 256, 128, Cfg::kSboG), 1);
            }
            wgmma_commit();
        }
        wgmma_wait<0>();
#pragma unroll
        for (int ii = 0; ii < Cfg::kTiles; ++ii) { wgmma_acc_ready(z[ii][0]); wgmma_acc_ready(z[ii][1]); }
        __syncthreads();                                     // every warp's GEMM2 has read G: Z takes its place
        {
            float* zs = reinterpret_cast<float*>(smem + Cfg::kOffG);       // [tile][row][frame]
#pragma unroll
            for (int ii = 0; ii < Cfg::kTiles; ++ii)
#pragma unroll
                for (int m = 0; m < 2; ++m)
#pragma unroll
                    for (int hh = 0; hh < 2; ++hh)
#pragma unroll
                        for (int j = 0; j < kWG; ++j)
                            *reinterpret_cast<float2*>(zs + ((wg * Cfg::kTiles + ii) * 128 + 64 * m + frow + 8 * hh) * P + 8 * j + 2 * fq) =
                                make_float2(z[ii][m][4 * j + 2 * hh], z[ii][m][4 * j + 2 * hh + 1]);
        }
        __syncthreads();
        // ---- residual, LN2, outputs
        float xv[8][4];
        asm volatile("cp.async.wait_group 0;" ::: "memory");
#pragma unroll
        for (int sr = 0; sr < 8; ++sr) {                     // this thread's own copies: no CTA-wide barrier needed
            float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
            if (f0 + sr < S) v = *reinterpret_cast<const float4*>(smem + Cfg::kOffX + (f0 + sr) * 2048 + t * 16);
            xv[sr][0] = v.x; xv[sr][1] = v.y; xv[sr][2] = v.z; xv[sr][3] = v.w;
        }
        {
            const float* zs = reinterpret_cast<const float*>(smem + Cfg::kOffG);
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const float* zr = zs + (i * 128 + t) * P + f0;
                const float4 z0 = *reinterpret_cast<const float4*>(zr), z1 = *reinterpret_cast<const float4*>(zr + 4);
                const float zz[8] = {z0.x, z0.y, z0.z, z0.w, z1.x, z1.y, z1.z, z1.w};
#pragma unroll
                for (int s = 0; s < 8; ++s) xv[s][i] += zz[s] + s_b2[f0 + s];
            }
        }
#pragma unroll
        for (int s = 0; s < 8; ++s)
            if (f0 + s < S) *reinterpret_cast<float4*>(x + base + (f0 + s) * 512) = make_float4(xv[s][0], xv[s][1], xv[s][2], xv[s][3]);
        {
            float yv[8][4];
            const float4 g2 = __ldg(reinterpret_cast<const float4*>(ln2_w + t * 4)), c2 = __ldg(reinterpret_cast<const float4*>(ln2_b + t * 4));
            layernorm8_fast<kWG>(xv, yv, g2, c2, red);            // its __syncthreads also order the Z reads before the next track's G
#pragma unroll
            for (int s = 0; s < 8; ++s)
                if (f0 + s < S) store_row4(yv[s], base + (f0 + s) * 512, y_hi, y_lo, nullptr);
        }
    }
}

template <int kWG, bool kFull>
static int tokenmix_tc_run(float* x, int seqs, int S, const float* ln1_w, const float* ln1_b, const float* w1, const float* b1,
                           const float* w2, const float* b2, const float* ln2_w, const float* ln2_b, void* y_hi, void* y_lo,
                           cudaStream_t st) {
    using Cfg = TtCfg<kWG>;
    static bool attr[kMaxDevices] = {};
    {
        cudaError_t e = ensure_dyn_smem(tokenmix_tc_kernel<kWG, kFull>, attr, static_cast<int>(Cfg::kSmem));
        if (e != cudaSuccess) return fail_cuda("pips_tokenmix (tc): smem attribute", e);
    }
    const int cap = (kFull ? Cfg::kCtasPerSm : Cfg::kCtasPerSmPadded) * sm_count();
    const int grid = seqs < cap ? seqs : cap;
    cudaError_t e = launch_pdl(tokenmix_tc_kernel<kWG, kFull>, dim3(grid), dim3(Cfg::kThreads), Cfg::kSmem, st, x, seqs, S, ln1_w, ln1_b,
                               w1, b1, w2, b2, ln2_w, ln2_b, static_cast<__nv_bfloat16*>(y_hi), static_cast<__nv_bfloat16*>(y_lo));
    if (e == cudaSuccess) e = cudaGetLastError();
    return e == cudaSuccess ? 0 : fail_cuda("pips_tokenmix (tc): launch", e);
}

}  // namespace pips

using namespace pips;

// called by pips_tokenmix_s (mixer_simt.cu) for the bf16 / bf16x3 precisions; 2 <= S <= PIPS_S_MAX
int tokenmix_tc_launch(float* x, int seqs, int S, const float* ln1_w, const float* ln1_b, const float* w1, const float* b1,
                       const float* w2, const float* b2, const float* ln2_w, const float* ln2_b, void* y_hi, void* y_lo,
                       cudaStream_t st) {
    if (S == 8) return tokenmix_tc_run<1, true>(x, seqs, S, ln1_w, ln1_b, w1, b1, w2, b2, ln2_w, ln2_b, y_hi, y_lo, st);
    if (S < 8) return tokenmix_tc_run<1, false>(x, seqs, S, ln1_w, ln1_b, w1, b1, w2, b2, ln2_w, ln2_b, y_hi, y_lo, st);
    if (S == 16) return tokenmix_tc_run<2, true>(x, seqs, S, ln1_w, ln1_b, w1, b1, w2, b2, ln2_w, ln2_b, y_hi, y_lo, st);
    return tokenmix_tc_run<2, false>(x, seqs, S, ln1_w, ln1_b, w1, b1, w2, b2, ln2_w, ln2_b, y_hi, y_lo, st);
}

// explicit entry points of the tensor-core variant (same contract as pips_tokenmix_s with bf16 outputs)
extern "C" int pips_tokenmix_tc_s(float* x, int seqs, int S, const float* ln1_w, const float* ln1_b, const float* w1,
                                  const float* b1, const float* w2, const float* b2, const float* ln2_w, const float* ln2_b,
                                  void* y_hi, void* y_lo, void* stream) {
    if (!x || !ln1_w || !ln1_b || !w1 || !b1 || !w2 || !b2 || !ln2_w || !ln2_b || !y_hi) return fail("pips_tokenmix_tc: null pointer");
    if (seqs <= 0) return fail("pips_tokenmix_tc: no sequences");
    if (S < 2 || S > PIPS_S_MAX) return fail("pips_tokenmix_tc: S must be in 2..16");
    return tokenmix_tc_launch(x, seqs, S, ln1_w, ln1_b, w1, b1, w2, b2, ln2_w, ln2_b, y_hi, y_lo, static_cast<cudaStream_t>(stream));
}

extern "C" int pips_tokenmix_tc(float* x, int seqs, const float* ln1_w, const float* ln1_b, const float* w1, const float* b1,
                                const float* w2, const float* b2, const float* ln2_w, const float* ln2_b, void* y_hi, void* y_lo,
                                void* stream) {
    return pips_tokenmix_tc_s(x, seqs, PIPS_S, ln1_w, ln1_b, w1, b1, w2, b2, ln2_w, ln2_b, y_hi, y_lo, stream);
}
