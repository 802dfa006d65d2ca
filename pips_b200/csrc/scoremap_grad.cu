// Backward of the fused score-map loss (scoremap_loss.cu): the gradients of
//
//   loss = sum_{i, r kept} softplus(-s_i[r,t]) / (eps+K)  +  sum_{i, r kept, p != t} softplus(s_i[r,p]) / (eps+K(P-1))
//
// with s_i[r,p] = <F_i[r], G[f(r),p]> (rows r = (b,s,n), F_i the ffeats at the start of iteration i, f(r) = b*S + s,
// K = kept rows x iterations), without the dense score maps.  With the upstream gradient g, the score gradient is
//
//   c_i[r,p] = g (sigma(s) - 1) / (eps+K) at p = t,   g sigma(s) / (eps+K(P-1)) elsewhere,   0 for a dropped row
//
// and   dF_i[r,:] = sum_p c_i[r,p] G[f(r),p,:]          (pips_scoremap_grad_feats)
//       dG[f,p,:] = sum_i sum_{r in f} c_i[r,p] F_i[r,:]  (pips_scoremap_grad_basis)
//       dlevel_l  = interp_l^T(dG) / sqrt(C)            (pips_scoremap_basis_grad)
//
// The two GEMM kernels share one structure, the recomputation of FlashAttention's backward: a resident 128-row tile X
// (bf16 hi/lo in shared memory) meets 64-row tiles Y streamed through a 4-stage TMA ring (warp 0 produces, two consumer
// warpgroups of 64 rows each).  Per tile, in bf16x3 (hi.hi + lo.hi + hi.lo):
//   S = X Y^T        wgmma, both operands K-major from shared memory (the forward's score GEMM)
//   c(S)             in registers, from the accumulator fragment, split into (hi, lo) bf16 pairs
//   O += c Y         wgmma with c as the register A operand and the SAME shared-memory Y stage as B, read MN-major:
//                    a 64-byte-swizzled K-block of 32 channels is a stack of MN-major SW64 atoms (wgmma_desc_sw64_mn)
//   grad_feats: X = F_i (128 particles of one frame and iteration), Y = G (64 pixels), O = dF_i
//   grad_basis: X = G (128 pixels of one frame),                    Y = F_i (64 particles), O = dG
// Each CTA owns its 128 output rows and sums over its tiles in a fixed order: no atomics, and the result depends on the
// shape only.  The two coefficients g/(eps+K), g/(eps+K(P-1)) are read from device memory (no host round trip).
#include "scoremap_common.cuh"

namespace pips {
namespace {
using namespace smap;

constexpr int L = PIPS_LEVELS;

struct GradArgs {
    const float* feats;                                // grad_feats: F (iters, frames, N, C) fp32
    const __nv_bfloat16* g_hi;                         // grad_basis: G (frames, P, C)
    const __nv_bfloat16* g_lo;
    const int* target;                                 // (frames, N): target pixel, or -1
    const float* coef;                                 // [g/(eps+K), g/(eps+K(P-1))]
    float* out;                                        // dF (iters, frames, N, C) or dG (frames, P, C), fp32
    int frames, N, P, iters;
};

// dloss/ds for a kept row: at the target g (sigma(s) - 1)/(eps+K) = -cpos / (1 + e^s) (no cancellation near sigma = 1),
// elsewhere cneg sigma(s) = cneg / (1 + e^-s)
__device__ __forceinline__ float score_grad(float s, bool at_target, float cpos, float cneg) {
    return at_target ? -cpos / (1.0f + __expf(s)) : cneg / (1.0f + __expf(-s));
}

// BASIS = false: pips_scoremap_grad_feats, grid (particle tiles, frames, iters).
// BASIS = true:  pips_scoremap_grad_basis, grid (pixel tiles, frames).
template <bool BASIS>
__global__ void __launch_bounds__(THREADS, 1)
scoremap_grad_kernel(const __grid_constant__ CUtensorMap y_hi, const __grid_constant__ CUtensorMap y_lo, const GradArgs a) {
    uint8_t* smem = aligned_smem();
    Ring ring = y_ring(smem);

    const int x_base = blockIdx.x * BM;             // first resident row: particle (feats) or pixel (basis)
    const int frame = blockIdx.y;
    const int it = BASIS ? 0 : blockIdx.z;
    const int x_rows = BASIS ? a.P : a.N;
    const int y_per_pass = ((BASIS ? a.N : a.P) + BN - 1) / BN;   // streamed tiles per frame (and iteration)
    const int tiles = BASIS ? a.iters * y_per_pass : y_per_pass;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

    if (threadIdx.x == 0) {
        tma_prefetch_desc(&y_hi);
        tma_prefetch_desc(&y_lo);
        ring.init(2);                                      // one arrival per consumer warpgroup
    }
    __syncthreads();

    if (warp < 4) {
        if (warp == 0 && lane == 0) {
            // ------------------------------------------------------------ TMA producer
            for (int t = 0; t < tiles; ++t) {
                // rows past this frame's pixels (particles) belong to the next frame (iteration), or are zero-filled
                // past the tensor: their coefficients are 0
                int row;
                if constexpr (BASIS) {
                    const int i = t / y_per_pass;
                    row = (i * a.frames + frame) * a.N + (t - i * y_per_pass) * BN;
                } else {
                    row = frame * a.P + t * BN;
                }
                load_y(ring, &y_hi, &y_lo, row);
            }
        }
        return;
    }

    // ---------------------------------------------------------------- consumers
    const int ct = threadIdx.x - 128;                      // 0..255
    const int wg = ct >> 7;
    // the resident tile, K-major, 64-byte swizzled; rows past the frame's particles (pixels) are zero
    if constexpr (BASIS) {
        for (int i = ct; i < BM * (C / 8); i += 256) {     // 16-byte chunks of 8 channels
            const int r = i >> 4, c8 = i & 15;
            const int p = x_base + r;
            uint4 h = make_uint4(0, 0, 0, 0), l = h;
            if (p < a.P) {
                const size_t off = (static_cast<size_t>(frame) * a.P + p) * C;
                h = __ldg(reinterpret_cast<const uint4*>(a.g_hi + off) + c8);
                l = __ldg(reinterpret_cast<const uint4*>(a.g_lo + off) + c8);
            }
            const int k = 8 * c8, kb = k / KB;
            const uint32_t o = sw64(r, (k % KB) * 2);
            *reinterpret_cast<uint4*>(smem + kb * X_KB_BYTES + o) = h;
            *reinterpret_cast<uint4*>(smem + (NKB + kb) * X_KB_BYTES + o) = l;
        }
    } else {
        const float* f = a.feats + (static_cast<size_t>(it) * a.frames + frame) * a.N * C;
        fill_x_f32(smem, ct, x_base, a.N, [&](int n) { return f + static_cast<size_t>(n) * C; });
    }
    fence_proxy_async_smem();                              // the generic-proxy writes become visible to wgmma
    named_bar_sync(1, 256);

    const float cpos = __ldg(a.coef), cneg = __ldg(a.coef + 1);
    // this thread's fragment rows: r0 and r0 + 8 of the warpgroup's 64; columns cq, cq + 1 of every 8
    const int r0 = wg * 64 + (warp & 3) * 16 + (lane >> 2);
    const int cq = 2 * (lane & 3);
    int xt[2];                                             // feats: the row's target pixel; basis: the row's pixel
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        const int x = x_base + r0 + 8 * h;
        if constexpr (BASIS) xt[h] = x;
        else xt[h] = x < a.N ? __ldg(a.target + static_cast<size_t>(frame) * a.N + x) : -1;
    }
    const bool releaser = (ct & 127) == 0;
    const uint32_t x_hi0 = smem_u32(smem) + wg * (X_KB_BYTES / 2);
    const uint32_t x_lo0 = smem_u32(smem + NKB * X_KB_BYTES) + wg * (X_KB_BYTES / 2);
    float sacc[BN / 2];
    float oacc[C / 2];
#pragma unroll
    for (int j = 0; j < C / 2; ++j) oacc[j] = 0.0f;
    auto omma = [&](const uint32_t* c, uint64_t y, uint32_t accumulate) {
        wgmma_n128_rA_tb(oacc, c[0], c[1], c[2], c[3], y, accumulate);
    };
    for (int t = 0; t < tiles; ++t) {
        const uint32_t base = ring.wait();
        score_mma(sacc, x_hi0, x_lo0, base);

        // c from the fragment: column 8j + cq + e of rows r0 (h = 0) and r0 + 8 (h = 1) is sacc[4j + 2h + e]
        int y0, y_lim;                                     // streamed row of column 0; columns >= y_lim are not ours
        if constexpr (BASIS) {
            const int i = t / y_per_pass;
            y0 = (t - i * y_per_pass) * BN;
            y_lim = a.N - y0;
        } else {
            y0 = t * BN;
            y_lim = a.P - y0;
        }
        uint32_t c_hi[BN / 4], c_lo[BN / 4];
#pragma unroll
        for (int j = 0; j < BN / 8; ++j) {
            int yt[2];                                     // basis: the column's target pixel
            if constexpr (BASIS) {
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    const int col = 8 * j + cq + e;
                    yt[e] = col < y_lim ? __ldg(a.target + static_cast<size_t>(frame) * a.N + y0 + col) : -1;
                }
            }
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                float c[2];
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    const int col = 8 * j + cq + e;
                    const float s = sacc[4 * j + 2 * h + e];
                    if constexpr (BASIS) {
                        c[e] = yt[e] >= 0 ? score_grad(s, yt[e] == xt[h], cpos, cneg) : 0.0f;
                    } else {
                        c[e] = (xt[h] >= 0 && col < y_lim) ? score_grad(s, y0 + col == xt[h], cpos, cneg) : 0.0f;
                    }
                }
                const uint32_t hi = cvt_bf16x2(c[0], c[1]);
                const uint32_t lo = cvt_bf16x2(c[0] - __uint_as_float(hi << 16), c[1] - __uint_as_float(hi & 0xffff0000u));
                c_hi[2 * j + h] = hi;
                c_lo[2 * j + h] = lo;
            }
        }

        // O += c Y: K step k covers columns 16k..16k+15 of c = streamed rows 16k..16k+15 (1 KB into each K-block);
        // its A fragment is c[4k .. 4k+3] in the order (r0, lo cols), (r0+8, lo cols), (r0, hi cols), (r0+8, hi cols)
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < BN / MMA_K; ++k) {
            const uint64_t yh = wgmma_desc_sw64_mn(base + k * 1024, Y_KB_BYTES);
            const uint64_t yl = wgmma_desc_sw64_mn(base + NKB * Y_KB_BYTES + k * 1024, Y_KB_BYTES);
            mma_bf16x3(omma, &c_hi[4 * k], &c_lo[4 * k], yh, yl, 1);
        }
        wgmma_commit();
        wgmma_wait<0>();
        wgmma_acc_ready(oacc);
        if (releaser) ring.release(ring.stage);            // both GEMMs have read the stage
        ring.advance();
    }

    // O rows r0, r0 + 8: channel 8j + cq + e is oacc[4j + 2h + e]
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        const int x = x_base + r0 + 8 * h;
        if (x >= x_rows) continue;
        float* o = a.out + ((BASIS ? static_cast<size_t>(frame) : (static_cast<size_t>(it) * a.frames + frame)) * x_rows + x) * C;
#pragma unroll
        for (int j = 0; j < C / 8; ++j)
            *reinterpret_cast<float2*>(o + 8 * j + cq) = make_float2(oacc[4 * j + 2 * h], oacc[4 * j + 2 * h + 1]);
    }
}

// ---------------------------------------------------------------------------------- the adjoint of the basis

struct LevelGrads {
    float* lvl[L];
    int H[L], W[L];
};

// the fine coordinates v in [lo, hi] whose bilinear taps (align_corners=True, the index math of scoremap_basis_kernel)
// can touch coarse coordinate V, at scale s = (coarse - 1) / (fine - 1), with slack for rounding
__device__ __forceinline__ void fine_range(int V, float s, int fine, int& lo, int& hi) {
    if (s > 0.0f) {
        lo = max(0, static_cast<int>(floorf((V - 1) / s)) - 2);
        hi = min(fine - 1, static_cast<int>(ceilf((V + 1) / s)) + 2);
    } else {
        lo = 0;
        hi = fine - 1;
    }
}

// the weight of coarse coordinate V in the interpolation at fine coordinate v (the forward's arithmetic)
__device__ __forceinline__ float tap_weight(int v, int V, float s, int coarse) {
    const float f = s * v;
    const int v0 = static_cast<int>(f);
    const int vp = v0 < coarse - 1 ? 1 : 0;
    const float lf = f - v0;
    return (v0 == V ? 1.0f - lf : 0.0f) + (v0 + vp == V ? lf : 0.0f);
}

// one thread per (frame, coarse pixel, 4 channels) of level blockIdx.y: a gather over the fine pixels whose bilinear
// weights touch it, in a fixed order (rows, then columns), times 1/sqrt(C).  No atomics.
__global__ void __launch_bounds__(256) scoremap_basis_grad_kernel(const float* __restrict__ dG, int frames, int H8, int W8,
                                                                  LevelGrads lg) {
    const float scale = 0.08838834764831845f;            // 1 / sqrt(128)
    const int l = blockIdx.y;
    const int h = lg.H[l], w = lg.W[l];
    const float sy = H8 > 1 ? static_cast<float>(h - 1) / static_cast<float>(H8 - 1) : 0.0f;
    const float sx = W8 > 1 ? static_cast<float>(w - 1) / static_cast<float>(W8 - 1) : 0.0f;
    const size_t total = static_cast<size_t>(frames) * h * w * (C / 4);
    for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < total;
         i += static_cast<size_t>(gridDim.x) * blockDim.x) {
        const int c4 = static_cast<int>(i & 31);
        const size_t pix = i >> 5;
        const int X = static_cast<int>(pix % w);
        const size_t r = pix / w;
        const int Y = static_cast<int>(r % h);
        const size_t frame = r / h;
        int ylo, yhi, xlo, xhi;
        fine_range(Y, sy, H8, ylo, yhi);
        fine_range(X, sx, W8, xlo, xhi);
        const float4* g = reinterpret_cast<const float4*>(dG + frame * H8 * W8 * C) + c4;
        float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
        for (int y = ylo; y <= yhi; ++y) {
            const float wy = tap_weight(y, Y, sy, h);
            if (wy == 0.0f) continue;
            for (int x = xlo; x <= xhi; ++x) {
                const float wx = tap_weight(x, X, sx, w);
                if (wx == 0.0f) continue;
                const float wt = wy * wx;
                const float4 v = __ldg(g + static_cast<size_t>(y * W8 + x) * (C / 4));
                acc.x = fmaf(wt, v.x, acc.x);
                acc.y = fmaf(wt, v.y, acc.y);
                acc.z = fmaf(wt, v.z, acc.z);
                acc.w = fmaf(wt, v.w, acc.w);
            }
        }
        acc.x *= scale; acc.y *= scale; acc.z *= scale; acc.w *= scale;
        reinterpret_cast<float4*>(lg.lvl[l] + pix * C)[c4] = acc;
    }
}

// the shared host side of the two GEMM kernels: tensor maps over the streamed operand (rows x 128 bf16) and the launch
template <bool BASIS>
int launch_grad(const char* name, const void* y_hi, const void* y_lo, long long y_rows, dim3 grid, const GradArgs& a,
                void* stream) {
    CUtensorMap map_hi, map_lo;
    cuuint64_t gdim[2] = {static_cast<cuuint64_t>(C), static_cast<cuuint64_t>(y_rows)};
    cuuint64_t gstride[1] = {static_cast<cuuint64_t>(C) * 2};
    cuuint32_t box[2] = {static_cast<cuuint32_t>(KB), static_cast<cuuint32_t>(BN)};
    cuuint32_t estr[2] = {1, 1};
    if (!encode_tiled_pair(&map_hi, &map_lo, y_hi, y_lo, 2, gdim, gstride, box, estr, CU_TENSOR_MAP_SWIZZLE_64B))
        return fail(BASIS ? "pips_scoremap_grad_basis: tensor map (F) failed" : "pips_scoremap_grad_feats: tensor map (G) failed");
    return launch_kernel<scoremap_grad_kernel<BASIS>>(name, false, grid, THREADS, SMEM_BYTES, static_cast<cudaStream_t>(stream),
                                                      map_hi, map_lo, a);
}

}  // namespace
}  // namespace pips

using namespace pips;

// pips_scoremap_grad_feats (S == 8) and pips_scoremap_grad_feats_window (2 <= S <= PIPS_S_MAX): the kernel indexes frames
// as b*S + s and never reads S itself
static int scoremap_grad_feats_entry(int s_min, int s_max, const void* G_hi, const void* G_lo, const float* ffeats, int iters,
                                     int B, int S, int N, int H8, int W8, const int* target, const float* coef, float* dffeats,
                                     void* stream) {
    if (!G_hi || !G_lo || !ffeats || !target || !coef || !dffeats) return fail("pips_scoremap_grad_feats: null pointer");
    if (iters <= 0 || B <= 0 || S <= 0 || N <= 0 || H8 <= 0 || W8 <= 0) return fail("pips_scoremap_grad_feats: empty problem");
    if (S < s_min || S > s_max)
        return fail(s_min == s_max ? "pips_scoremap_grad_feats: S must be 8 (pips_scoremap_grad_feats_window takes 2..16)"
                                   : "pips_scoremap_grad_feats_window: S must be in 2..16");
    if ((reinterpret_cast<uintptr_t>(G_hi) | reinterpret_cast<uintptr_t>(G_lo) | reinterpret_cast<uintptr_t>(ffeats)
         | reinterpret_cast<uintptr_t>(dffeats)) & 15)
        return fail("pips_scoremap_grad_feats: G_hi, G_lo, ffeats and dffeats must be 16-byte aligned");
    const long long rows = static_cast<long long>(B) * S * H8 * W8;
    if (rows > 0x7fffffffLL || (N + BM - 1) / BM > 65535 || B * S > 65535 || iters > 65535)
        return fail("pips_scoremap_grad_feats: problem too large");
    GradArgs a = {};
    a.feats = ffeats; a.target = target; a.coef = coef; a.out = dffeats;
    a.frames = B * S; a.N = N; a.P = H8 * W8; a.iters = iters;
    return launch_grad<false>("pips_scoremap_grad_feats", G_hi, G_lo, rows, dim3((N + BM - 1) / BM, B * S, iters), a,
                              stream);
}

// pips_scoremap_grad_basis (S == 8) and pips_scoremap_grad_basis_window (2 <= S <= PIPS_S_MAX)
static int scoremap_grad_basis_entry(int s_min, int s_max, const void* G_hi, const void* G_lo, const void* F_hi,
                                     const void* F_lo, int iters, int B, int S, int N, int H8, int W8, const int* target,
                                     const float* coef, float* dG, void* stream) {
    if (!G_hi || !G_lo || !F_hi || !F_lo || !target || !coef || !dG) return fail("pips_scoremap_grad_basis: null pointer");
    if (iters <= 0 || B <= 0 || S <= 0 || N <= 0 || H8 <= 0 || W8 <= 0) return fail("pips_scoremap_grad_basis: empty problem");
    if (S < s_min || S > s_max)
        return fail(s_min == s_max ? "pips_scoremap_grad_basis: S must be 8 (pips_scoremap_grad_basis_window takes 2..16)"
                                   : "pips_scoremap_grad_basis_window: S must be in 2..16");
    if ((reinterpret_cast<uintptr_t>(G_hi) | reinterpret_cast<uintptr_t>(G_lo) | reinterpret_cast<uintptr_t>(F_hi)
         | reinterpret_cast<uintptr_t>(F_lo) | reinterpret_cast<uintptr_t>(dG)) & 15)
        return fail("pips_scoremap_grad_basis: G_hi, G_lo, F_hi, F_lo and dG must be 16-byte aligned");
    const long long rows = static_cast<long long>(iters) * B * S * N;
    const int P = H8 * W8;
    if (rows > 0x7fffffffLL || static_cast<long long>(B) * S * P > 0x7fffffffLL || B * S > 65535)
        return fail("pips_scoremap_grad_basis: problem too large");
    GradArgs a = {};
    a.g_hi = static_cast<const __nv_bfloat16*>(G_hi); a.g_lo = static_cast<const __nv_bfloat16*>(G_lo);
    a.target = target; a.coef = coef; a.out = dG;
    a.frames = B * S; a.N = N; a.P = P; a.iters = iters;
    return launch_grad<true>("pips_scoremap_grad_basis", F_hi, F_lo, rows, dim3((P + BM - 1) / BM, B * S), a, stream);
}

extern "C" int pips_scoremap_grad_feats(const void* G_hi, const void* G_lo, const float* ffeats, int iters, int B, int S,
                                        int N, int H8, int W8, const int* target, const float* coef, float* dffeats,
                                        void* stream) {
    return scoremap_grad_feats_entry(PIPS_S, PIPS_S, G_hi, G_lo, ffeats, iters, B, S, N, H8, W8, target, coef, dffeats, stream);
}

extern "C" int pips_scoremap_grad_feats_window(const void* G_hi, const void* G_lo, const float* ffeats, int iters, int B,
                                               int S, int N, int H8, int W8, const int* target, const float* coef,
                                               float* dffeats, void* stream) {
    return scoremap_grad_feats_entry(2, PIPS_S_MAX, G_hi, G_lo, ffeats, iters, B, S, N, H8, W8, target, coef, dffeats,
                                     stream);
}

extern "C" int pips_scoremap_grad_basis(const void* G_hi, const void* G_lo, const void* F_hi, const void* F_lo, int iters,
                                        int B, int S, int N, int H8, int W8, const int* target, const float* coef, float* dG,
                                        void* stream) {
    return scoremap_grad_basis_entry(PIPS_S, PIPS_S, G_hi, G_lo, F_hi, F_lo, iters, B, S, N, H8, W8, target, coef, dG, stream);
}

extern "C" int pips_scoremap_grad_basis_window(const void* G_hi, const void* G_lo, const void* F_hi, const void* F_lo,
                                               int iters, int B, int S, int N, int H8, int W8, const int* target,
                                               const float* coef, float* dG, void* stream) {
    return scoremap_grad_basis_entry(2, PIPS_S_MAX, G_hi, G_lo, F_hi, F_lo, iters, B, S, N, H8, W8, target, coef, dG,
                                     stream);
}

extern "C" int pips_scoremap_basis_grad(const float* dG, int frames, int H8, int W8, float* const* dlvl_f32, void* stream) {
    if (!dG || !dlvl_f32) return fail("pips_scoremap_basis_grad: null pointer");
    if (frames <= 0) return fail("pips_scoremap_basis_grad: empty problem");
    if ((H8 >> (PIPS_LEVELS - 1)) < 1 || (W8 >> (PIPS_LEVELS - 1)) < 1)
        return fail("pips_scoremap_basis_grad: feature map too small for 4 levels");
    if (reinterpret_cast<uintptr_t>(dG) & 15) return fail("pips_scoremap_basis_grad: dG and the levels must be 16-byte aligned");
    LevelGrads lg;
    int h = H8, w = W8;
    for (int l = 0; l < PIPS_LEVELS; ++l) {
        if (!dlvl_f32[l]) return fail("pips_scoremap_basis_grad: null pyramid level");
        if (reinterpret_cast<uintptr_t>(dlvl_f32[l]) & 15)
            return fail("pips_scoremap_basis_grad: dG and the levels must be 16-byte aligned");
        lg.lvl[l] = dlvl_f32[l];
        lg.H[l] = h;
        lg.W[l] = w;
        h /= 2;
        w /= 2;
    }
    const size_t total = static_cast<size_t>(frames) * H8 * W8 * (C / 4);     // of level 0, the largest
    const size_t blocks = (total + 255) / 256;
    const int cap = sm_count() * 8;
    scoremap_basis_grad_kernel<<<dim3(static_cast<unsigned>(blocks < static_cast<size_t>(cap) ? blocks : cap), PIPS_LEVELS), 256,
                                 0, static_cast<cudaStream_t>(stream)>>>(dG, frames, H8, W8, lg);
    cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? 0 : fail_cuda("pips_scoremap_basis_grad", e);
}
