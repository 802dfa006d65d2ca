// Score-map loss of nets/pips.py:58-90,:603 (score_map_loss) without the dense score maps.
//
// Bilinear upsampling is linear, so the per-iteration score map of nets/pips.py:504-511 factors through a basis that
// depends on the pyramid only:
//
//   fcp[b,s,n,p] = sum_l interp_l( <ffeats[b,s,n], fmap_l[b,s]> / sqrt(C) )(p) = <ffeats[b,s,n], G[b,s,p]>,
//   G[b,s,p,:]   = sum_l interp_l(fmap_l[b,s])(p,:) / sqrt(C)
//
// interp_l is F.interpolate(bilinear, align_corners=True) from level l to (H8,W8), the index math of
// heat_upsample_kernel (heatmap.cu).  pips_scoremap_basis builds G once per forward as a bf16 (hi, lo) pair,
// (frames, H8*W8, 128), K-major.  Every iteration's score maps of frame (b,s) are then one GEMM (M = particles,
// N = pixels, K = 128), and pips_scoremap_loss reduces them in the epilogue of that GEMM to the two terms of the
// balanced CE (nets/pips.py:14-37) of each row (b,s,n) with target pixel t:
//
//   pos = softplus(-fcp[t])           neg = sum_{p != t} softplus(fcp[p])
//
// so no score ever reaches global memory.  Structure of the loss kernel (one CTA per frame x 128 particles x pixel
// split):
//   warp 0       TMA producer: 64-pixel tiles of G (hi and lo, all of K) -> 4-stage shared-memory ring
//   warps 4..7   consumer warpgroup 0: particles 0..63 of the tile  } wgmma m64n64k16, bf16x3 (hi.hi + lo.hi + hi.lo),
//   warps 8..11  consumer warpgroup 1: particles 64..127            } then softplus + row sums from the fragment
// The particle tile (A) is read from the fp32, S-strided ffeats once, split into (hi, lo) in registers and stays
// resident in shared memory while the pixel tiles stream past.  While one warpgroup is in its epilogue (the MUFU /
// FMA-bound part), the other one's MMAs keep the tensor cores busy.
//
// Determinism: a row's partial sum depends on its own data, its split and a fixed order (tiles, then fragment columns,
// then the quad of lanes that share the row); the grid depends on the shape only -- not on particle chunking, on graph
// or eager launch, or on the SM count.
#include "scoremap_common.cuh"

namespace pips {
namespace {
using namespace smap;                                  // X: the particle tile, Y: pixel tiles of G

constexpr int L = PIPS_LEVELS;
constexpr int SPLIT_PIX = 512;                         // pixels per split (8 ring stages)
static_assert(SPLIT_PIX % BN == 0, "a split is whole pixel tiles");

struct LossArgs {
    const float* ffeats;                               // ((b*N + n), s, c)
    const int* target;                                 // (B,S,N): y*W8 + x, or -1
    float* neg_part;                                   // (B*S*N, n_split)
    float* pos_part;                                   // (B*S*N)
    int S, N, P, n_split;
};

// softplus(v) = log(1 + e^v), overflow-safe: max(v, 0) + log1p(e^-|v|).  log1pf keeps the small terms (e^-|v| << 1)
// accurate to a few ulp, which the 1e-4 relative tolerance on a row's neg sum needs.
__device__ __forceinline__ float softplus(float v) {
    return fmaxf(v, 0.0f) + log1pf(__expf(-fabsf(v)));
}

__global__ void __launch_bounds__(THREADS, 1)
scoremap_loss_kernel(const __grid_constant__ CUtensorMap g_hi, const __grid_constant__ CUtensorMap g_lo, const LossArgs a) {
    uint8_t* smem = aligned_smem();
    Ring ring = y_ring(smem);

    const int split = blockIdx.x;
    const int n_base = blockIdx.y * BM;
    const int frame = blockIdx.z;                          // b * S + s
    const int b = frame / a.S, s = frame - b * a.S;
    const int p_begin = split * SPLIT_PIX;
    const int p_end = min(a.P, p_begin + SPLIT_PIX);
    const int tiles = (p_end - p_begin + BN - 1) / BN;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

    if (threadIdx.x == 0) {
        tma_prefetch_desc(&g_hi);
        tma_prefetch_desc(&g_lo);
        ring.init(2);                                      // one arrival per consumer warpgroup
    }
    __syncthreads();

    if (warp < 4) {
        if (warp == 0 && lane == 0) {
            // ------------------------------------------------------------ TMA producer (G does not depend on ffeats)
            // rows past this frame's pixels belong to the next frame (or are zero-filled past the tensor): the epilogue
            // ignores their columns
            for (int t = 0; t < tiles; ++t) load_y(ring, &g_hi, &g_lo, frame * a.P + p_begin + t * BN);
        }
        return;
    }

    // ---------------------------------------------------------------- consumers
    const int ct = threadIdx.x - 128;                      // 0..255
    const int wg = ct >> 7;
    // the particle tile: fp32 ffeats rows (frame s of track (b, n)); rows past N are zero
    fill_x_f32(smem, ct, n_base, a.N, [&](int n) { return a.ffeats + (static_cast<size_t>(b * a.N + n) * a.S + s) * C; });
    fence_proxy_async_smem();                              // the generic-proxy writes become visible to wgmma
    named_bar_sync(1, 256);

    // this thread's fragment rows (ptx.cuh): r0 and r0 + 8 of the warpgroup's 64; columns cq, cq + 1 of every 8
    const int r0 = wg * 64 + (warp & 3) * 16 + (lane >> 2);
    const int cq = 2 * (lane & 3);
    int tgt[2];
    size_t grow[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        const int n = n_base + r0 + 8 * h;
        grow[h] = static_cast<size_t>(frame) * a.N + n;
        tgt[h] = n < a.N ? __ldg(a.target + grow[h]) : -2;    // -2: no such particle (no output)
    }
    float neg[2] = {0.0f, 0.0f};
    const bool releaser = (ct & 127) == 0;
    const uint32_t x_hi0 = smem_u32(smem) + wg * (X_KB_BYTES / 2);
    const uint32_t x_lo0 = smem_u32(smem + NKB * X_KB_BYTES) + wg * (X_KB_BYTES / 2);
    float acc[BN / 2];
    for (int t = 0; t < tiles; ++t) {
        score_mma(acc, x_hi0, x_lo0, ring.wait());
        if (releaser) ring.release(ring.stage);            // the slot is free while this warpgroup runs its epilogue
        ring.advance();

        const int p0 = p_begin + t * BN;
        const int lim = p_end - p0;                        // columns >= lim are outside this split (or frame)
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            if (tgt[h] < 0) continue;
            const int tl = tgt[h] - p0;                    // the target's column in this tile (any value if elsewhere)
#pragma unroll
            for (int j = 0; j < BN / 8; ++j) {
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    const int col = 8 * j + cq + e;
                    const float v = acc[4 * j + 2 * h + e];
                    if (col >= lim) continue;
                    if (col == tl) a.pos_part[grow[h]] = softplus(-v);
                    else neg[h] += softplus(v);
                }
            }
        }
    }
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        float v = neg[h];
        v += __shfl_xor_sync(0xffffffffu, v, 1);           // commutative adds: all four lanes hold the same bits
        v += __shfl_xor_sync(0xffffffffu, v, 2);
        if ((lane & 3) == 0 && tgt[h] != -2) {
            a.neg_part[grow[h] * a.n_split + split] = v;   // 0 for a row without a target
            if (tgt[h] == -1 && split == 0) a.pos_part[grow[h]] = 0.0f;
        }
    }
}

// ---------------------------------------------------------------------------------- the basis G

struct BasisLevels {
    const float* lvl[L];
    int H[L], W[L];
};

// one thread per (frame, pixel, 4 channels): the 4 bilinear taps of every level (ATen's upsample_bilinear2d with
// align_corners=True, as heat_upsample_kernel), summed over the levels in the reference's order, times 1/sqrt(C)
__global__ void __launch_bounds__(256) scoremap_basis_kernel(BasisLevels lv, int H8, int W8, size_t total,
                                                             __nv_bfloat16* __restrict__ g_hi, __nv_bfloat16* __restrict__ g_lo) {
    const float scale = 0.08838834764831845f;            // 1 / sqrt(128), nets/pips.py:396
    for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < total;
         i += static_cast<size_t>(gridDim.x) * blockDim.x) {
        const int c4 = static_cast<int>(i & 31);
        const size_t pix = i >> 5;
        const int x = static_cast<int>(pix % W8);
        const size_t r = pix / W8;
        const int y = static_cast<int>(r % H8);
        const size_t frame = r / H8;
        float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
        for (int l = 0; l < L; ++l) {
            const int h = lv.H[l], w = lv.W[l];
            const float sy = H8 > 1 ? static_cast<float>(h - 1) / static_cast<float>(H8 - 1) : 0.0f;
            const float sx = W8 > 1 ? static_cast<float>(w - 1) / static_cast<float>(W8 - 1) : 0.0f;
            const float fy = sy * y, fx = sx * x;
            const int y0 = static_cast<int>(fy), x0 = static_cast<int>(fx);
            const int yp = y0 < h - 1 ? 1 : 0, xp = x0 < w - 1 ? 1 : 0;
            const float ly = fy - y0, lx = fx - x0;
            const float hy = 1.0f - ly, hx = 1.0f - lx;
            const float4* m = reinterpret_cast<const float4*>(lv.lvl[l] + frame * h * w * C) + c4;
            const float4 v00 = __ldg(m + (y0 * w + x0) * (C / 4)), v01 = __ldg(m + (y0 * w + x0 + xp) * (C / 4));
            const float4 v10 = __ldg(m + ((y0 + yp) * w + x0) * (C / 4)), v11 = __ldg(m + ((y0 + yp) * w + x0 + xp) * (C / 4));
            acc.x += hy * (hx * v00.x + lx * v01.x) + ly * (hx * v10.x + lx * v11.x);
            acc.y += hy * (hx * v00.y + lx * v01.y) + ly * (hx * v10.y + lx * v11.y);
            acc.z += hy * (hx * v00.z + lx * v01.z) + ly * (hx * v10.z + lx * v11.z);
            acc.w += hy * (hx * v00.w + lx * v01.w) + ly * (hx * v10.w + lx * v11.w);
        }
        acc.x *= scale; acc.y *= scale; acc.z *= scale; acc.w *= scale;
        const uint32_t h01 = cvt_bf16x2(acc.x, acc.y), h23 = cvt_bf16x2(acc.z, acc.w);
        const uint32_t l01 = cvt_bf16x2(acc.x - __uint_as_float(h01 << 16), acc.y - __uint_as_float(h01 & 0xffff0000u));
        const uint32_t l23 = cvt_bf16x2(acc.z - __uint_as_float(h23 << 16), acc.w - __uint_as_float(h23 & 0xffff0000u));
        reinterpret_cast<uint2*>(g_hi + pix * C)[c4] = make_uint2(h01, h23);
        reinterpret_cast<uint2*>(g_lo + pix * C)[c4] = make_uint2(l01, l23);
    }
}

}  // namespace
}  // namespace pips

using namespace pips;

extern "C" int pips_scoremap_splits(int H8, int W8) {
    if (H8 <= 0 || W8 <= 0) return 0;
    return (H8 * W8 + SPLIT_PIX - 1) / SPLIT_PIX;
}

extern "C" int pips_scoremap_basis(const float* const* lvl_f32, int frames, int H8, int W8, void* G_hi, void* G_lo, void* stream) {
    if (!lvl_f32 || !G_hi || !G_lo) return fail("pips_scoremap_basis: null pointer");
    if (frames <= 0) return fail("pips_scoremap_basis: empty problem");
    if ((H8 >> (PIPS_LEVELS - 1)) < 1 || (W8 >> (PIPS_LEVELS - 1)) < 1) return fail("pips_scoremap_basis: feature map too small for 4 levels");
    BasisLevels lv;
    int h = H8, w = W8;
    for (int l = 0; l < PIPS_LEVELS; ++l) {
        if (!lvl_f32[l]) return fail("pips_scoremap_basis: null pyramid level");
        lv.lvl[l] = lvl_f32[l];
        lv.H[l] = h;
        lv.W[l] = w;
        h /= 2;
        w /= 2;
    }
    const size_t total = static_cast<size_t>(frames) * H8 * W8 * (C / 4);
    const size_t blocks = (total + 255) / 256;
    const int cap = sm_count() * 16;
    scoremap_basis_kernel<<<static_cast<unsigned>(blocks < static_cast<size_t>(cap) ? blocks : cap), 256, 0,
                            static_cast<cudaStream_t>(stream)>>>(lv, H8, W8, total, static_cast<__nv_bfloat16*>(G_hi),
                                                                 static_cast<__nv_bfloat16*>(G_lo));
    cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? 0 : fail_cuda("pips_scoremap_basis", e);
}

// pips_scoremap_loss (S == 8) and pips_scoremap_loss_window (2 <= S <= PIPS_S_MAX): the kernel decodes frame = b*S + s
static int scoremap_loss_entry(int s_min, int s_max, const void* G_hi, const void* G_lo, const float* ffeats, int B, int S, int N,
                               int H8, int W8, const int* target, float* neg_part, float* pos_part, void* stream) {
    if (!G_hi || !G_lo || !ffeats || !target || !neg_part || !pos_part) return fail("pips_scoremap_loss: null pointer");
    if (B <= 0 || S <= 0 || N <= 0 || H8 <= 0 || W8 <= 0) return fail("pips_scoremap_loss: empty problem");
    if (S < s_min || S > s_max)
        return fail(s_min == s_max ? "pips_scoremap_loss: S must be 8 (pips_scoremap_loss_window takes 2..16)"
                                   : "pips_scoremap_loss_window: S must be in 2..16");
    if ((reinterpret_cast<uintptr_t>(G_hi) | reinterpret_cast<uintptr_t>(G_lo) | reinterpret_cast<uintptr_t>(ffeats)) & 15)
        return fail("pips_scoremap_loss: G_hi, G_lo and ffeats must be 16-byte aligned");
    const long long rows = static_cast<long long>(B) * S * H8 * W8;
    if (rows > 0x7fffffffLL || (N + BM - 1) / BM > 65535 || B * S > 65535)
        return fail("pips_scoremap_loss: problem too large");
    CUtensorMap map_hi, map_lo;
    {
        cuuint64_t gdim[2] = {static_cast<cuuint64_t>(C), static_cast<cuuint64_t>(rows)};
        cuuint64_t gstride[1] = {static_cast<cuuint64_t>(C) * 2};
        cuuint32_t box[2] = {static_cast<cuuint32_t>(KB), static_cast<cuuint32_t>(BN)};
        cuuint32_t estr[2] = {1, 1};
        if (!encode_tiled_pair(&map_hi, &map_lo, G_hi, G_lo, 2, gdim, gstride, box, estr, CU_TENSOR_MAP_SWIZZLE_64B))
            return fail("pips_scoremap_loss: tensor map (G) failed");
    }
    LossArgs a;
    a.ffeats = ffeats; a.target = target; a.neg_part = neg_part; a.pos_part = pos_part;
    a.S = S; a.N = N; a.P = H8 * W8; a.n_split = pips_scoremap_splits(H8, W8);
    // a plain launch: the next iteration's PDL-launched kernels cannot start before this one has read ffeats
    return launch_kernel<scoremap_loss_kernel>("pips_scoremap_loss", false, dim3(a.n_split, (N + BM - 1) / BM, B * S), THREADS,
                                               SMEM_BYTES, static_cast<cudaStream_t>(stream), map_hi, map_lo, a);
}

extern "C" int pips_scoremap_loss(const void* G_hi, const void* G_lo, const float* ffeats, int B, int S, int N, int H8, int W8,
                                  const int* target, float* neg_part, float* pos_part, void* stream) {
    return scoremap_loss_entry(PIPS_S, PIPS_S, G_hi, G_lo, ffeats, B, S, N, H8, W8, target, neg_part, pos_part, stream);
}

extern "C" int pips_scoremap_loss_window(const void* G_hi, const void* G_lo, const float* ffeats, int B, int S, int N, int H8,
                                         int W8, const int* target, float* neg_part, float* pos_part, void* stream) {
    return scoremap_loss_entry(2, PIPS_S_MAX, G_hi, G_lo, ffeats, B, S, N, H8, W8, target, neg_part, pos_part, stream);
}
