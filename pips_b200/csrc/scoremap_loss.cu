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
#include "gemm_common.cuh"

namespace pips {
namespace {

constexpr int C = PIPS_C;                              // 128 = K of the score GEMM
constexpr int L = PIPS_LEVELS;
constexpr int SL_BM = 128;                             // particles per CTA: two consumer warpgroups of 64
constexpr int SL_BN = 64;                              // pixels per ring stage
constexpr int SL_KB = 32;                              // K-block: 32 bf16 = one 64-byte swizzle row
constexpr int SL_NKB = C / SL_KB;                      // 4
constexpr int SPLIT_PIX = 512;                         // pixels per split (8 ring stages)
constexpr int SL_STAGES = 4;
constexpr int SL_THREADS = 384;                        // producer warpgroup + 2 consumer warpgroups
constexpr uint32_t A_KB_BYTES = SL_BM * SL_KB * 2;     // 8 KB: one K-block of the particle tile (hi or lo)
constexpr uint32_t A_BYTES = 2 * SL_NKB * A_KB_BYTES;  // 64 KB: hi and lo, all of K
constexpr uint32_t G_KB_BYTES = SL_BN * SL_KB * 2;     // 4 KB
constexpr uint32_t STAGE_BYTES = 2 * SL_NKB * G_KB_BYTES;   // 32 KB
constexpr uint32_t SL_SMEM_BYTES = 1024 /*align*/ + A_BYTES + SL_STAGES * STAGE_BYTES + 256 /*barriers*/;
static_assert(SL_SMEM_BYTES <= 227u * 1024u, "particle tile + ring must fit in 227 KB");
static_assert(SPLIT_PIX % SL_BN == 0, "a split is whole pixel tiles");

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

// byte `byte` of row `row` in a K-block of 64-byte rows, swizzled the way TMA writes CU_TENSOR_MAP_SWIZZLE_64B
// (the 16-byte unit is XORed with (row / 2) % 4): the layout wgmma_desc_sw64 describes
__device__ __forceinline__ uint32_t sw64(int row, int byte) {
    const uint32_t o = static_cast<uint32_t>(row * 64 + byte);
    return o ^ (((o >> 7) & 3u) << 4);
}

__global__ void __launch_bounds__(SL_THREADS, 1)
scoremap_loss_kernel(const __grid_constant__ CUtensorMap g_hi, const __grid_constant__ CUtensorMap g_lo, const LossArgs a) {
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~static_cast<uintptr_t>(1023));
    uint8_t* ring = smem + A_BYTES;
    uint64_t* bars = reinterpret_cast<uint64_t*>(ring + SL_STAGES * STAGE_BYTES);
    const uint32_t full0 = smem_u32(bars);                 // full[SL_STAGES], empty[SL_STAGES]
    const uint32_t empty0 = full0 + 8 * SL_STAGES;

    const int split = blockIdx.x;
    const int n_base = blockIdx.y * SL_BM;
    const int frame = blockIdx.z;                          // b * S + s
    const int b = frame / a.S, s = frame - b * a.S;
    const int p_begin = split * SPLIT_PIX;
    const int p_end = min(a.P, p_begin + SPLIT_PIX);
    const int tiles = (p_end - p_begin + SL_BN - 1) / SL_BN;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

    if (threadIdx.x == 0) {
        tma_prefetch_desc(&g_hi);
        tma_prefetch_desc(&g_lo);
        for (int st = 0; st < SL_STAGES; ++st) {
            mbar_init(full0 + 8 * st, 1);
            mbar_init(empty0 + 8 * st, 2);             // one arrival per consumer warpgroup
        }
        fence_barrier_init();
    }
    __syncthreads();

    if (warp < 4) {
        if (warp == 0 && lane == 0) {
            // ------------------------------------------------------------ TMA producer (G does not depend on ffeats)
            uint32_t stage = 0, phase = 0;
            for (int t = 0; t < tiles; ++t) {
                mbar_wait(empty0 + 8 * stage, phase ^ 1);
                const uint32_t fb = full0 + 8 * stage;
                mbar_arrive_expect_tx(fb, STAGE_BYTES);
                const uint32_t base = smem_u32(ring + stage * STAGE_BYTES);
                // rows past this frame's pixels belong to the next frame (or are zero-filled past the tensor): the
                // epilogue ignores their columns
                const int row = frame * a.P + p_begin + t * SL_BN;
#pragma unroll
                for (int kb = 0; kb < SL_NKB; ++kb) {
                    tma_load_2d(base + kb * G_KB_BYTES, &g_hi, fb, kb * SL_KB, row);
                    tma_load_2d(base + (SL_NKB + kb) * G_KB_BYTES, &g_lo, fb, kb * SL_KB, row);
                }
                if (++stage == SL_STAGES) { stage = 0; phase ^= 1; }
            }
        }
        return;
    }

    // ---------------------------------------------------------------- consumers
    const int ct = threadIdx.x - 128;                      // 0..255
    const int wg = ct >> 7;
    // the particle tile: fp32 ffeats rows (frame s of track (b, n)) -> (hi, lo) bf16, K-major, 64-byte swizzled;
    // rows past N are zero
    for (int i = ct; i < SL_BM * (C / 4); i += 256) {
        const int r = i >> 5, c4 = i & 31;
        const int n = n_base + r;
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        if (n < a.N) v = __ldg(reinterpret_cast<const float4*>(a.ffeats + (static_cast<size_t>(b * a.N + n) * a.S + s) * C) + c4);
        const uint32_t h01 = cvt_bf16x2(v.x, v.y), h23 = cvt_bf16x2(v.z, v.w);
        const uint32_t l01 = cvt_bf16x2(v.x - __uint_as_float(h01 << 16), v.y - __uint_as_float(h01 & 0xffff0000u));
        const uint32_t l23 = cvt_bf16x2(v.z - __uint_as_float(h23 << 16), v.w - __uint_as_float(h23 & 0xffff0000u));
        const int k = 4 * c4, kb = k / SL_KB;
        const uint32_t off = sw64(r, (k % SL_KB) * 2);
        const uint32_t hi = smem_u32(smem + kb * A_KB_BYTES) + off;
        const uint32_t lo = smem_u32(smem + (SL_NKB + kb) * A_KB_BYTES) + off;
        asm volatile("st.shared.v2.b32 [%0], {%1, %2};" ::"r"(hi), "r"(h01), "r"(h23) : "memory");
        asm volatile("st.shared.v2.b32 [%0], {%1, %2};" ::"r"(lo), "r"(l01), "r"(l23) : "memory");
    }
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
    const uint32_t a_hi0 = smem_u32(smem) + wg * (A_KB_BYTES / 2);
    const uint32_t a_lo0 = smem_u32(smem + SL_NKB * A_KB_BYTES) + wg * (A_KB_BYTES / 2);
    float acc[SL_BN / 2];
    uint32_t stage = 0, phase = 0;
    for (int t = 0; t < tiles; ++t) {
        mbar_wait(full0 + 8 * stage, phase);
        const uint32_t base = smem_u32(ring + stage * STAGE_BYTES);
        wgmma_fence();
#pragma unroll
        for (int kb = 0; kb < SL_NKB; ++kb) {
            const uint64_t ah = wgmma_desc_sw64(a_hi0 + kb * A_KB_BYTES);
            const uint64_t al = wgmma_desc_sw64(a_lo0 + kb * A_KB_BYTES);
            const uint64_t gh = wgmma_desc_sw64(base + kb * G_KB_BYTES);
            const uint64_t gl = wgmma_desc_sw64(base + (SL_NKB + kb) * G_KB_BYTES);
#pragma unroll
            for (int k = 0; k < SL_KB / MMA_K; ++k) {
                const uint64_t adv = static_cast<uint64_t>((k * MMA_K * 2) >> 4);   // 32 B per K=16 step
                wgmma_n64(acc, ah + adv, gh + adv, (kb | k) != 0);
                wgmma_n64(acc, al + adv, gh + adv, 1);
                wgmma_n64(acc, ah + adv, gl + adv, 1);
            }
        }
        wgmma_commit();
        wgmma_wait<0>();
        wgmma_acc_ready(acc);
        if (releaser) mbar_arrive(empty0 + 8 * stage);     // the slot is free while this warpgroup runs its epilogue
        if (++stage == SL_STAGES) { stage = 0; phase ^= 1; }

        const int p0 = p_begin + t * SL_BN;
        const int lim = p_end - p0;                        // columns >= lim are outside this split (or frame)
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            if (tgt[h] < 0) continue;
            const int tl = tgt[h] - p0;                    // the target's column in this tile (any value if elsewhere)
#pragma unroll
            for (int j = 0; j < SL_BN / 8; ++j) {
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

extern "C" int pips_scoremap_loss(const void* G_hi, const void* G_lo, const float* ffeats, int B, int S, int N, int H8, int W8,
                                  const int* target, float* neg_part, float* pos_part, void* stream) {
    if (!G_hi || !G_lo || !ffeats || !target || !neg_part || !pos_part) return fail("pips_scoremap_loss: null pointer");
    if (B <= 0 || S <= 0 || N <= 0 || H8 <= 0 || W8 <= 0) return fail("pips_scoremap_loss: empty problem");
    if (S != PIPS_S) return fail("pips_scoremap_loss: S must be 8");
    if ((reinterpret_cast<uintptr_t>(G_hi) | reinterpret_cast<uintptr_t>(G_lo) | reinterpret_cast<uintptr_t>(ffeats)) & 15)
        return fail("pips_scoremap_loss: G_hi, G_lo and ffeats must be 16-byte aligned");
    const long long rows = static_cast<long long>(B) * S * H8 * W8;
    if (rows > 0x7fffffffLL || (N + SL_BM - 1) / SL_BM > 65535 || B * S > 65535)
        return fail("pips_scoremap_loss: problem too large");
    CUtensorMap maps[2];
    const void* src[2] = {G_hi, G_lo};
    for (int i = 0; i < 2; ++i) {
        cuuint64_t gdim[2] = {static_cast<cuuint64_t>(C), static_cast<cuuint64_t>(rows)};
        cuuint64_t gstride[1] = {static_cast<cuuint64_t>(C) * 2};
        cuuint32_t box[2] = {static_cast<cuuint32_t>(SL_KB), static_cast<cuuint32_t>(SL_BN)};
        cuuint32_t estr[2] = {1, 1};
        if (!encode_tiled(&maps[i], CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(src[i]), gdim, gstride, box, estr,
                          CU_TENSOR_MAP_SWIZZLE_64B))
            return fail("pips_scoremap_loss: tensor map (G) failed");
    }
    static bool attr[kMaxDevices] = {};
    {
        cudaError_t e = ensure_dyn_smem(scoremap_loss_kernel, attr, SL_SMEM_BYTES);
        if (e != cudaSuccess) return fail_cuda("pips_scoremap_loss: smem attribute", e);
    }
    LossArgs a;
    a.ffeats = ffeats; a.target = target; a.neg_part = neg_part; a.pos_part = pos_part;
    a.S = S; a.N = N; a.P = H8 * W8; a.n_split = pips_scoremap_splits(H8, W8);
    // a plain launch: the next iteration's PDL-launched kernels cannot start before this one has read ffeats
    dim3 grid(a.n_split, (N + SL_BM - 1) / SL_BM, B * S);
    scoremap_loss_kernel<<<grid, SL_THREADS, SL_SMEM_BYTES, static_cast<cudaStream_t>(stream)>>>(maps[0], maps[1], a);
    cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? 0 : fail_cuda("pips_scoremap_loss", e);
}
