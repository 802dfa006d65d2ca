// Backward of the local correlation (corr_gather.cu's columns 128:324) with respect to the ffeats and the 4 pyramid
// levels; the coordinates are detached at the top of every iteration (nets/pips.py:500), so they get no gradient.
//
// Per unit u = (b, s, n) (mixer row (b*N + n)*8 + s) and level l, the forward blends the dot products of the unit's 8x8
// footprint (origin o = floor(c) - 3, c the clamped level-l position, fractional part (fx, fy)) into 49 taps:
//   corr[l*49 + i*7 + j] = sum_{dy,dx in {0,1}} w_{dy,dx} <ffeat_u, level_l[frame, o_y + j + dy, o_x + i + dx]> / sqrt(128)
// Its adjoint is one 8x8 matrix of weights per unit and level,
//   A[j][i] = (1/sqrt(128)) sum_{dy,dx} w_{dy,dx} dcorr[l*49 + (i-dx)*7 + (j-dy)]     (terms with 0 <= i-dx, j-dy < 7)
// and the two gradients are
//   dffeat_u          = sum_l sum_{j,i} A[j][i] level_l[frame, o_y + j, o_x + i]       (pixels outside the map are 0)
//   dlevel_l[f, y, x] = sum_{u in frame f whose footprint holds (y, x)} A_u[y - o_y][x - o_x] ffeat_u
//
// corr_grad_feats_kernel: one warp per unit on corr_gather's data path (the same tensor maps and boxes, a per-warp TMA
// ring); each lane owns 4 channels.  corr_grad_levels_kernel: owner computes -- one CTA per (frame, level, 8x8 tile)
// walks the frame's units in ascending n, keeps those whose footprint overlaps the tile and accumulates A * ffeat into
// its 64 px x 128 ch.  Every output element is written once, summed in a fixed order: no atomics, and the bits do not
// depend on the launch or the SM count.
#include <cstdio>

#include "corr_common.cuh"
#include "ptx.cuh"

namespace pips {

constexpr float kRsqrtC = 0.08838834764831845f;     // 1 / sqrt(128): the forward divides every dot product by sqrt(128)

// A[j][i] of one level from the unit's 196 dcorr values, in a fixed term order
__device__ __forceinline__ float adjoint_weight(const float* dc, TapWeights w, int j, int i) {
    float s = 0.f;
    if (i < 7 && j < 7) s = w.w00 * dc[i * 7 + j];
    if (i > 0 && j < 7) s = fmaf(w.w01, dc[(i - 1) * 7 + j], s);
    if (i < 7 && j > 0) s = fmaf(w.w10, dc[i * 7 + j - 1], s);
    if (i > 0 && j > 0) s = fmaf(w.w11, dc[(i - 1) * 7 + j - 1], s);
    return s * kRsqrtC;
}

// ------------------------------------------------------------------------------------------------ dffeat
constexpr int CF_WARPS = 8;
constexpr int CF_STAGES = 3;
constexpr uint32_t CF_BOX_BYTES = CG_ROWS_PER_BOX * 8 * 128 * 4;                  // 8 KB
constexpr uint32_t CF_AUX_BYTES = 64 * 4 + 64;                                    // per warp: A, 3 mbarriers
constexpr uint32_t CF_SMEM_BYTES = CF_WARPS * (CF_STAGES * CF_BOX_BYTES + CF_AUX_BYTES) + 128;

struct CfArgs {
    CgArgs a;                 // B, N, H, W, coords (frame_base null)
    const float* dcorr;       // (B*N*8, ld) fp32, columns [0, 196) used
    int ld;
    float* dffeat;            // (B*N*8, 128)
};

// one CTA per SM (its shared memory fills the SM): the register budget is the whole file's, no spills
__global__ void __launch_bounds__(CF_WARPS * 32, 1)
corr_grad_feats_kernel(const __grid_constant__ CgMaps maps, const CfArgs g) {
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 127) & ~static_cast<uintptr_t>(127));
    const CgArgs& a = g.a;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const uint8_t* stage_buf = smem + static_cast<size_t>(warp) * CF_STAGES * CF_BOX_BYTES;
    float* A = reinterpret_cast<float*>(smem + CF_WARPS * CF_STAGES * CF_BOX_BYTES + warp * CF_AUX_BYTES);
    const uint32_t bar0 = smem_u32(A + 64);
    const uint32_t stage0 = smem_u32(stage_buf);

    const int total = a.B * 8 * a.N;
    const int nwarps = static_cast<int>(gridDim.x) * CF_WARPS;
    int u = static_cast<int>(blockIdx.x) * CF_WARPS + warp;
    if (u >= total) return;                         // whole warp exits together
    if (lane == 0) {
        for (int s = 0; s < CF_STAGES; ++s) mbar_init(bar0 + 8 * s, 1);
        fence_barrier_init();
    }
    __syncwarp();

    // box j of a unit: level = j >> 2, rows 2 (j & 3), 2 (j & 3) + 1 of the level's 8x8 footprint
    auto issue = [&](const UnitInfo& ui, int level, int part, int slot) {
        const int x0 = __shfl_sync(0xffffffffu, ui.ox, level);
        const int y0 = __shfl_sync(0xffffffffu, ui.oy, level) + part * CG_ROWS_PER_BOX;
        if (lane == 0) {
            const uint32_t bar = bar0 + 8 * slot;
            mbar_arrive_expect_tx(bar, CF_BOX_BYTES);
            tma_load_4d(stage0 + slot * CF_BOX_BYTES, &maps.m[level], bar, 0, x0, y0, ui.frame);
        }
    };

    UnitInfo cur = load_unit(a, u, total);
    UnitInfo nxt = load_unit(a, u + nwarps, total);
    issue(cur, 0, 0, 0);
    issue(cur, 0, 1, 1);
    int slot = 0;
    uint32_t parity = 0;

    for (; u < total; u += nwarps) {
        const UnitInfo nxt2 = load_unit(a, u + 2 * nwarps, total);
        const float* dc = g.dcorr + static_cast<size_t>(u) * g.ld;
        float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll 1
        for (int level = 0; level < PIPS_LEVELS; ++level) {
            {
                const TapWeights w = tap_weights(cur.cx, cur.cy, level, a.W[level], a.H[level]);
                for (int p = lane; p < 64; p += 32) A[p] = adjoint_weight(dc + level * 49, w, p >> 3, p & 7);
                __syncwarp();
            }
#pragma unroll
            for (int part = 0; part < 4; ++part) {
                // keep the ring full: the box two ahead (same level, next level, or the next unit's first two)
                {
                    int slot2 = slot + 2;
                    if (slot2 >= CF_STAGES) slot2 -= CF_STAGES;
                    if (part < 2) issue(cur, level, part + 2, slot2);
                    else if (level < PIPS_LEVELS - 1) issue(cur, level + 1, part - 2, slot2);
                    else if (nxt.valid) issue(nxt, 0, part - 2, slot2);
                }
                mbar_wait(bar0 + 8 * slot, parity);
                // box pixel i is footprint row 2 part + (i >> 3), column i & 7: A[part * 16 + i]
                const float* sb = reinterpret_cast<const float*>(stage_buf + static_cast<size_t>(slot) * CF_BOX_BYTES) + lane * 4;
#pragma unroll
                for (int i = 0; i < 16; ++i) {
                    const float4 v = *reinterpret_cast<const float4*>(sb + i * 128);
                    const float w = A[part * 16 + i];
                    acc.x = fmaf(w, v.x, acc.x); acc.y = fmaf(w, v.y, acc.y);
                    acc.z = fmaf(w, v.z, acc.z); acc.w = fmaf(w, v.w, acc.w);
                }
                __syncwarp();                           // stage slot fully consumed (and A, after the last part)
                if (++slot == CF_STAGES) { slot = 0; parity ^= 1; }
            }
        }
        *reinterpret_cast<float4*>(g.dffeat + static_cast<size_t>(u) * 128 + lane * 4) = acc;
        cur = nxt;
        nxt = nxt2;
    }
}

// ------------------------------------------------------------------------------------------------ dlevel
constexpr int CL_THREADS = 256;       // warp r owns tile row r, lane c channels 4c..4c+3
constexpr int CL_BATCH = 32;          // overlapping units staged in shared memory per pass

struct ClArgs {
    int N;
    int H[PIPS_LEVELS], W[PIPS_LEVELS];
    int tiles_x[PIPS_LEVELS];
    int tile0[PIPS_LEVELS + 1];       // first tile of each level in a frame's tile list; tile0[4] = tiles per frame
    const float* coords;              // (B,S,N,2)
    const float* ffeat;               // (B*N*8, 128)
    const float* dcorr;               // (B*N*8, ld)
    int ld;
    float* dlvl[PIPS_LEVELS];         // (B*8, H_l, W_l, 128)
};

__global__ void __launch_bounds__(CL_THREADS)
corr_grad_levels_kernel(const __grid_constant__ ClArgs g) {
    __shared__ float4 sF[CL_BATCH][32];             // ffeats of the staged units
    __shared__ float sA[CL_BATCH][8][8];            // their adjoint weights on this tile's pixels (0 off the footprint)
    __shared__ int sN[CL_THREADS], sOx[CL_THREADS], sOy[CL_THREADS];
    __shared__ float4 sW[CL_THREADS];
    __shared__ int wcount[CL_THREADS / 32];

    const int frame = blockIdx.y, b = frame >> 3, s = frame & 7;
    const int tile = blockIdx.x;
    const int level = (tile >= g.tile0[1]) + (tile >= g.tile0[2]) + (tile >= g.tile0[3]);
    const int t = tile - g.tile0[level];
    const int ty = t / g.tiles_x[level];
    const int x0 = (t - ty * g.tiles_x[level]) * 8, y0 = ty * 8;
    const int H = g.H[level], W = g.W[level], N = g.N;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const float* coords = g.coords + static_cast<size_t>(frame) * N * 2;
    const float sc = 1.0f / static_cast<float>(1 << level);

    float4 acc[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) acc[i] = make_float4(0.f, 0.f, 0.f, 0.f);

    for (int n0 = 0; n0 < N; n0 += CL_THREADS) {
        // which of the next 256 units have a footprint on this tile: load_unit's origin, from 8 bytes each
        const int n = n0 + tid;
        bool hit = false;
        float cx = 0.f, cy = 0.f;
        int ox = 0, oy = 0;
        if (n < N) {
            const float2 c = *reinterpret_cast<const float2*>(coords + static_cast<size_t>(n) * 2);
            cx = c.x; cy = c.y;
            const float cxl = fminf(fmaxf(c.x * sc, -8.0f), static_cast<float>(W) + 8.0f);
            const float cyl = fminf(fmaxf(c.y * sc, -8.0f), static_cast<float>(H) + 8.0f);
            ox = static_cast<int>(floorf(cxl)) - PIPS_RADIUS;
            oy = static_cast<int>(floorf(cyl)) - PIPS_RADIUS;
            hit = ox < x0 + 8 && ox + 8 > x0 && oy < y0 + 8 && oy + 8 > y0;
        }
        // stable compaction: the hits keep ascending n
        const uint32_t ballot = __ballot_sync(0xffffffffu, hit);
        if (lane == 0) wcount[warp] = __popc(ballot);
        __syncthreads();
        int base = 0, hits = 0;
#pragma unroll
        for (int w = 0; w < CL_THREADS / 32; ++w) {
            base += w < warp ? wcount[w] : 0;
            hits += wcount[w];
        }
        if (hit) {
            const int k = base + __popc(ballot & ((1u << lane) - 1u));
            const TapWeights tw = tap_weights(cx, cy, level, W, H);
            sN[k] = n; sOx[k] = ox; sOy[k] = oy;
            sW[k] = make_float4(tw.w00, tw.w01, tw.w10, tw.w11);
        }
        __syncthreads();

        for (int k0 = 0; k0 < hits; k0 += CL_BATCH) {
            const int nb = min(CL_BATCH, hits - k0);
            for (int e = tid; e < nb * 64; e += CL_THREADS) {
                const int k = e >> 6, py = (e >> 3) & 7, px = e & 7;
                const int j = y0 + py - sOy[k0 + k], i = x0 + px - sOx[k0 + k];
                float v = 0.f;
                if (j >= 0 && j < 8 && i >= 0 && i < 8) {
                    const float4 w4 = sW[k0 + k];
                    const size_t u = (static_cast<size_t>(b) * N + sN[k0 + k]) * 8 + s;
                    v = adjoint_weight(g.dcorr + u * g.ld + level * 49, TapWeights{w4.x, w4.y, w4.z, w4.w}, j, i);
                }
                sA[k][py][px] = v;
            }
            for (int e = tid; e < nb * 32; e += CL_THREADS) {
                const int k = e >> 5, c4 = e & 31;
                const size_t u = (static_cast<size_t>(b) * N + sN[k0 + k]) * 8 + s;
                sF[k][c4] = *reinterpret_cast<const float4*>(g.ffeat + u * 128 + c4 * 4);
            }
            __syncthreads();
            for (int k = 0; k < nb; ++k) {
                const float4 f = sF[k][lane];
                const float4 a0 = *reinterpret_cast<const float4*>(&sA[k][warp][0]);
                const float4 a1 = *reinterpret_cast<const float4*>(&sA[k][warp][4]);
                const float av[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
#pragma unroll
                for (int i = 0; i < 8; ++i) {
                    acc[i].x = fmaf(av[i], f.x, acc[i].x); acc[i].y = fmaf(av[i], f.y, acc[i].y);
                    acc[i].z = fmaf(av[i], f.z, acc[i].z); acc[i].w = fmaf(av[i], f.w, acc[i].w);
                }
            }
            __syncthreads();
        }
    }

    const int y = y0 + warp;
    if (y < H) {
        float* row = g.dlvl[level] + (static_cast<size_t>(frame) * H + y) * W * 128 + lane * 4;
#pragma unroll
        for (int i = 0; i < 8; ++i)
            if (x0 + i < W) *reinterpret_cast<float4*>(row + static_cast<size_t>(x0 + i) * 128) = acc[i];
    }
}

// the checks both entry points share; `who` prefixes every message
static int check_problem(const char* who, int B, int S, int N, int H, int W, const float* coords, const float* dcorr,
                         int ld_dcorr) {
    char msg[160];
    auto bad = [&](const char* what) {
        snprintf(msg, sizeof msg, "%s: %s", who, what);
        return fail(msg);
    };
    if (!coords || !dcorr) return bad("null pointer");
    if (S != PIPS_S) return bad("S must be 8");
    if (B <= 0 || N <= 0) return bad("empty problem");
    if (H < 8 || W < 8) return bad("level-0 map must be at least 8x8");
    if (ld_dcorr < 4 * 49) return bad("ld_dcorr must be >= 196");
    if (static_cast<long long>(B) * S * N >= (1LL << 31)) return bad("more than 2^31 units in one call");
    if ((reinterpret_cast<uintptr_t>(coords) & 7) || (reinterpret_cast<uintptr_t>(dcorr) & 3))
        return bad("coords must be 8-byte and dcorr 4-byte aligned");
    return 0;
}

}  // namespace pips

using namespace pips;

extern "C" int pips_corr_grad_feats(const float* const* lvl, int B, int S, int N, int H, int W, const float* coords,
                                    const float* dcorr, int ld_dcorr, float* dffeat_rows, void* stream) {
    if (!lvl || !dffeat_rows) return fail("pips_corr_grad_feats: null pointer");
    if (check_problem("pips_corr_grad_feats", B, S, N, H, W, coords, dcorr, ld_dcorr)) return 1;
    CfArgs g = {};
    g.a.B = B; g.a.S = S; g.a.N = N; g.a.T = S;
    for (int l = 0, h = H, w = W; l < PIPS_LEVELS; ++l, h /= 2, w /= 2) {
        if (!lvl[l]) return fail("pips_corr_grad_feats: null level pointer");
        if (reinterpret_cast<uintptr_t>(lvl[l]) & 15) return fail("pips_corr_grad_feats: the levels and dffeat_rows must be 16-byte aligned");
        g.a.H[l] = h; g.a.W[l] = w;
    }
    if (reinterpret_cast<uintptr_t>(dffeat_rows) & 15) return fail("pips_corr_grad_feats: the levels and dffeat_rows must be 16-byte aligned");
    g.a.coords = coords;
    g.dcorr = dcorr; g.ld = ld_dcorr; g.dffeat = dffeat_rows;
    CgMaps maps;
    if (encode_level_maps(maps, reinterpret_cast<const void* const*>(lvl), CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, g.a.H, g.a.W, B * S,
                          "pips_corr_grad_feats: cuTensorMapEncodeTiled failed"))
        return 1;
    const long long units = static_cast<long long>(B) * S * N;
    long long grid = (units + CF_WARPS - 1) / CF_WARPS;
    const long long cap = static_cast<long long>(sm_count());      // 8 warps x (3 x 8 KB + 320 B) fill one SM
    if (grid > cap) grid = cap;
    return launch_kernel<corr_grad_feats_kernel>("pips_corr_grad_feats: launch", false, dim3(static_cast<unsigned>(grid)),
                                                 dim3(CF_WARPS * 32), CF_SMEM_BYTES, static_cast<cudaStream_t>(stream), maps, g);
}

extern "C" int pips_corr_grad_levels(int B, int S, int N, int H, int W, const float* coords, const float* ffeat_rows,
                                     const float* dcorr, int ld_dcorr, float* const* dlvl, void* stream) {
    if (!ffeat_rows || !dlvl) return fail("pips_corr_grad_levels: null pointer");
    if (check_problem("pips_corr_grad_levels", B, S, N, H, W, coords, dcorr, ld_dcorr)) return 1;
    if (reinterpret_cast<uintptr_t>(ffeat_rows) & 15) return fail("pips_corr_grad_levels: ffeat_rows and the levels must be 16-byte aligned");
    ClArgs g = {};
    g.N = N;
    g.tile0[0] = 0;
    for (int l = 0, h = H, w = W; l < PIPS_LEVELS; ++l, h /= 2, w /= 2) {
        if (!dlvl[l]) return fail("pips_corr_grad_levels: null level pointer");
        if (reinterpret_cast<uintptr_t>(dlvl[l]) & 15) return fail("pips_corr_grad_levels: ffeat_rows and the levels must be 16-byte aligned");
        g.H[l] = h; g.W[l] = w; g.dlvl[l] = dlvl[l];
        g.tiles_x[l] = (w + 7) / 8;
        g.tile0[l + 1] = g.tile0[l] + g.tiles_x[l] * ((h + 7) / 8);
    }
    g.coords = coords; g.ffeat = ffeat_rows; g.dcorr = dcorr; g.ld = ld_dcorr;
    if (B * S > 65535) return fail("pips_corr_grad_levels: more than 65535 frames in one call");
    return launch_kernel<corr_grad_levels_kernel>("pips_corr_grad_levels: launch", false, dim3(g.tile0[PIPS_LEVELS], B * S),
                                                  dim3(CL_THREADS), 0, static_cast<cudaStream_t>(stream), g);
}
