// Fused local correlation + motion embedding + mixer-input packing (the "corr_gather" kernel).
//
// Replaces, per refinement iteration, CorrBlock.corr (all-pairs matmul, nets/pips.py:384-398),
// CorrBlock.sample (4x grid_sample, :355-382 + :313-328), the permute/reshape/cat glue (:517-522,
// :307-308) and get_3d_embedding (utils/misc.py:44-69).  The all-pairs volume is never formed: by
// linearity, bilinearly sampling the dot-product map at the 49 taps of a level equals blending the
// dot products with the 8x8 pixel footprint those taps share (they have one common fractional
// offset).  Zero padding outside the map (grid_sample's default) is exactly the TMA out-of-bounds fill.
//
// Work unit = one (b, s, n): for each of the 4 pyramid levels four TMA boxes {128 ch, 8 px, 2 rows}
// are staged into shared memory (channels-last pyramid => every pixel is one contiguous 512 B / 256 B
// line), each lane owns 4 channels, the 16 partial dot products of a box are reduced with a 16-shuffle
// butterfly that leaves pixel i's total in lanes 2i, 2i+1, and the 7x7 blend, the sin/cos embedding and the
// feature copy are assembled in a per-warp row buffer that is written out as one contiguous mixer row.
// Every warp runs its own 3-deep TMA ring (it is both producer and consumer, so only "full" mbarriers
// are needed); 8 warps per CTA, persistent grid.
//
// Round 2: the round-1 kernel used 4-row boxes (16 KB in fp32), i.e. 50 KB of smem per warp and 4 warps per SM --
// ncu showed it latency-bound (6 % of the warp slots active, issue 26 %, L2 35 %), not bandwidth-bound.  Two-row
// boxes halve the ring (27 KB per warp) and give 8 warps per SM with the same number of bytes in flight per SM.
//
// Algorithmic bytes per unit (SURVEY.md 8d): 4 levels x 64 px x 128 ch x e_f  +  128 x 4 (query)
// +  output row.
#include <cstdio>

#include "corr_common.cuh"
#include "ptx.cuh"

namespace pips {

constexpr int CG_WARPS = 8;
constexpr int CG_STAGES = 3;
constexpr int CG_ROWBUF = PIPS_KITCHEN_PAD;   // 576 floats
constexpr uint32_t CG_AUX_BYTES = CG_ROWBUF * 4 + 64 * 4 + 128;    // per warp: row buffer, 64 dot products, 3 mbarriers

template <typename T>
struct CgCfg {
    static constexpr uint32_t kPixBytes = 128 * sizeof(T);                      // one pixel = 128 channels
    static constexpr uint32_t kBoxBytes = CG_ROWS_PER_BOX * 8 * kPixBytes;      // 8 KB (fp32) / 4 KB (bf16)
    // [warp][stage] boxes first, each aligned to its own size (the pixel order inside a box is XOR-permuted per lane,
    // which needs the box base to have zero bits where the pixel index goes), then the per-warp auxiliary blocks
    static constexpr uint32_t kSmemBytes = CG_WARPS * CG_STAGES * kBoxBytes + CG_WARPS * CG_AUX_BYTES + kBoxBytes;
};

__device__ __forceinline__ float4 ld_chan4(const float* p) { return *reinterpret_cast<const float4*>(p); }
__device__ __forceinline__ float4 ld_chan4(const __nv_bfloat16* p) {
    const uint2 u = *reinterpret_cast<const uint2*>(p);
    float4 r;
    r.x = __uint_as_float(u.x << 16);
    r.y = __uint_as_float(u.x & 0xffff0000u);
    r.z = __uint_as_float(u.y << 16);
    r.w = __uint_as_float(u.y & 0xffff0000u);
    return r;
}

// kClips: each track reads its window inside its own clip of the pyramid (CgArgs::clip, clip_window_frame).
// Maps = CgGroupMaps (with kClips): the grouped mode -- the clip table also names each track's pyramid group, whose
// tensor maps and level dims its boxes, clamps and taps use.
template <typename T, bool kClips, typename Maps = CgMaps>
__global__ void __launch_bounds__(CG_WARPS * 32)
corr_gather_kernel(const __grid_constant__ Maps maps, const CgArgs a) {
    using Cfg = CgCfg<T>;
    pdl_trigger();
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + Cfg::kBoxBytes - 1) &
                                               ~static_cast<uintptr_t>(Cfg::kBoxBytes - 1));
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    uint8_t* stage_buf = smem + static_cast<size_t>(warp) * CG_STAGES * Cfg::kBoxBytes;
    float* rowbuf = reinterpret_cast<float*>(smem + CG_WARPS * CG_STAGES * Cfg::kBoxBytes + warp * CG_AUX_BYTES);
    float* dots = rowbuf + CG_ROWBUF;
    const uint32_t bar0 = smem_u32(dots + 64);
    const uint32_t stage0 = smem_u32(stage_buf);

    const int total = a.B * a.S * a.N;
    const int nwarps = static_cast<int>(gridDim.x) * CG_WARPS;
    int u = static_cast<int>(blockIdx.x) * CG_WARPS + warp;
    if (u >= total) return;                         // whole warp exits together

    if (lane == 0) {
        for (int s = 0; s < CG_STAGES; ++s) mbar_init(bar0 + 8 * s, 1);
        fence_barrier_init();
    }
    for (int i = PIPS_KITCHEN + lane; i < CG_ROWBUF; i += 32) rowbuf[i] = 0.f;     // zero K padding, written once
    __syncwarp();

    // Lane l accumulates pixel (i ^ (l >> 1)) of a box in acc[i]: with that order every butterfly step is
    // "keep the low half, send the high half" for ALL lanes -- no per-lane selects (2 FSEL per exchanged value before).
    const uint32_t pix_xor = static_cast<uint32_t>(lane >> 1) * Cfg::kPixBytes;
    const uint32_t lane_off = static_cast<uint32_t>(lane) * 4 * sizeof(T);

    // box j of a unit: level = j >> 2, rows 2 (j & 3), 2 (j & 3) + 1 of the level's 8x8 footprint
    auto issue = [&](const UnitInfo& ui, int level, int part, int slot) {
        const int x0 = __shfl_sync(0xffffffffu, ui.ox, level);
        const int y0 = __shfl_sync(0xffffffffu, ui.oy, level) + part * CG_ROWS_PER_BOX;
        if (lane == 0) {
            const uint32_t bar = bar0 + 8 * slot;
            mbar_arrive_expect_tx(bar, Cfg::kBoxBytes);
            tma_load_4d(stage0 + slot * Cfg::kBoxBytes, level_map(maps, ui.group, level), bar, 0, x0, y0, ui.frame);
        }
    };

    pdl_wait();                                     // coords / ffeats / pyramid come from earlier kernels of the chain
    UnitInfo cur = load_unit<kClips>(a, u, total, &maps);
    UnitInfo nxt = load_unit<kClips>(a, u + nwarps, total, &maps);
    float4 q = *reinterpret_cast<const float4*>(a.ffeats + static_cast<size_t>(u) * 128 + lane * 4);
    issue(cur, 0, 0, 0);
    issue(cur, 0, 1, 1);
    int slot = 0;
    uint32_t parity = 0;

    for (; u < total; u += nwarps) {
        // prefetch the next unit's query while this one is processed
        float4 nq = make_float4(0.f, 0.f, 0.f, 0.f);
        if (nxt.valid) nq = *reinterpret_cast<const float4*>(a.ffeats + static_cast<size_t>(u + nwarps) * 128 + lane * 4);
        const UnitInfo nxt2 = load_unit<kClips>(a, u + 2 * nwarps, total, &maps);

#pragma unroll 1
        for (int level = 0; level < PIPS_LEVELS; ++level) {
#pragma unroll
            for (int part = 0; part < 4; ++part) {
                // keep the ring full: the box two ahead (same level, next level, or the next unit's first two)
                {
                    int slot2 = slot + 2;
                    if (slot2 >= CG_STAGES) slot2 -= CG_STAGES;
                    if (part < 2) issue(cur, level, part + 2, slot2);
                    else if (level < PIPS_LEVELS - 1) issue(cur, level + 1, part - 2, slot2);
                    else if (nxt.valid) issue(nxt, 0, part - 2, slot2);
                }
                mbar_wait(bar0 + 8 * slot, parity);
                const uint8_t* sb = stage_buf + static_cast<size_t>(slot) * Cfg::kBoxBytes + lane_off;
                float acc[16];
#pragma unroll
                for (int i = 0; i < 16; ++i) {
                    const float4 v = ld_chan4(reinterpret_cast<const T*>(sb + ((static_cast<uint32_t>(i) * Cfg::kPixBytes) ^ pix_xor)));
                    acc[i] = fmaf(q.w, v.w, fmaf(q.z, v.z, fmaf(q.y, v.y, q.x * v.x)));
                }
                // butterfly: after the 5 steps lanes 2p and 2p+1 hold the full dot product of pixel p of this box
#pragma unroll
                for (int i = 0; i < 8; ++i) acc[i] += __shfl_xor_sync(0xffffffffu, acc[i + 8], 16);
#pragma unroll
                for (int i = 0; i < 4; ++i) acc[i] += __shfl_xor_sync(0xffffffffu, acc[i + 4], 8);
#pragma unroll
                for (int i = 0; i < 2; ++i) acc[i] += __shfl_xor_sync(0xffffffffu, acc[i + 2], 4);
                acc[0] += __shfl_xor_sync(0xffffffffu, acc[1], 2);
                acc[0] += __shfl_xor_sync(0xffffffffu, acc[0], 1);
                // corrs / sqrt(C)  (nets/pips.py:397); dots[by * 8 + ax], by = 2 part + box row, ax = pixel in the row
                if (!(lane & 1)) dots[part * 16 + (lane >> 1)] = __fdiv_rn(acc[0], 11.313708498984761f);
                __syncwarp();                           // stage slot fully consumed, dots visible
                if (++slot == CG_STAGES) { slot = 0; parity ^= 1; }
            }
            {
                const float sc = 1.0f / static_cast<float>(1 << level);
                const float cxl = fminf(fmaxf(cur.cx * sc, -8.0f), static_cast<float>(level_w(a, &maps, cur.group, level)) + 8.0f);
                const float cyl = fminf(fmaxf(cur.cy * sc, -8.0f), static_cast<float>(level_h(a, &maps, cur.group, level)) + 8.0f);
                const float fx = cxl - floorf(cxl), fy = cyl - floorf(cyl);
                const float w00 = (1.f - fx) * (1.f - fy), w01 = fx * (1.f - fy), w10 = (1.f - fx) * fy, w11 = fx * fy;
#pragma unroll
                for (int k = lane; k < 49; k += 32) {
                    const int ax = k / 7, by = k - ax * 7;        // channel k = a*7+b samples x = cx+(a-3), y = cy+(b-3)
                    const float* d = dots + by * 8 + ax;
                    rowbuf[PIPS_C + level * 49 + k] = ((w00 * d[0] + w01 * d[1]) + w10 * d[8]) + w11 * d[9];
                }
                __syncwarp();                       // dots are rewritten by the next level
            }
        }

        // feature copy + motion embedding (utils/misc.py:44-69; flows nets/pips.py:518-520)
        {
            const float2 c0 = *reinterpret_cast<const float2*>(a.coords + (static_cast<size_t>(cur.b) * a.S * a.N + cur.n) * 2);
            const float flow_x = cur.cx - c0.x, flow_y = cur.cy - c0.y, t = a.times[cur.s];
            *reinterpret_cast<float4*>(rowbuf + lane * 4) = q;
            const float div = static_cast<float>(lane) * 31.25f;          // arange(0,64,2) * (1000/64)
            float sn, cs;
            sincosf(__fmul_rn(flow_x, div), &sn, &cs);
            rowbuf[324 + 2 * lane] = sn; rowbuf[325 + 2 * lane] = cs;
            sincosf(__fmul_rn(flow_y, div), &sn, &cs);
            rowbuf[388 + 2 * lane] = sn; rowbuf[389 + 2 * lane] = cs;
            sincosf(__fmul_rn(t, div), &sn, &cs);
            rowbuf[452 + 2 * lane] = sn; rowbuf[453 + 2 * lane] = cs;
            if (lane == 0) { rowbuf[516] = flow_x; rowbuf[517] = flow_y; rowbuf[518] = t; }
        }
        __syncwarp();
        {
            const size_t ro = static_cast<size_t>(u) * a.ldx;
            for (int g = lane; g < CG_ROWBUF / 4; g += 32) {
                const float4 v = *reinterpret_cast<const float4*>(rowbuf + g * 4);
                if (a.x_f32) *reinterpret_cast<float4*>(a.x_f32 + ro + g * 4) = v;
                if (a.x_hi) {
                    // v ~= hi + lo, both bf16 (same roundings as split_bf16, on packed pairs)
                    const uint32_t h0 = cvt_bf16x2(v.x, v.y), h1 = cvt_bf16x2(v.z, v.w);
                    *reinterpret_cast<uint2*>(a.x_hi + ro + g * 4) = make_uint2(h0, h1);
                    if (a.x_lo) {
                        const float2 l0 = fma2(make_float2(__uint_as_float(h0 << 16), __uint_as_float(h0 & 0xffff0000u)), bcast2(-1.0f),
                                               make_float2(v.x, v.y));
                        const float2 l1 = fma2(make_float2(__uint_as_float(h1 << 16), __uint_as_float(h1 & 0xffff0000u)), bcast2(-1.0f),
                                               make_float2(v.z, v.w));
                        *reinterpret_cast<uint2*>(a.x_lo + ro + g * 4) = make_uint2(cvt_bf16x2(l0.x, l0.y), cvt_bf16x2(l1.x, l1.y));
                    }
                }
            }
        }
        __syncwarp();
        cur = nxt;
        nxt = nxt2;
        q = nq;
    }
}

template <typename T, bool kClips, typename Maps>
static int launch_corr_gather(const Maps& maps, const CgArgs& args, cudaStream_t st) {
    using Cfg = CgCfg<T>;
    static bool attr[kMaxDevices] = {};
    {
        cudaError_t e = ensure_dyn_smem(corr_gather_kernel<T, kClips, Maps>, attr, static_cast<int>(Cfg::kSmemBytes));
        if (e != cudaSuccess) return fail_cuda("pips_corr_gather: smem attribute", e);
    }
    const long long units = static_cast<long long>(args.B) * args.S * args.N;
    if (units >= (1LL << 31)) return fail("pips_corr_gather: more than 2^31 units in one call");
    const int ctas_per_sm = 1;                                // 8 warps x (3 x 8 KB + 2.6 KB) fill one SM's shared memory (fp32)
    long long grid = (units + CG_WARPS - 1) / CG_WARPS;
    const long long cap = static_cast<long long>(sm_count()) * ctas_per_sm;
    if (grid > cap) grid = cap;
    cudaError_t e = launch_pdl(corr_gather_kernel<T, kClips, Maps>, dim3(static_cast<unsigned>(grid)), dim3(CG_WARPS * 32), Cfg::kSmemBytes, st, maps, args);
    if (e == cudaSuccess) e = cudaGetLastError();
    return e == cudaSuccess ? 0 : fail_cuda("pips_corr_gather: launch", e);
}

template <typename T, bool kClips>
static int launch_corr_gather(const void* const* lvl, CUtensorMapDataType dt, const CgArgs& args, int frames, cudaStream_t st) {
    CgMaps maps;
    if (encode_level_maps(maps, lvl, dt, sizeof(T), args.H, args.W, frames, "pips_corr_gather: cuTensorMapEncodeTiled failed"))
        return 1;
    return launch_corr_gather<T, kClips, CgMaps>(maps, args, st);
}

// The grouped mode: group g's 4 level maps and dims; its levels are (frames[g], H[g] >> l, W[g] >> l, 128).
template <typename T>
static int launch_corr_gather_groups(const pips_groups& g, CUtensorMapDataType dt, const CgArgs& args, cudaStream_t st) {
    CgGroupMaps maps;
    for (int k = 0; k < g.G; ++k) {
        int h = g.H[k], w = g.W[k];
        for (int l = 0; l < PIPS_LEVELS; ++l) {
            maps.H[k][l] = h; maps.W[k][l] = w; h /= 2; w /= 2;
        }
        CgMaps one;
        if (encode_level_maps(one, g.lvl[k], dt, sizeof(T), maps.H[k], maps.W[k], g.frames[k],
                              "pips_corr_gather_groups: cuTensorMapEncodeTiled failed"))
            return 1;
        for (int l = 0; l < PIPS_LEVELS; ++l) maps.m[k][l] = one.m[l];
    }
    return launch_corr_gather<T, true, CgGroupMaps>(maps, args, st);
}

}  // namespace pips

using namespace pips;

// pips_corr_gather and pips_corr_gather_clips: `who` names the entry point in error messages
static int corr_gather_entry(const char* who, const void* const* lvl, int feat_dtype, int B, int S, int N, int H, int W,
                             const float* coords, const float* ffeats, const float* times, const int* frame_base,
                             int frames_per_batch, const int* clip, void* x_hi, void* x_lo, float* x_f32, int ldx,
                             void* stream) {
    char msg[160];
    auto err = [&](const char* what) {
        snprintf(msg, sizeof(msg), "%s: %s", who, what);
        return fail(msg);
    };
    if (!lvl || !coords || !ffeats || !times) return err("null pointer");
    if (clip ? S != PIPS_S : (S < 2 || S > PIPS_S_MAX)) return err(clip ? "S must be 8" : "S must be in 2..16");
    if (B <= 0 || N <= 0) return err("empty problem");
    if (H < 8 || W < 8) return err("level-0 map must be at least 8x8");
    if (!x_hi && !x_f32) return err("no output buffer");
    if (x_lo && !x_hi) return err("x_lo without x_hi");
    if (ldx < PIPS_KITCHEN_PAD || (ldx % 8)) return err("ldx must be >= 576 and a multiple of 8");
    CgArgs a;
    a.B = B; a.S = S; a.N = N;
    int h = H, w = W;
    for (int l = 0; l < PIPS_LEVELS; ++l) {
        if (!lvl[l]) return err("null level pointer");
        a.H[l] = h; a.W[l] = w; h /= 2; w /= 2;
    }
    if (frame_base && frames_per_batch <= 0) return err("frame_base needs frames_per_batch > 0");
    if (clip && !frame_base) return err("a clip table needs frame_base");
    a.coords = coords; a.ffeats = ffeats; a.times = times;
    a.frame_base = frame_base; a.T = frame_base ? frames_per_batch : S;
    a.x_hi = static_cast<__nv_bfloat16*>(x_hi); a.x_lo = static_cast<__nv_bfloat16*>(x_lo); a.x_f32 = x_f32; a.ldx = ldx;
    a.clip = clip;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    if (feat_dtype == PIPS_FEAT_F32)
        return clip ? launch_corr_gather<float, true>(lvl, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, a, B * a.T, st)
                    : launch_corr_gather<float, false>(lvl, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, a, B * a.T, st);
    if (feat_dtype == PIPS_FEAT_BF16)
        return clip ? launch_corr_gather<__nv_bfloat16, true>(lvl, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, a, B * a.T, st)
                    : launch_corr_gather<__nv_bfloat16, false>(lvl, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, a, B * a.T, st);
    return err("unknown feat_dtype");
}

extern "C" int pips_corr_gather(const void* const* lvl, int feat_dtype, int B, int S, int N, int H, int W, const float* coords,
                                const float* ffeats, const float* times, const int* frame_base, int frames_per_batch,
                                void* x_hi, void* x_lo, float* x_f32, int ldx, void* stream) {
    return corr_gather_entry("pips_corr_gather", lvl, feat_dtype, B, S, N, H, W, coords, ffeats, times, frame_base,
                             frames_per_batch, nullptr, x_hi, x_lo, x_f32, ldx, stream);
}

extern "C" int pips_corr_gather_clips(const void* const* lvl, int feat_dtype, int B, int S, int N, int H, int W,
                                      const float* coords, const float* ffeats, const float* times, const int* frame_base,
                                      int frames_per_batch, const int* clip, void* x_hi, void* x_lo, float* x_f32, int ldx,
                                      void* stream) {
    return corr_gather_entry("pips_corr_gather_clips", lvl, feat_dtype, B, S, N, H, W, coords, ffeats, times, frame_base,
                             frames_per_batch, clip, x_hi, x_lo, x_f32, ldx, stream);
}

extern "C" int pips_corr_gather_groups(const pips_groups* groups, int feat_dtype, int B, int S, int N, const float* coords,
                                       const float* ffeats, const float* times, const int* frame_base, const int* table,
                                       void* x_hi, void* x_lo, float* x_f32, int ldx, void* stream) {
    const char* who = "pips_corr_gather_groups";
    char msg[160];
    auto err = [&](const char* what) {
        snprintf(msg, sizeof(msg), "%s: %s", who, what);
        return fail(msg);
    };
    if (!groups || !coords || !ffeats || !times) return err("null pointer");
    if (!frame_base || !table) return err("the grouped mode needs frame_base and a table");
    if (S != PIPS_S) return err("S must be 8");
    if (B <= 0 || N <= 0) return err("empty problem");
    if (groups->G < 1 || groups->G > PIPS_MAX_GROUPS) return err("need 1 <= G <= PIPS_MAX_GROUPS");
    for (int k = 0; k < groups->G; ++k) {
        if (groups->H[k] < 8 || groups->W[k] < 8) return err("every group's level-0 map must be at least 8x8");
        if (groups->frames[k] < 1) return err("every group needs frames >= 1");
        for (int l = 0; l < PIPS_LEVELS; ++l)
            if (!groups->lvl[k][l]) return err("null level pointer");
    }
    if (!x_hi && !x_f32) return err("no output buffer");
    if (x_lo && !x_hi) return err("x_lo without x_hi");
    if (ldx < PIPS_KITCHEN_PAD || (ldx % 8)) return err("ldx must be >= 576 and a multiple of 8");
    CgArgs a = {};
    a.B = B; a.S = S; a.N = N;
    a.coords = coords; a.ffeats = ffeats; a.times = times;
    a.frame_base = frame_base; a.T = 0;                        // frames and dims come from each track's group
    a.x_hi = static_cast<__nv_bfloat16*>(x_hi); a.x_lo = static_cast<__nv_bfloat16*>(x_lo); a.x_f32 = x_f32; a.ldx = ldx;
    a.clip = table;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    if (feat_dtype == PIPS_FEAT_F32) return launch_corr_gather_groups<float>(*groups, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, a, st);
    if (feat_dtype == PIPS_FEAT_BF16)
        return launch_corr_gather_groups<__nv_bfloat16>(*groups, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, a, st);
    return err("unknown feat_dtype");
}
