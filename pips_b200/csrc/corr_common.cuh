// What the local correlation's forward (corr_gather.cu) and its backward (corr_grad.cu) share: the unit decode, the
// box origins of a unit's 8x8 footprints and the tensor maps the footprint boxes are read through.  A footprint is the
// same pixels in both directions only if both use this arithmetic.
#pragma once
#include "common.cuh"

namespace pips {

constexpr int CG_ROWS_PER_BOX = 2;     // a footprint is read as 4 boxes {128 ch, 8 px, 2 rows}

struct CgMaps {
    static constexpr bool kGroups = false;
    CUtensorMap m[PIPS_LEVELS];
};

// The grouped mode of pips_corr_gather (several pyramids of different map sizes in one call): each track's clip table
// entry names its group, and group g's levels are read through m[g][l] with the dims H[g][l], W[g][l].  A
// __grid_constant__ kernel parameter, so that the per-track indexing by group reads the parameter bank directly.
struct CgGroupMaps {
    static constexpr bool kGroups = true;
    CUtensorMap m[PIPS_MAX_GROUPS][PIPS_LEVELS];
    int H[PIPS_MAX_GROUPS][PIPS_LEVELS], W[PIPS_MAX_GROUPS][PIPS_LEVELS];
};

struct CgArgs {
    int B, S, N;
    int H[PIPS_LEVELS], W[PIPS_LEVELS];
    const float* coords;     // (B,S,N,2)
    const float* ffeats;     // (B*N,S,128)
    const float* times;      // [S]
    const int* frame_base;   // optional [B*N]: window start of each track inside its clip of T frames (chained tracking)
    int T;                   // frames per batch element in the pyramid (== S when frame_base is null)
    __nv_bfloat16* x_hi;
    __nv_bfloat16* x_lo;
    float* x_f32;
    int ldx;
    const int* clip;         // optional [B*N][2] {first, count}: each track's clip in the pyramid (clip_window_frame);
                             // [B*N][4] {first, count, group, 0} in the grouped mode (CgGroupMaps)
};

// Kernel parameters are limited to 32 764 bytes (CUDA >= 12.1 on sm_70+); the grouped mode passes all its maps there.
static_assert(sizeof(CgGroupMaps) + sizeof(CgArgs) <= 32764, "grouped corr_gather parameters exceed the 32 764-byte limit");

// Frame index, inside its clip of T frames, of step s of a chained track's window (pips_init_gather reads step 0,
// pips_corr_gather steps 0..7).  base >= 0: a forward window from frame base, min(base + s, T-1) -- past the clip's
// end the last frame is replicated (chain_demo.py:50-52).  base < 0: a backward window from frame t = ~base (base =
// -1-t), max(t - s, 0) -- the same chain run on the time-reversed clip, whose last frame is frame 0 (t is clamped
// to T-1, as base is on the forward side).  Both kernels decode through this helper so that they agree on which
// frame a window starts at.
__device__ __forceinline__ int window_frame(int base, int s, int T) {
    return base >= 0 ? min(base + s, T - 1) : max(min(~base, T - 1) - s, 0);
}

// Pyramid frame of step s of track seq when every track carries its own clip (several videos in one pyramid):
// clip[seq] = {first, count} is the clip's first pyramid frame and its number of frames, and base = frame_base[seq] is
// decoded inside the clip by window_frame.  A window therefore replicates the clip's last frame going forward and
// clamps at its frame 0 going backward, and never reads another clip's frames.
__device__ __forceinline__ int clip_window_frame(const int* clip, int seq, int base, int s) {
    const int2 c = reinterpret_cast<const int2*>(clip)[seq];
    return c.x + window_frame(base, s, c.y);
}

// Level dims and tensor map of level l for a unit of pyramid group g: the call's own (CgArgs / CgMaps, g ignored) or
// group g's (CgGroupMaps).
__device__ __forceinline__ int level_w(const CgArgs& a, const CgMaps*, int, int l) { return a.W[l]; }
__device__ __forceinline__ int level_h(const CgArgs& a, const CgMaps*, int, int l) { return a.H[l]; }
__device__ __forceinline__ int level_w(const CgArgs&, const CgGroupMaps* m, int g, int l) { return m->W[g][l]; }
__device__ __forceinline__ int level_h(const CgArgs&, const CgGroupMaps* m, int g, int l) { return m->H[g][l]; }
__device__ __forceinline__ const CUtensorMap* level_map(const CgMaps& m, int, int l) { return &m.m[l]; }
__device__ __forceinline__ const CUtensorMap* level_map(const CgGroupMaps& m, int g, int l) { return &m.m[g][l]; }

struct UnitInfo {
    float cx, cy;      // coords of (b,s,n), level-0 pixels
    int frame;         // pyramid frame index (inside the track's group in the grouped mode)
    int group;         // pyramid group (grouped mode; 0 otherwise)
    int b, n, s;
    int valid;
    int ox, oy;        // lane l < 4: TMA box origin (first column, first row) of pyramid level l for this unit
};

// Unit u = (seq, s) with seq = b*N + n and s < S (the mixer's row order).  Besides the unit's coordinates every lane
// computes the box origin of ONE pyramid level (lane & 3), so that issuing a TMA box later costs two shuffles instead
// of a clamp / floor / convert chain executed by lane 0 alone while 31 lanes wait.  Coordinates are clamped in float
// so that diverged or non-finite tracks cannot overflow the int conversion (beyond +-8 px of the map all taps are zero).
// kClips: the frame comes from the per-track clip table (a.clip and a.frame_base both set).  With CgGroupMaps the table
// entry is one int4 {first, count, group, 0}, and the level dims are the group's.
template <bool kClips = false, typename Maps = CgMaps>
__device__ __forceinline__ UnitInfo load_unit(const CgArgs& a, int u, int total, const Maps* maps = nullptr) {
    UnitInfo ui;
    ui.valid = u < total;
    ui.cx = 0.f; ui.cy = 0.f; ui.frame = 0; ui.group = 0; ui.b = 0; ui.n = 0; ui.s = 0; ui.ox = 0; ui.oy = 0;
    if (ui.valid) {
        const int seq = u / a.S;
        ui.s = u - seq * a.S;
        ui.b = seq / a.N; ui.n = seq - ui.b * a.N;
        const float2 c = *reinterpret_cast<const float2*>(a.coords + ((static_cast<size_t>(ui.b) * a.S + ui.s) * a.N + ui.n) * 2);
        ui.cx = c.x; ui.cy = c.y;
        if constexpr (Maps::kGroups) {
            const int4 e = reinterpret_cast<const int4*>(a.clip)[seq];
            ui.frame = e.x + window_frame(a.frame_base[seq], ui.s, e.y);
            ui.group = e.z;
        } else if (kClips) {
            ui.frame = clip_window_frame(a.clip, seq, a.frame_base[seq], ui.s);
        } else {
            ui.frame = a.frame_base ? ui.b * a.T + window_frame(a.frame_base[seq], ui.s, a.T) : ui.b * a.S + ui.s;
        }
        const int level = threadIdx.x & 3;
        const float sc = 1.0f / static_cast<float>(1 << level);        // coords / 2**i  (nets/pips.py:373), exact
        const float cxl = fminf(fmaxf(c.x * sc, -8.0f), static_cast<float>(level_w(a, maps, ui.group, level)) + 8.0f);
        const float cyl = fminf(fmaxf(c.y * sc, -8.0f), static_cast<float>(level_h(a, maps, ui.group, level)) + 8.0f);
        ui.ox = static_cast<int>(floorf(cxl)) - PIPS_RADIUS;
        ui.oy = static_cast<int>(floorf(cyl)) - PIPS_RADIUS;
    }
    return ui;
}

// The bilinear weights of level `level` for a unit at (cx, cy): the fractional part of the clamped position, as
// load_unit clamps it.  w00 weighs footprint pixel (j, i) for tap (i, j), w01 (j, i+1), w10 (j+1, i), w11 (j+1, i+1).
struct TapWeights {
    float w00, w01, w10, w11;
};

__device__ __forceinline__ TapWeights tap_weights(float cx, float cy, int level, int W, int H) {
    const float sc = 1.0f / static_cast<float>(1 << level);
    const float cxl = fminf(fmaxf(cx * sc, -8.0f), static_cast<float>(W) + 8.0f);
    const float cyl = fminf(fmaxf(cy * sc, -8.0f), static_cast<float>(H) + 8.0f);
    const float fx = cxl - floorf(cxl), fy = cyl - floorf(cyl);
    return {(1.f - fx) * (1.f - fy), fx * (1.f - fy), (1.f - fx) * fy, fx * fy};
}

// The 4 level maps the footprint boxes {128 ch, 8 px, CG_ROWS_PER_BOX rows} are loaded through: level l is
// (frames, H[l], W[l], 128) channels-last of `es`-byte elements.  `who` prefixes the error message.
inline int encode_level_maps(CgMaps& maps, const void* const* lvl, CUtensorMapDataType dt, cuuint64_t es, const int* H,
                             const int* W, int frames, const char* who) {
    for (int l = 0; l < PIPS_LEVELS; ++l) {
        cuuint64_t gdim[4] = {128, static_cast<cuuint64_t>(W[l]), static_cast<cuuint64_t>(H[l]), static_cast<cuuint64_t>(frames)};
        cuuint64_t gstr[3] = {128 * es, static_cast<cuuint64_t>(W[l]) * 128 * es, static_cast<cuuint64_t>(H[l]) * W[l] * 128 * es};
        cuuint32_t box[4] = {128, 8, CG_ROWS_PER_BOX, 1};
        cuuint32_t estr[4] = {1, 1, 1, 1};
        if (!encode_tiled(&maps.m[l], dt, 4, const_cast<void*>(lvl[l]), gdim, gstr, box, estr, CU_TENSOR_MAP_SWIZZLE_NONE))
            return fail(who);
    }
    return 0;
}

}  // namespace pips
