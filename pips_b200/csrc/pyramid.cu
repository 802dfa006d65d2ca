// Correlation pyramid and initial feature gather (run once per forward, upstream of the loop).
//   pips_pyramid_build  nets/pips.py:346-352   NCHW fp32 fmaps -> 4 channels-last levels (fp32, + optional bf16 copy)
//   pips_init_gather    utils/samp.py:5-78     bilinear sample of frame 0 at the queries, indices clamped
#include <cstdio>

#include "corr_common.cuh"   // window_frame / clip_window_frame: the chained-window decode pips_corr_gather uses

namespace pips {

// level 0: per frame (128, H*W) -> (H*W, 128); 32x32 tiles through smem so both sides are coalesced
__global__ void nchw_to_nhwc_kernel(const float* __restrict__ in, float* __restrict__ out, __nv_bfloat16* out_bf, int HW) {
    __shared__ float tile[32][33];
    const int f = blockIdx.z;
    const int p0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
    const float* src = in + static_cast<size_t>(f) * 128 * HW;
    for (int i = threadIdx.y; i < 32; i += blockDim.y) {
        const int p = p0 + threadIdx.x;
        tile[i][threadIdx.x] = p < HW ? src[static_cast<size_t>(c0 + i) * HW + p] : 0.f;
    }
    __syncthreads();
    for (int i = threadIdx.y; i < 32; i += blockDim.y) {
        const int p = p0 + i;
        if (p < HW) {
            const size_t o = (static_cast<size_t>(f) * HW + p) * 128 + c0 + threadIdx.x;
            const float v = tile[threadIdx.x][i];
            out[o] = v;
            if (out_bf) out_bf[o] = __float2bfloat16_rn(v);
        }
    }
}

// level l from level l-1: F.avg_pool2d(., 2, stride=2): floor output size, sum of the 2x2 window / 4
__global__ void avgpool2_nhwc_kernel(const float* __restrict__ in, float* __restrict__ out, __nv_bfloat16* out_bf,
                                     int frames, int Hi, int Wi, int Ho, int Wo) {
    const size_t total = static_cast<size_t>(frames) * Ho * Wo * 32;           // float4 granules
    for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < total; i += static_cast<size_t>(gridDim.x) * blockDim.x) {
        const int c4 = static_cast<int>(i & 31);
        size_t p = i >> 5;
        const int x = static_cast<int>(p % Wo); p /= Wo;
        const int y = static_cast<int>(p % Ho);
        const int f = static_cast<int>(p / Ho);
        const float4* r0 = reinterpret_cast<const float4*>(in + ((static_cast<size_t>(f) * Hi + 2 * y) * Wi + 2 * x) * 128) + c4;
        const float4* r1 = r0 + static_cast<size_t>(Wi) * 32;
        const float4 a = r0[0], b = r0[32], c = r1[0], d = r1[32];
        float4 o;
        o.x = (((a.x + b.x) + c.x) + d.x) * 0.25f;
        o.y = (((a.y + b.y) + c.y) + d.y) * 0.25f;
        o.z = (((a.z + b.z) + c.z) + d.z) * 0.25f;
        o.w = (((a.w + b.w) + c.w) + d.w) * 0.25f;
        const size_t oo = ((static_cast<size_t>(f) * Ho + y) * Wo + x) * 128 + c4 * 4;
        *reinterpret_cast<float4*>(out + oo) = o;
        if (out_bf) {
            *reinterpret_cast<uint2*>(out_bf + oo) = make_uint2(pack_bf16(__float2bfloat16_rn(o.x), __float2bfloat16_rn(o.y)),
                                                                pack_bf16(__float2bfloat16_rn(o.z), __float2bfloat16_rn(o.w)));
        }
    }
}

__global__ void f32_to_bf16_kernel(const float* __restrict__ in, __nv_bfloat16* __restrict__ out, size_t n4) {
    for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < n4; i += static_cast<size_t>(gridDim.x) * blockDim.x) {
        const float4 v = reinterpret_cast<const float4*>(in)[i];
        reinterpret_cast<uint2*>(out)[i] = make_uint2(pack_bf16(__float2bfloat16_rn(v.x), __float2bfloat16_rn(v.y)),
                                                      pack_bf16(__float2bfloat16_rn(v.z), __float2bfloat16_rn(v.w)));
    }
}

// Track `warp` = (b, n) of one init_gather warp: 4 clamped taps x 128 channels of frame `frame` of the H x W level 0,
// unclamped weights, result broadcast to the S rows.
__device__ __forceinline__ void init_gather_track(const float* __restrict__ lvl0, int S, int H, int W, int frame, float x,
                                                  float y, int warp, int lane, float* __restrict__ ffeat,
                                                  float* __restrict__ ffeats) {
    const float x0f = floorf(x), y0f = floorf(y);
    const float x1f = x0f + 1.0f, y1f = y0f + 1.0f;
    // clamp in float first so that huge / non-finite coordinates cannot overflow the int conversion
    const int x0 = static_cast<int>(fminf(fmaxf(x0f, 0.f), static_cast<float>(W - 1)));
    const int x1 = static_cast<int>(fminf(fmaxf(x1f, 0.f), static_cast<float>(W - 1)));
    const int y0 = static_cast<int>(fminf(fmaxf(y0f, 0.f), static_cast<float>(H - 1)));
    const int y1 = static_cast<int>(fminf(fmaxf(y1f, 0.f), static_cast<float>(H - 1)));
    const float w00 = (x1f - x) * (y1f - y), w01 = (x - x0f) * (y1f - y);
    const float w10 = (x1f - x) * (y - y0f), w11 = (x - x0f) * (y - y0f);
    const float* img = lvl0 + static_cast<size_t>(frame) * H * W * 128;
    const float4 a = *reinterpret_cast<const float4*>(img + (static_cast<size_t>(y0) * W + x0) * 128 + lane * 4);
    const float4 bq = *reinterpret_cast<const float4*>(img + (static_cast<size_t>(y0) * W + x1) * 128 + lane * 4);
    const float4 c = *reinterpret_cast<const float4*>(img + (static_cast<size_t>(y1) * W + x0) * 128 + lane * 4);
    const float4 d = *reinterpret_cast<const float4*>(img + (static_cast<size_t>(y1) * W + x1) * 128 + lane * 4);
    float4 o;   // same association as utils/samp.py:64-65
    o.x = ((w00 * a.x + w01 * bq.x) + w10 * c.x) + w11 * d.x;
    o.y = ((w00 * a.y + w01 * bq.y) + w10 * c.y) + w11 * d.y;
    o.z = ((w00 * a.z + w01 * bq.z) + w10 * c.z) + w11 * d.z;
    o.w = ((w00 * a.w + w01 * bq.w) + w10 * c.w) + w11 * d.w;
    *reinterpret_cast<float4*>(ffeat + static_cast<size_t>(warp) * 128 + lane * 4) = o;
    for (int s = 0; s < S; ++s)
        *reinterpret_cast<float4*>(ffeats + (static_cast<size_t>(warp) * S + s) * 128 + lane * 4) = o;
}

// one warp per (b, n).  kClips: the window starts inside the track's own clip of the pyramid (clip_window_frame).
template <bool kClips>
__global__ void init_gather_kernel(const float* __restrict__ lvl0, int B, int S, int N, int H, int W,
                                   const float* __restrict__ coords, const int* __restrict__ frame_base, int T,
                                   float* __restrict__ ffeat, float* __restrict__ ffeats, const int* __restrict__ clip) {
    const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (warp >= B * N) return;
    const int b = warp / N, n = warp % N;
    const size_t ci = ((static_cast<size_t>(b) * S + 0) * N + n) * 2;
    const float x = coords[ci], y = coords[ci + 1];
    const int frame = kClips ? clip_window_frame(clip, warp, frame_base[warp], 0)           // first frame of the track's window
                             : frame_base ? b * T + window_frame(frame_base[warp], 0, T) : b * S;
    init_gather_track(lvl0, S, H, W, frame, x, y, warp, lane, ffeat, ffeats);
}

// Level 0 of each pyramid group of pips_init_gather_groups.
struct IgGroups {
    const float* lvl0[PIPS_MAX_GROUPS];
    int H[PIPS_MAX_GROUPS], W[PIPS_MAX_GROUPS];
};

// init_gather_kernel<true> over several pyramids: table[warp] = {first, count, group, 0} (pips_corr_gather_groups).
__global__ void init_gather_groups_kernel(const __grid_constant__ IgGroups g, int B, int S, int N,
                                          const float* __restrict__ coords, const int* __restrict__ frame_base,
                                          const int4* __restrict__ table, float* __restrict__ ffeat,
                                          float* __restrict__ ffeats) {
    const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (warp >= B * N) return;
    const int b = warp / N, n = warp % N;
    const size_t ci = ((static_cast<size_t>(b) * S + 0) * N + n) * 2;
    const int4 e = table[warp];
    const int frame = e.x + window_frame(frame_base[warp], 0, e.y);
    init_gather_track(g.lvl0[e.z], S, g.H[e.z], g.W[e.z], frame, coords[ci], coords[ci + 1], warp, lane, ffeat, ffeats);
}

}  // namespace pips

using namespace pips;

static int pyramid_common(const float* fmaps, bool nhwc, int frames, int H, int W, float* const* lvl_f32,
                          void* const* lvl_bf16, void* stream) {
    if (!fmaps || !lvl_f32) return fail("pips_pyramid_build: null pointer");
    if (frames <= 0 || H < 8 || W < 8) return fail("pips_pyramid_build: need frames > 0 and H, W >= 8 (4 pooled levels)");
    for (int l = 0; l < PIPS_LEVELS; ++l)
        if (!lvl_f32[l] || (lvl_bf16 && !lvl_bf16[l])) return fail("pips_pyramid_build: null level pointer");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const int HW = H * W;
    cudaError_t e;
    if (nhwc) {
        const size_t n = static_cast<size_t>(frames) * HW * 128;
        if (fmaps != lvl_f32[0]) {
            e = cudaMemcpyAsync(lvl_f32[0], fmaps, n * sizeof(float), cudaMemcpyDeviceToDevice, st);
            if (e != cudaSuccess) return fail_cuda("pips_pyramid_build: level 0 copy", e);
        }
        if (lvl_bf16) {
            size_t blocks = (n / 4 + 255) / 256;
            if (blocks > sm_count() * 8) blocks = sm_count() * 8;
            f32_to_bf16_kernel<<<static_cast<unsigned>(blocks), 256, 0, st>>>(fmaps, static_cast<__nv_bfloat16*>(lvl_bf16[0]), n / 4);
        }
    } else {
        dim3 grid((HW + 31) / 32, 4, frames), block(32, 8);
        nchw_to_nhwc_kernel<<<grid, block, 0, st>>>(fmaps, lvl_f32[0], lvl_bf16 ? static_cast<__nv_bfloat16*>(lvl_bf16[0]) : nullptr, HW);
    }
    e = cudaGetLastError();
    if (e != cudaSuccess) return fail_cuda("pips_pyramid_build: level 0", e);
    int hi = H, wi = W;
    for (int l = 1; l < PIPS_LEVELS; ++l) {
        const int ho = hi / 2, wo = wi / 2;
        const size_t total = static_cast<size_t>(frames) * ho * wo * 32;
        size_t blocks = (total + 255) / 256;
        if (blocks > sm_count() * 8) blocks = sm_count() * 8;
        avgpool2_nhwc_kernel<<<static_cast<unsigned>(blocks), 256, 0, st>>>(
            lvl_f32[l - 1], lvl_f32[l], lvl_bf16 ? static_cast<__nv_bfloat16*>(lvl_bf16[l]) : nullptr, frames, hi, wi, ho, wo);
        e = cudaGetLastError();
        if (e != cudaSuccess) return fail_cuda("pips_pyramid_build: pooled level", e);
        hi = ho; wi = wo;
    }
    return 0;
}

extern "C" int pips_pyramid_build(const float* fmaps_nchw, int frames, int H, int W, float* const* lvl_f32,
                                  void* const* lvl_bf16, void* stream) {
    return pyramid_common(fmaps_nchw, false, frames, H, W, lvl_f32, lvl_bf16, stream);
}

extern "C" int pips_pyramid_build_nhwc(const float* fmaps_nhwc, int frames, int H, int W, float* const* lvl_f32,
                                       void* const* lvl_bf16, void* stream) {
    return pyramid_common(fmaps_nhwc, true, frames, H, W, lvl_f32, lvl_bf16, stream);
}

static int init_gather_entry(const char* who, const float* lvl0_f32, int B, int S, int N, int H, int W, const float* coords,
                             const int* frame_base, int frames_per_batch, const int* clip, float* ffeat, float* ffeats,
                             void* stream) {
    char msg[160];
    if (!lvl0_f32 || !coords || !ffeat || !ffeats) {
        snprintf(msg, sizeof(msg), "%s: null pointer", who);
        return fail(msg);
    }
    if (B <= 0 || N <= 0 || S <= 0) {
        snprintf(msg, sizeof(msg), "%s: empty problem", who);
        return fail(msg);
    }
    if (clip && !frame_base) {
        snprintf(msg, sizeof(msg), "%s: a clip table needs frame_base", who);
        return fail(msg);
    }
    const int warps = B * N;
    const dim3 grid((warps * 32 + 127) / 128), block(128);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    if (clip)
        init_gather_kernel<true><<<grid, block, 0, st>>>(lvl0_f32, B, S, N, H, W, coords, frame_base, frames_per_batch, ffeat, ffeats, clip);
    else
        init_gather_kernel<false><<<grid, block, 0, st>>>(lvl0_f32, B, S, N, H, W, coords, frame_base, frames_per_batch, ffeat, ffeats, nullptr);
    cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? 0 : fail_cuda(who, e);
}

extern "C" int pips_init_gather(const float* lvl0_f32, int B, int S, int N, int H, int W, const float* coords,
                                const int* frame_base, int frames_per_batch, float* ffeat, float* ffeats, void* stream) {
    return init_gather_entry("pips_init_gather", lvl0_f32, B, S, N, H, W, coords, frame_base, frames_per_batch, nullptr,
                             ffeat, ffeats, stream);
}

extern "C" int pips_init_gather_clips(const float* lvl0_f32, int B, int S, int N, int H, int W, const float* coords,
                                      const int* frame_base, int frames_per_batch, const int* clip, float* ffeat,
                                      float* ffeats, void* stream) {
    return init_gather_entry("pips_init_gather_clips", lvl0_f32, B, S, N, H, W, coords, frame_base, frames_per_batch, clip,
                             ffeat, ffeats, stream);
}

extern "C" int pips_init_gather_groups(const pips_groups* groups, int B, int S, int N, const float* coords,
                                       const int* frame_base, const int* table, float* ffeat, float* ffeats,
                                       void* stream) {
    if (!groups || !coords || !ffeat || !ffeats) return fail("pips_init_gather_groups: null pointer");
    if (!frame_base || !table) return fail("pips_init_gather_groups: the grouped mode needs frame_base and a table");
    if (B <= 0 || N <= 0 || S <= 0) return fail("pips_init_gather_groups: empty problem");
    if (groups->G < 1 || groups->G > PIPS_MAX_GROUPS) return fail("pips_init_gather_groups: need 1 <= G <= PIPS_MAX_GROUPS");
    IgGroups g = {};
    for (int k = 0; k < groups->G; ++k) {
        if (groups->H[k] < 8 || groups->W[k] < 8)
            return fail("pips_init_gather_groups: every group's level-0 map must be at least 8x8");
        if (groups->frames[k] < 1) return fail("pips_init_gather_groups: every group needs frames >= 1");
        if (!groups->lvl[k][0]) return fail("pips_init_gather_groups: null level pointer");
        g.lvl0[k] = static_cast<const float*>(groups->lvl[k][0]);
        g.H[k] = groups->H[k]; g.W[k] = groups->W[k];
    }
    const int warps = B * N;
    init_gather_groups_kernel<<<(warps * 32 + 127) / 128, 128, 0, static_cast<cudaStream_t>(stream)>>>(
        g, B, S, N, coords, frame_base, reinterpret_cast<const int4*>(table), ffeat, ffeats);
    cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? 0 : fail_cuda("pips_init_gather_groups", e);
}
