// LayerNorm / row-store helpers shared by the token-mixing kernels (mixer_simt.cu, tokenmix_tc.cu).
#pragma once
#include "common.cuh"

namespace pips {

// ------------------------------------------------------------------------------------------ LN helpers
// One CTA of 128 threads owns 8 rows x 512 channels of one sequence, thread t holds channels 4t..4t+3 of
// every row.  Row statistics need a 128-thread reduction: warp shuffle + 4-entry smem exchange.
constexpr int TM_THREADS = 128;

__device__ __forceinline__ void block_sum8(float (&v)[8], float (*red)[8]) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
#pragma unroll
    for (int s = 0; s < 8; ++s) v[s] = warp_sum(v[s]);
    __syncthreads();                       // previous use of `red` is finished
    if (lane == 0) {
#pragma unroll
        for (int s = 0; s < 8; ++s) red[warp][s] = v[s];
    }
    __syncthreads();
#pragma unroll
    for (int s = 0; s < 8; ++s) v[s] = red[0][s] + red[1][s] + red[2][s] + red[3][s];
}

// two-pass LayerNorm over 512 channels (biased variance, eps 1e-5) of the 8 rows held as x[s][0..3]
__device__ __forceinline__ void layernorm8(const float (&x)[8][4], float (&y)[8][4], const float4 g, const float4 b, float (*red)[8]) {
    float m[8], q[8];
#pragma unroll
    for (int s = 0; s < 8; ++s) m[s] = (x[s][0] + x[s][1]) + (x[s][2] + x[s][3]);
    block_sum8(m, red);
#pragma unroll
    for (int s = 0; s < 8; ++s) {
        m[s] *= (1.0f / 512.0f);
        float d0 = x[s][0] - m[s], d1 = x[s][1] - m[s], d2 = x[s][2] - m[s], d3 = x[s][3] - m[s];
        q[s] = (d0 * d0 + d1 * d1) + (d2 * d2 + d3 * d3);
    }
    block_sum8(q, red);
#pragma unroll
    for (int s = 0; s < 8; ++s) {
        const float r = rsqrtf(q[s] * (1.0f / 512.0f) + 1e-5f);
        y[s][0] = (x[s][0] - m[s]) * r * g.x + b.x;
        y[s][1] = (x[s][1] - m[s]) * r * g.y + b.y;
        y[s][2] = (x[s][2] - m[s]) * r * g.z + b.z;
        y[s][3] = (x[s][3] - m[s]) * r * g.w + b.w;
    }
}

// layernorm8 for CTAs of several 128-thread groups, each normalising its own 8 rows: `red` is [warps of the CTA][8]
// and the sums run over the 4 warps of the thread's group, in layernorm8's order.
__device__ __forceinline__ void block_sum8_wg(float (&v)[8], float (*red)[8]) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, w0 = warp & ~3;
#pragma unroll
    for (int s = 0; s < 8; ++s) v[s] = warp_sum(v[s]);
    __syncthreads();
    if (lane == 0) {
#pragma unroll
        for (int s = 0; s < 8; ++s) red[warp][s] = v[s];
    }
    __syncthreads();
#pragma unroll
    for (int s = 0; s < 8; ++s) v[s] = red[w0][s] + red[w0 + 1][s] + red[w0 + 2][s] + red[w0 + 3][s];
}

__device__ __forceinline__ void layernorm8_wg(const float (&x)[8][4], float (&y)[8][4], const float4 g, const float4 b, float (*red)[8]) {
    float m[8], q[8];
#pragma unroll
    for (int s = 0; s < 8; ++s) m[s] = (x[s][0] + x[s][1]) + (x[s][2] + x[s][3]);
    block_sum8_wg(m, red);
#pragma unroll
    for (int s = 0; s < 8; ++s) {
        m[s] *= (1.0f / 512.0f);
        float d0 = x[s][0] - m[s], d1 = x[s][1] - m[s], d2 = x[s][2] - m[s], d3 = x[s][3] - m[s];
        q[s] = (d0 * d0 + d1 * d1) + (d2 * d2 + d3 * d3);
    }
    block_sum8_wg(q, red);
#pragma unroll
    for (int s = 0; s < 8; ++s) {
        const float r = rsqrtf(q[s] * (1.0f / 512.0f) + 1e-5f);
        y[s][0] = (x[s][0] - m[s]) * r * g.x + b.x;
        y[s][1] = (x[s][1] - m[s]) * r * g.y + b.y;
        y[s][2] = (x[s][2] - m[s]) * r * g.z + b.z;
        y[s][3] = (x[s][3] - m[s]) * r * g.w + b.w;
    }
}

__device__ __forceinline__ void store_row4(const float (&v)[4], size_t off, __nv_bfloat16* hi, __nv_bfloat16* lo, float* f32) {
    if (f32) *reinterpret_cast<float4*>(f32 + off) = make_float4(v[0], v[1], v[2], v[3]);
    if (hi) {
        __nv_bfloat16 h[4], l[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) split_bf16(v[i], h[i], l[i]);
        *reinterpret_cast<uint2*>(hi + off) = make_uint2(pack_bf16(h[0], h[1]), pack_bf16(h[2], h[3]));
        if (lo) *reinterpret_cast<uint2*>(lo + off) = make_uint2(pack_bf16(l[0], l[1]), pack_bf16(l[2], l[3]));
    }
}


}  // namespace pips
