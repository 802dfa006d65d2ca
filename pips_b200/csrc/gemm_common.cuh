// Shared pieces of the wgmma kernels (gemm_tc.cu, conv_tc.cu, conv_rows.cu).
#pragma once
#include <cuda_bf16.h>

#include "common.cuh"
#include "ptx.cuh"

namespace pips {

constexpr int BK = 64;                       // 64 bf16 = one 128-byte swizzle row
constexpr int MMA_K = 16;

struct GemmArgs {
    int M, N, K;                 // valid rows / cols, K multiple of 64
    const float* bias;           // [N]
    int epilogue;                // PIPS_EPI_*
    float* out_f32;              // BIAS / BIAS_RESID target (row stride ldo)
    int ldo;
    __nv_bfloat16* out_hi;       // BIAS_GELU target (row stride ldh); out_lo may be null
    __nv_bfloat16* out_lo;
    int ldh;
};

// Epilogue of a warpgroup's 64 x BN accumulator (wgmma fragment layout, ptx.cuh): bias, then GELU + (hi, lo) split, or
// fp32 store with optional residual.  Every thread owns column pairs (col, col + 1) of two rows, so stores are 8-byte
// (fp32) or 4-byte (bf16 pair) pieces and the four threads of a quad cover 32 / 16 contiguous bytes of a row.
// `row0` is the first of the warpgroup's 64 rows, `n0` the tile's first column.
template <int BN>
__device__ __forceinline__ void epilogue_frag(const GemmArgs& args, const float (&acc)[BN / 2], int row0, int n0) {
    const int lane = threadIdx.x & 31;
    const int r0 = row0 + ((threadIdx.x >> 5) & 3) * 16 + (lane >> 2);
    const bool gelu = args.epilogue == PIPS_EPI_BIAS_GELU, resid = args.epilogue == PIPS_EPI_BIAS_RESID;
#pragma unroll
    for (int j = 0; j < BN / 8; ++j) {
        const int col = n0 + 8 * j + 2 * (lane & 3);
        if (col >= args.N) continue;
        const bool two = col + 1 < args.N;
        const float2 b = make_float2(__ldg(args.bias + col), two ? __ldg(args.bias + col + 1) : 0.f);
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int row = r0 + 8 * h;
            if (row >= args.M) continue;
            const float2 f = add2(make_float2(acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1]), b);
            if (gelu) {
                const float2 g = gelu_fast2_abs(f);
                const uint32_t hw = cvt_bf16x2(g.x, g.y);
                const float2 lo = fma2(make_float2(__uint_as_float(hw << 16), __uint_as_float(hw & 0xffff0000u)), bcast2(-1.0f), g);   // g - hi, one rounding
                const uint32_t lw = cvt_bf16x2(lo.x, lo.y);
                const size_t o = static_cast<size_t>(row) * args.ldh + col;
                if (two) {
                    *reinterpret_cast<uint32_t*>(args.out_hi + o) = hw;
                    if (args.out_lo) *reinterpret_cast<uint32_t*>(args.out_lo + o) = lw;
                } else {
                    args.out_hi[o] = __ushort_as_bfloat16(static_cast<unsigned short>(hw & 0xffffu));
                    if (args.out_lo) args.out_lo[o] = __ushort_as_bfloat16(static_cast<unsigned short>(lw & 0xffffu));
                }
            } else {
                float* po = args.out_f32 + static_cast<size_t>(row) * args.ldo + col;
                if (two) {
                    float2 o = f;
                    if (resid) { const float2 r = *reinterpret_cast<const float2*>(po); o.x += r.x; o.y += r.y; }
                    *reinterpret_cast<float2*>(po) = o;
                } else {
                    po[0] = resid ? po[0] + f.x : f.x;
                }
            }
        }
    }
}

}  // namespace pips
