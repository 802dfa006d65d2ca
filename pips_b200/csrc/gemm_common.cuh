// Shared pieces of the wgmma kernels (gemm_tc.cu, conv_tc.cu, conv_rows.cu).
#pragma once
#include <cuda_bf16.h>

#include "common.cuh"
#include "ptx.cuh"

namespace pips {

constexpr int BK = 64;                       // 64 bf16 = one 128-byte swizzle row
constexpr int MMA_K = 16;

}  // namespace pips
