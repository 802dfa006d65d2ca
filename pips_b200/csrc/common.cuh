// Shared host/device helpers of libpips_b200.
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/pips_b200.h"

namespace pips {

// error reporting (thread-local message behind pips_last_error())
int fail(const char* msg);
int fail_cuda(const char* where, cudaError_t e);

int sm_count();          // of the CURRENT device (cached per device)

// Opt-in to > 48 KB of dynamic shared memory.  cudaFuncSetAttribute applies to the current device only, so the
// "already done" flag is kept per device (a process that drives several GPUs -- nn.DataParallel -- needs it on each).
constexpr int kMaxDevices = 64;
int current_device();
template <typename F>
inline cudaError_t ensure_dyn_smem(F* func, bool (&done)[kMaxDevices], int bytes) {
    const int dev = current_device();
    if (dev >= 0 && dev < kMaxDevices && done[dev]) return cudaSuccess;
    cudaError_t e = cudaFuncSetAttribute(func, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
    if (e == cudaSuccess && dev >= 0 && dev < kMaxDevices) done[dev] = true;
    return e;
}

// cuTensorMapEncodeTiled through the runtime's driver entry point (the library does not link libcuda,
// so it also loads on a machine without a driver -- the CPU-side ABI tests rely on that).
bool encode_tiled(CUtensorMap* map, CUtensorMapDataType dtype, uint32_t rank, void* base, const cuuint64_t* gdim,
                  const cuuint64_t* gstride_bytes, const cuuint32_t* box, const cuuint32_t* estride,
                  CUtensorMapSwizzle swizzle);

// the tensor maps of a bf16 (hi, lo) pair of tensors with the same geometry
inline bool encode_tiled_pair(CUtensorMap* map_hi, CUtensorMap* map_lo, const void* hi, const void* lo, uint32_t rank,
                              const cuuint64_t* gdim, const cuuint64_t* gstride_bytes, const cuuint32_t* box,
                              const cuuint32_t* estride, CUtensorMapSwizzle swizzle) {
    return encode_tiled(map_hi, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, rank, const_cast<void*>(hi), gdim, gstride_bytes, box, estride, swizzle) &&
           encode_tiled(map_lo, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, rank, const_cast<void*>(lo), gdim, gstride_bytes, box, estride, swizzle);
}

// ---- programmatic dependent launch (PDL).  Kernels of the per-iteration chain are launched with
// cudaLaunchAttributeProgrammaticStreamSerialization: the next kernel's CTAs may become resident and run their
// prologue (barrier init, tensor-map prefetch, weight staging into shared memory) while the previous
// kernel drains; pdl_wait() blocks until every prerequisite grid has completed and its writes are visible, so it must
// precede the first access to any buffer another kernel of the chain writes (and any global write).  pdl_trigger()
// (issued at kernel entry) lets the dependent grid be scheduled as soon as all CTAs of this grid have started.
// RULE: only kernels that call pdl_wait() may be launched through launch_pdl().
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

bool pdl_enabled();          // PIPS_B200_PDL != "0" (abi.cu)

// `pdl` = false: a plain launch
template <typename... KArgs, typename... Args>
inline cudaError_t launch_ex(void (*kernel)(KArgs...), bool pdl, dim3 grid, dim3 block, size_t smem, cudaStream_t st, Args&&... args) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = st;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = pdl && pdl_enabled() ? 1 : 0;
    return cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);
}

template <typename... KArgs, typename... Args>
inline cudaError_t launch_pdl(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, Args&&... args) {
    return launch_ex(kernel, true, grid, block, smem, st, static_cast<Args&&>(args)...);
}

// A kernel with `smem` bytes of dynamic shared memory: sets the opt-in on the current device (once per device and
// kernel), launches with PDL when `pdl` (see the RULE above) and reports a failure as `name`'s.
template <auto Kernel, typename... Args>
inline int launch_kernel(const char* name, bool pdl, dim3 grid, dim3 block, uint32_t smem, cudaStream_t st, Args&&... args) {
    static bool smem_set[kMaxDevices] = {};
    cudaError_t e = ensure_dyn_smem(Kernel, smem_set, static_cast<int>(smem));
    if (e == cudaSuccess) e = launch_ex(Kernel, pdl, grid, block, smem, st, static_cast<Args&&>(args)...);
    if (e == cudaSuccess) e = cudaGetLastError();
    return e == cudaSuccess ? 0 : fail_cuda(name, e);
}

__device__ __forceinline__ uint32_t pack_bf16(__nv_bfloat16 a, __nv_bfloat16 b) {
    return static_cast<uint32_t>(__bfloat16_as_ushort(a)) | (static_cast<uint32_t>(__bfloat16_as_ushort(b)) << 16);
}

// v ~= hi + lo
__device__ __forceinline__ void split_bf16(float v, __nv_bfloat16& hi, __nv_bfloat16& lo) {
    hi = __float2bfloat16_rn(v);
    lo = __float2bfloat16_rn(v - __bfloat162float(hi));
}

// InstanceNorm partial statistics are (count, mean, M2 = sum of squared deviations from the mean): sums of squares
// about zero cancel catastrophically in q/n - mean^2 when the mean is large against the spread (flat frames), while
// every term of this pairwise update (Chan, Golub & LeVeque) is non-negative.  (mean, m2) of n values absorbs (mb, m2b)
// of nb values, with f = nb / (n + nb) and g = n * f (callers that merge many columns of equal counts compute them once).
__device__ __forceinline__ void chan_merge(float f, float g, float& mean, float& m2, float mb, float m2b) {
    const float d = mb - mean;
    mean = fmaf(d, f, mean);
    m2 += m2b + d * d * g;
}

__device__ __forceinline__ void chan_merge_n(float n, float& mean, float& m2, float nb, float mb, float m2b) {
    const float f = nb / (n + nb);
    chan_merge(f, n * f, mean, m2, mb, m2b);
}

// two floats -> packed bf16x2 (round to nearest even), `lo_elem` in the low half
__device__ __forceinline__ uint32_t cvt_bf16x2(float lo_elem, float hi_elem) {
    uint32_t r;
    asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(hi_elem), "f"(lo_elem));
    return r;
}

__device__ __forceinline__ float gelu_exact(float v) {
    // nn.GELU() default (approximate='none'): 0.5 x (1 + erf(x / sqrt(2)))
    return 0.5f * v * (1.0f + erff(v * 0.70710678118654752440f));
}

// d/dx of the exact GELU: Phi(x) + x phi(x), with erfc so that the negative tail keeps its relative accuracy
__device__ __forceinline__ float gelu_grad_exact(float v) {
    return 0.5f * erfcf(-v * 0.70710678118654752440f) + v * 0.39894228040143267794f * expf(-0.5f * v * v);
}

// GELU(x) = x * Phi(x) with Phi(-|x|) = 0.5 erfc(|x|/sqrt2) ~= 0.5 (a1 t + ... + a6 t^6) exp(-x^2/2),
// t = 1/(1 + p |x|/sqrt2): a 6-term Abramowitz-Stegun-form fit (max error of the fit 7.8e-9, about
// 4e-7 relative after fp32 evaluation -- the same class as an erff-based evaluation, ~12 instructions
// instead of ~30 and branch-free).  Phi(x) for x > 0 is 1 - Phi(-x), so the negative tail has no
// cancellation.  Used where GELU sits on a hot epilogue (FC1, token mixing).
__device__ __forceinline__ float gelu_fast(float x) {
    // constants folded: t = 1/(1 + (p/sqrt2)|x|), coefficients pre-multiplied by 0.5, exponent -(x^2/2) log2(e)
    float t;
    asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(t) : "f"(fmaf(0.27599915312530316f, fabsf(x), 1.0f)));
    float q = -0.11345264142344407f;
    q = fmaf(q, t, 0.44082137646110525f);
    q = fmaf(q, t, -0.31387114090663395f);
    q = fmaf(q, t, 0.3221595132029044f);
    q = fmaf(q, t, 0.04671841449512236f);
    q = fmaf(q, t, 0.11762447426235381f);
    float e;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(x * x * -0.7213475204444817f));
    q = q * t * e;                                     // Phi(-|x|)
    return x * (x > 0.0f ? 1.0f - q : q);
}

// ---- fp32 pairs: the same roundings per element as the scalar intrinsics (no contraction across calls) ----
__device__ __forceinline__ float2 fma2(float2 a, float2 b, float2 c) { return make_float2(__fmaf_rn(a.x, b.x, c.x), __fmaf_rn(a.y, b.y, c.y)); }
__device__ __forceinline__ float2 mul2(float2 a, float2 b) { return make_float2(__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y)); }
__device__ __forceinline__ float2 add2(float2 a, float2 b) { return make_float2(__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y)); }
__device__ __forceinline__ float2 bcast2(float v) { return make_float2(v, v); }

// gelu_fast on two values at once: identical arithmetic per lane (same roundings).
__device__ __forceinline__ float2 gelu_fast2(float2 x) {
    const float2 d = fma2(bcast2(0.27599915312530316f), make_float2(fabsf(x.x), fabsf(x.y)), bcast2(1.0f));
    float2 t;
    asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(t.x) : "f"(d.x));
    asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(t.y) : "f"(d.y));
    float2 q = fma2(bcast2(-0.11345264142344407f), t, bcast2(0.44082137646110525f));
    q = fma2(q, t, bcast2(-0.31387114090663395f));
    q = fma2(q, t, bcast2(0.3221595132029044f));
    q = fma2(q, t, bcast2(0.04671841449512236f));
    q = fma2(q, t, bcast2(0.11762447426235381f));
    const float2 ea = mul2(mul2(x, x), bcast2(-0.7213475204444817f));
    float2 e;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e.x) : "f"(ea.x));
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e.y) : "f"(ea.y));
    q = mul2(mul2(q, t), e);                           // Phi(-|x|)
    const float2 omq = fma2(q, bcast2(-1.0f), bcast2(1.0f));
    return mul2(x, make_float2(x.x > 0.0f ? omq.x : q.x, x.y > 0.0f ? omq.y : q.y));
}

// GELU(x) = x Phi(x) on two values, written without the sign select of gelu_fast2 (above):
//   Phi(-|x|) = q(t) e^{-x^2/2},  t = 1 / (1 + p |x|)      (same 6-term fit)
//   x Phi(x)  = x/2 + |x| (1/2 - Phi(-|x|))                 for both signs
// The rearrangement rounds 1/2 - Phi(-|x|) once more: an ABSOLUTE error of
// <= |x| 3e-8 (1e-7 at x = -3), far below the 2^-17 relative error of the bf16 (hi, lo) pair the value is then split into.
__device__ __forceinline__ float2 gelu_fast2_abs(float2 x) {
    const float2 a = make_float2(fabsf(x.x), fabsf(x.y));
    const float2 d = fma2(bcast2(0.27599915312530316f), a, bcast2(1.0f));
    float2 t;
    asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(t.x) : "f"(d.x));
    asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(t.y) : "f"(d.y));
    float2 q = fma2(bcast2(0.11345264142344407f), t, bcast2(-0.44082137646110525f));      // coefficients negated: q = -poly
    q = fma2(q, t, bcast2(0.31387114090663395f));
    q = fma2(q, t, bcast2(-0.3221595132029044f));
    q = fma2(q, t, bcast2(-0.04671841449512236f));
    q = fma2(q, t, bcast2(-0.11762447426235381f));
    const float2 ea = mul2(mul2(x, x), bcast2(-0.7213475204444817f));
    float2 e;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e.x) : "f"(ea.x));
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e.y) : "f"(ea.y));
    const float2 w = fma2(mul2(q, t), e, bcast2(0.5f));                                    // 1/2 - Phi(-|x|)
    return fma2(a, w, mul2(x, bcast2(0.5f)));
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

}  // namespace pips
