// Thin inline-PTX wrappers for the sm_90a features the kernels use:
// mbarrier, TMA (cp.async.bulk.tensor, with cluster multicast), warpgroup MMA (wgmma), clusters.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace pips {

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
    return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

__device__ __forceinline__ bool elect_one() {
    uint32_t pred;
    asm volatile("{\n\t.reg .pred p;\n\telect.sync _|p, 0xffffffff;\n\tselp.b32 %0, 1, 0, p;\n\t}" : "=r"(pred));
    return pred != 0;
}

// ---------------------------------------------------------------- mbarrier
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_barrier_init() {
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async_smem() {
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint32_t bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint32_t bar, uint32_t parity) {
    uint32_t ok;
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.b32 %0, 1, 0, p;\n\t}"
        : "=r"(ok)
        : "r"(bar), "r"(parity)
        : "memory");
    return ok != 0;
}
// Bounded wait: a pipeline bug must surface as a trap (launch error), never as a hung GPU.
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
    if (mbar_try_wait(bar, parity)) return;
    const long long t0 = clock64();
    while (!mbar_try_wait(bar, parity)) {
        if (clock64() - t0 > 4000000000LL) __trap();   // ~2 s at 2 GHz
    }
}

__device__ __forceinline__ void st_shared_u32(uint32_t addr, uint32_t v) {
    asm volatile("st.shared.b32 [%0], %1;" ::"r"(addr), "r"(v) : "memory");
}
__device__ __forceinline__ void st_shared_f32x2(uint32_t addr, float2 v) {
    asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(addr), "f"(v.x), "f"(v.y) : "memory");
}
__device__ __forceinline__ void st_shared_u32x2(uint32_t addr, uint32_t x, uint32_t y) {
    asm volatile("st.shared.v2.b32 [%0], {%1, %2};" ::"r"(addr), "r"(x), "r"(y) : "memory");
}
__device__ __forceinline__ void st_shared_f32x4(uint32_t addr, float4 v) {
    asm volatile("st.shared.v4.f32 [%0], {%1, %2, %3, %4};" ::"r"(addr), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
}
__device__ __forceinline__ float4 ld_shared_f32x4(uint32_t addr) {
    float4 v;
    asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(addr) : "memory");
    return v;
}

// ---------------------------------------------------------------- TMA
__device__ __forceinline__ void tma_prefetch_desc(const void* map) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(map)) : "memory");
}
__device__ __forceinline__ void tma_load_2d(uint32_t dst, const void* map, uint32_t bar, int c0, int c1) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
        ::"r"(dst), "l"(reinterpret_cast<uint64_t>(map)), "r"(bar), "r"(c0), "r"(c1)
        : "memory");
}
__device__ __forceinline__ void tma_load_4d(uint32_t dst, const void* map, uint32_t bar, int c0, int c1, int c2, int c3) {
    asm volatile(
        "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
        ::"r"(dst), "l"(reinterpret_cast<uint64_t>(map)), "r"(bar), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
        : "memory");
}

// shared -> global tensor stores; each issuing thread tracks its own bulk groups
__device__ __forceinline__ void tma_store_2d(const void* map, uint32_t src, int c0, int c1) {
    asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];"
                 ::"l"(reinterpret_cast<uint64_t>(map)), "r"(src), "r"(c0), "r"(c1)
                 : "memory");
}
// global[box] += shared[box], element-wise in the tensor map's data type
__device__ __forceinline__ void tma_reduce_add_2d(const void* map, uint32_t src, int c0, int c1) {
    asm volatile("cp.reduce.async.bulk.tensor.2d.global.shared::cta.add.tile.bulk_group [%0, {%2, %3}], [%1];"
                 ::"l"(reinterpret_cast<uint64_t>(map)), "r"(src), "r"(c0), "r"(c1)
                 : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
// at most N of this thread's groups still read their shared-memory source
template <int N>
__device__ __forceinline__ void bulk_wait_read() { asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory"); }
// at most N of this thread's groups are still in flight (writes included)
template <int N>
__device__ __forceinline__ void bulk_wait() { asm volatile("cp.async.bulk.wait_group %0;" ::"n"(N) : "memory"); }

// barrier among `threads` threads of the CTA (a warpgroup: 128) on hardware barrier `id` (0 is __syncthreads)
__device__ __forceinline__ void named_bar_sync(uint32_t id, uint32_t threads) {
    asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(threads) : "memory");
}

// ---------------------------------------------------------------- clusters
__device__ __forceinline__ uint32_t cluster_ctarank() {
    uint32_t r;
    asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
    return r;
}
__device__ __forceinline__ void cluster_sync_all() {
    asm volatile("barrier.cluster.arrive.aligned;\n\tbarrier.cluster.wait.aligned;" ::: "memory");
}
// arrive on the barrier at the same shared-memory offset in CTA `cta` of the cluster
__device__ __forceinline__ void mbar_arrive_cluster(uint32_t local_bar, uint32_t cta) {
    asm volatile(
        "{\n\t.reg .b32 ra;\n\tmapa.shared::cluster.u32 ra, %0, %1;\n\t"
        "mbarrier.arrive.shared::cluster.b64 _, [ra];\n\t}"
        ::"r"(local_bar), "r"(cta)
        : "memory");
}
// one load, written to the same offset (and signalled on the same barrier offset) in every CTA of `cta_mask`
__device__ __forceinline__ void tma_load_2d_multicast(uint32_t dst, const void* map, uint32_t bar, int c0, int c1, uint16_t cta_mask) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes.multicast::cluster [%0], [%1, {%3, %4}], [%2], %5;"
        ::"r"(dst), "l"(reinterpret_cast<uint64_t>(map)), "r"(bar), "r"(c0), "r"(c1), "h"(cta_mask)
        : "memory");
}

// ---------------------------------------------------------------- wgmma (warpgroup MMA, accumulators in registers)
// D[64 x N, registers of the 128 threads of a warpgroup] (+)= A[64 x 16, smem desc] * B[N x 16, smem desc]^T, bf16 inputs,
// fp32 accumulation, both operands K-major.  Thread (warp w of the warpgroup, lane l) holds, for every 8-column block j,
//   d[4j], d[4j+1]: row 16w + l/4,     columns 8j + 2(l%4), +1        d[4j+2], d[4j+3]: row 16w + l/4 + 8, same columns.
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int PENDING>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(PENDING) : "memory"); }
// keeps the compiler from reading accumulator registers before the wgmma_wait that makes them valid
template <int R>
__device__ __forceinline__ void wgmma_acc_ready(float (&d)[R]) {
#pragma unroll
    for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

#define PIPS_ACC4(d, i) "+f"(d[i]), "+f"(d[i + 1]), "+f"(d[i + 2]), "+f"(d[i + 3])
#define PIPS_ACC8(d, i) PIPS_ACC4(d, i), PIPS_ACC4(d, i + 4)
#define PIPS_ACC16(d, i) PIPS_ACC8(d, i), PIPS_ACC8(d, i + 8)
#define PIPS_ACC32(d, i) PIPS_ACC16(d, i), PIPS_ACC16(d, i + 16)
#define PIPS_ACC64(d, i) PIPS_ACC32(d, i), PIPS_ACC32(d, i + 32)

__device__ __forceinline__ void wgmma_n8(float (&d)[4], uint64_t a_desc, uint64_t b_desc, uint32_t accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %6, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n8k16.f32.bf16.bf16 "
        "{%0, %1, %2, %3}, "
        "%4, %5, p, 1, 1, 0, 0;\n\t}"
        : PIPS_ACC4(d, 0)
        : "l"(a_desc), "l"(b_desc), "r"(accumulate)
        : "memory");
}
__device__ __forceinline__ void wgmma_n16(float (&d)[8], uint64_t a_desc, uint64_t b_desc, uint32_t accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %10, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n16k16.f32.bf16.bf16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7}, "
        "%8, %9, p, 1, 1, 0, 0;\n\t}"
        : PIPS_ACC8(d, 0)
        : "l"(a_desc), "l"(b_desc), "r"(accumulate)
        : "memory");
}
__device__ __forceinline__ void wgmma_n32(float (&d)[16], uint64_t a_desc, uint64_t b_desc, uint32_t accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n32k16.f32.bf16.bf16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, "
        "%16, %17, p, 1, 1, 0, 0;\n\t}"
        : PIPS_ACC16(d, 0)
        : "l"(a_desc), "l"(b_desc), "r"(accumulate)
        : "memory");
}
__device__ __forceinline__ void wgmma_n64(float (&d)[32], uint64_t a_desc, uint64_t b_desc, uint32_t accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, "
        "%32, %33, p, 1, 1, 0, 0;\n\t}"
        : PIPS_ACC32(d, 0)
        : "l"(a_desc), "l"(b_desc), "r"(accumulate)
        : "memory");
}
__device__ __forceinline__ void wgmma_n128(float (&d)[64], uint64_t a_desc, uint64_t b_desc, uint32_t accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
        "%64, %65, p, 1, 1, 0, 0;\n\t}"
        : PIPS_ACC64(d, 0)
        : "l"(a_desc), "l"(b_desc), "r"(accumulate)
        : "memory");
}
__device__ __forceinline__ void wgmma_n256(float (&d)[128], uint64_t a_desc, uint64_t b_desc, uint32_t accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %130, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n256k16.f32.bf16.bf16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
        "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, "
        "%64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, %80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, "
        "%96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, %112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127}, "
        "%128, %129, p, 1, 1, 0, 0;\n\t}"
        : PIPS_ACC64(d, 0), PIPS_ACC64(d, 64)
        : "l"(a_desc), "l"(b_desc), "r"(accumulate)
        : "memory");
}

// D[64 x 128] (+)= A[64 x 16, registers] * B[16 x 128, smem desc, MN-major], bf16 inputs, fp32 accumulation.  A is held
// like the mma.m16n8k16 A fragment per warp (rows 16w..16w+15 of the warpgroup): a[0] = (row l/4, columns 2(l%4), +1),
// a[1] = row + 8, a[2] = columns + 8, a[3] = both -- so the accumulator columns 16k..16k+15 of an earlier wgmma,
// {d[8k], d[8k+1]}, {d[8k+2], d[8k+3]}, {d[8k+4], d[8k+5]}, {d[8k+6], d[8k+7]} packed to bf16x2, are an A fragment as they are.
__device__ __forceinline__ void wgmma_n128_rA_tb(float (&d)[64], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3,
                                                 uint64_t b_desc, uint32_t accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %69, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
        "{%64, %65, %66, %67}, %68, p, 1, 1, 1;\n\t}"
        : PIPS_ACC64(d, 0)
        : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "l"(b_desc), "r"(accumulate)
        : "memory");
}

// D[64 x 128] (+)= A[64 x 16] * B[16 x 128], both from shared memory MN-major (wgmma_desc_sw64_mn): the weight-gradient
// GEMM, whose two operands are stored with the contraction index as the row.
__device__ __forceinline__ void wgmma_n128_tt(float (&d)[64], uint64_t a_desc, uint64_t b_desc, uint32_t accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
        "%64, %65, p, 1, 1, 1, 1;\n\t}"
        : PIPS_ACC64(d, 0)
        : "l"(a_desc), "l"(b_desc), "r"(accumulate)
        : "memory");
}

// 64 x BN tile: BN = 256 as two N = 128 instructions on the two 128-row halves of the B tile (128-byte rows)
template <int BN>
__device__ __forceinline__ void wgmma_tile(float (&d)[BN / 2], uint64_t a_desc, uint64_t b_desc, uint32_t accumulate) {
    if constexpr (BN == 64) {
        wgmma_n64(d, a_desc, b_desc, accumulate);
    } else if constexpr (BN == 128) {
        wgmma_n128(d, a_desc, b_desc, accumulate);
    } else {
        static_assert(BN == 256, "tile widths: 64, 128, 256");
        wgmma_n128(*reinterpret_cast<float(*)[64]>(&d[0]), a_desc, b_desc, accumulate);
        wgmma_n128(*reinterpret_cast<float(*)[64]>(&d[64]), a_desc, b_desc + ((128 * 128) >> 4), accumulate);
    }
}

// K-major, 128-byte-swizzled operand tile (rows of 64 bf16 = 128 B, 8-row groups 1024 B apart):
// the layout TMA writes with CU_TENSOR_MAP_SWIZZLE_128B and a {64, rows} box.
__device__ __forceinline__ uint64_t wgmma_desc_sw128(uint32_t smem_addr) {
    uint64_t d = 0;
    d |= static_cast<uint64_t>((smem_addr & 0x3FFFF) >> 4);      // start address, 16 B units
    d |= static_cast<uint64_t>(1) << 16;                          // leading byte offset (unused: one swizzle atom along K)
    d |= static_cast<uint64_t>(1024 >> 4) << 32;                  // stride byte offset between 8-row groups
    d |= static_cast<uint64_t>(1) << 62;                          // SWIZZLE_128B
    return d;
}
// K-major, 64-byte-swizzled operand tile (rows of 32 bf16 = 64 B, 8-row groups 512 B apart):
// the layout TMA writes with CU_TENSOR_MAP_SWIZZLE_64B and a {32, rows} box.
__device__ __forceinline__ uint64_t wgmma_desc_sw64(uint32_t smem_addr) {
    uint64_t d = 0;
    d |= static_cast<uint64_t>((smem_addr & 0x3FFFF) >> 4);      // start address, 16 B units
    d |= static_cast<uint64_t>(1) << 16;                          // leading byte offset (unused: one swizzle atom along K)
    d |= static_cast<uint64_t>(512 >> 4) << 32;                   // stride byte offset between 8-row groups
    d |= static_cast<uint64_t>(2) << 62;                          // SWIZZLE_64B
    return d;
}
// MN-major, 64-byte-swizzled operand (transposed B): the same 64-byte rows as wgmma_desc_sw64, read with the row index as
// K and the 32 elements of a row as MN.  Each 8-row group of a buffer is one MN-major SW64 atom (32 MN x 8 K); atoms
// along K are 512 B apart (stride byte offset) and the 32-wide MN blocks are `mn_block_bytes` apart (leading byte offset).
__device__ __forceinline__ uint64_t wgmma_desc_sw64_mn(uint32_t smem_addr, uint32_t mn_block_bytes) {
    uint64_t d = 0;
    d |= static_cast<uint64_t>((smem_addr & 0x3FFFF) >> 4);      // start address, 16 B units
    d |= static_cast<uint64_t>((mn_block_bytes >> 4) & 0x3FFF) << 16;   // leading byte offset: next 32 MN elements
    d |= static_cast<uint64_t>(512 >> 4) << 32;                   // stride byte offset: next 8 K rows
    d |= static_cast<uint64_t>(2) << 62;                          // SWIZZLE_64B
    return d;
}

}  // namespace pips
