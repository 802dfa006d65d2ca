// Shared pieces of the score-map kernels (scoremap_loss.cu, scoremap_grad.cu).  Both are GEMMs over K = 128 channels
// between a resident tile X of 128 rows (bf16 hi and lo, all of K, in shared memory) and 64-row tiles Y streamed through
// a 4-stage TMA ring: warp 0 produces, two consumer warpgroups take 64 rows of X each.  Both operands are K-major in
// K-blocks of 32 channels (one 64-byte swizzle row), the hi K-blocks first, then the lo ones.
#pragma once
#include "gemm_common.cuh"

namespace pips {
namespace smap {

constexpr int C = PIPS_C;                              // 128 = K of the score GEMM
constexpr int BM = 128;                                // resident rows per CTA: two consumer warpgroups of 64
constexpr int BN = 64;                                 // streamed rows per ring stage
constexpr int KB = 32;                                 // K-block: 32 bf16 = one 64-byte swizzle row
constexpr int NKB = C / KB;                            // 4
constexpr int STAGES = 4;
constexpr int THREADS = 384;                           // producer warpgroup + 2 consumer warpgroups
constexpr uint32_t X_KB_BYTES = BM * KB * 2;           // 8 KB: one K-block of the resident tile (hi or lo)
constexpr uint32_t X_BYTES = 2 * NKB * X_KB_BYTES;     // 64 KB: hi and lo, all of K
constexpr uint32_t Y_KB_BYTES = BN * KB * 2;           // 4 KB
constexpr uint32_t Y_STAGE_BYTES = 2 * NKB * Y_KB_BYTES;   // 32 KB
constexpr uint32_t SMEM_BYTES = 1024 /*align*/ + X_BYTES + STAGES * Y_STAGE_BYTES + 256 /*barriers*/;
static_assert(SMEM_BYTES <= 227u * 1024u, "resident tile + ring must fit in 227 KB");

// byte `byte` of row `row` in a K-block of 64-byte rows, swizzled the way TMA writes CU_TENSOR_MAP_SWIZZLE_64B
// (the 16-byte unit is XORed with (row / 2) % 4): the layout wgmma_desc_sw64 describes
__device__ __forceinline__ uint32_t sw64(int row, int byte) {
    const uint32_t o = static_cast<uint32_t>(row * 64 + byte);
    return o ^ (((o >> 7) & 3u) << 4);
}

// the resident tile X at the start of shared memory, the ring behind it
__device__ __forceinline__ Ring y_ring(uint8_t* smem) {
    return Ring(smem + X_BYTES, Y_STAGE_BYTES, STAGES, reinterpret_cast<uint64_t*>(smem + X_BYTES + STAGES * Y_STAGE_BYTES), STAGES);
}

// producer: streamed rows row .. row + BN - 1, all of K, hi and lo, into the next ring slot
__device__ __forceinline__ void load_y(Ring& ring, const CUtensorMap* y_hi, const CUtensorMap* y_lo, int row) {
    ring.produce([&](uint32_t base, uint32_t fb) {
#pragma unroll
        for (int kb = 0; kb < NKB; ++kb) {
            tma_load_2d(base + kb * Y_KB_BYTES, y_hi, fb, kb * KB, row);
            tma_load_2d(base + (NKB + kb) * Y_KB_BYTES, y_lo, fb, kb * KB, row);
        }
    });
}

// The resident tile from fp32 rows split into (hi, lo) bf16: tile row r is row x0 + r, the C floats at row_ptr(x0 + r),
// or zero when x0 + r >= rows.  The 256 consumer threads (ct = 0..255) share the work.
template <typename RowPtr>
__device__ __forceinline__ void fill_x_f32(uint8_t* smem, int ct, int x0, int rows, RowPtr row_ptr) {
    for (int i = ct; i < BM * (C / 4); i += 256) {
        const int r = i >> 5, c4 = i & 31;
        const int x = x0 + r;
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        if (x < rows) v = __ldg(reinterpret_cast<const float4*>(row_ptr(x)) + c4);
        const uint32_t h01 = cvt_bf16x2(v.x, v.y), h23 = cvt_bf16x2(v.z, v.w);
        const uint32_t l01 = cvt_bf16x2(v.x - __uint_as_float(h01 << 16), v.y - __uint_as_float(h01 & 0xffff0000u));
        const uint32_t l23 = cvt_bf16x2(v.z - __uint_as_float(h23 << 16), v.w - __uint_as_float(h23 & 0xffff0000u));
        const int k = 4 * c4, kb = k / KB;
        const uint32_t off = sw64(r, (k % KB) * 2);
        const uint32_t hi = smem_u32(smem + kb * X_KB_BYTES) + off;
        const uint32_t lo = smem_u32(smem + (NKB + kb) * X_KB_BYTES) + off;
        asm volatile("st.shared.v2.b32 [%0], {%1, %2};" ::"r"(hi), "r"(h01), "r"(h23) : "memory");
        asm volatile("st.shared.v2.b32 [%0], {%1, %2};" ::"r"(lo), "r"(l01), "r"(l23) : "memory");
    }
}

// S = X Y^T in bf16x3 for the warpgroup's 64 rows of X (x_hi, x_lo: their first K-block) and the ring slot at `y`;
// returns with the MMAs complete
__device__ __forceinline__ void score_mma(float (&s)[BN / 2], uint32_t x_hi, uint32_t x_lo, uint32_t y) {
    wgmma_fence();
#pragma unroll
    for (int kb = 0; kb < NKB; ++kb) {
        const uint64_t xh = wgmma_desc_sw64(x_hi + kb * X_KB_BYTES);
        const uint64_t xl = wgmma_desc_sw64(x_lo + kb * X_KB_BYTES);
        const uint64_t yh = wgmma_desc_sw64(y + kb * Y_KB_BYTES);
        const uint64_t yl = wgmma_desc_sw64(y + (NKB + kb) * Y_KB_BYTES);
#pragma unroll
        for (int k = 0; k < KB / MMA_K; ++k) {
            const uint64_t adv = static_cast<uint64_t>((k * MMA_K * 2) >> 4);   // 32 B per K=16 step
            auto mma = [&](uint64_t a, uint64_t b, uint32_t accumulate) { wgmma_n64(s, a + adv, b + adv, accumulate); };
            mma_bf16x3(mma, xh, xl, yh, yl, (kb | k) != 0);
        }
    }
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_acc_ready(s);
}

}  // namespace smap
}  // namespace pips
