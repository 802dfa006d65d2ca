// 3x3 / stride-1 / pad-1 convolution with 64 input and 64 output channels -- the four convolutions of BasicEncoder's
// layer1 (nets/pips.py:135-136, :215) -- as an implicit GEMM that loads every input row ONCE.
//
// conv_tc.cu loads the A tile of each of the 9 filter taps as its own TMA box: 9 x 32 KB per 128-pixel tile, which at
// Cin = 64 (one K-chunk per tap) makes operand traffic from L2, not the tensor cores, the limit.  Here a tile is 64
// pixels of ONE output row and the CTA walks DOWN the image:
//   * the three input rows a tile needs (y-1, y, y+1; 66 pixels each with the left/right halo, zero-filled outside the
//     image by TMA) live in a 4-slot ring of row buffers; moving to the next output row loads ONE new row (16.5 KB for
//     the (hi, lo) pair) -- 8.7x less operand traffic than 9 boxes per tile;
//   * filter tap (dr, ds) is the 64 contiguous 128-byte pixels starting at pixel ds of ring row y+dr: a wgmma
//     descriptor whose start address is offset by ds pixels (the swizzle follows absolute address bits: base offset 0);
//   * all 9 taps' weights (144 KB, hi and lo) are loaded once per CTA and stay resident;
//   * one consumer warpgroup (wgmma m64n64k16, accumulator in registers) per CTA; a work item is (image, 256-pixel column
//     block, 8 rows, 128-pixel half "rank"), done as two 64-pixel strips;
//   * InstanceNorm statistics (nets/pips.py:154-157) are accumulated in the epilogue: per work item one partial (mean,
//     M2, count) per channel -- the layout pips_inorm_finalize merges in fp64, deterministic and independent of the
//     batch size; the separate statistics pass over the layer-1 activations disappears.
// Same bf16x3 products (hi*hi + lo*hi + hi*lo, fp32 accumulation) and K order (tap-major, then channel) as conv_tc.cu.
#include "gemm_common.cuh"

namespace pips {

constexpr int R_THREADS = 256;                       // warp 0 TMA, warps 1..3 idle, warps 4..7 the consumer warpgroup
constexpr int R_ROWS_PER_ITEM = 8;
constexpr int R_RING = 4;
constexpr int R_STRIP = 64;                          // output pixels per tile
constexpr int R_BOX_PX = R_STRIP + 2;                // + 1 halo pixel on each side
constexpr uint32_t R_ROW_TX = R_BOX_PX * 128;        // bytes TMA writes per row and operand half (hi or lo)
constexpr uint32_t R_ROW_BYTES = 9 * 1024;           // slot stride (1 KB aligned: SWIZZLE_128B pattern repeats every 1 KB)
constexpr uint32_t R_W_HALF = 64 * 128, R_W_TAP = 2 * R_W_HALF;   // per tap: [w_hi 64 rows x 128 B | w_lo]
constexpr uint32_t R_OFF_W = R_RING * 2 * R_ROW_BYTES;            // 72 KB
constexpr uint32_t R_OFF_COMB = R_OFF_W + 9 * R_W_TAP;            // +144 KB
constexpr uint32_t R_OFF_BARS = R_OFF_COMB + 4 * 64 * 2 * 4;      // 4 consumer warps x 64 channels x (mean, M2)
constexpr uint32_t R_SMEM_BYTES = R_OFF_BARS + 256 + 1024;

struct RowsArgs {
    int N, H, W;
    int px_blocks;              // ceil(W / 256)
    int row_chunks;             // ceil(H / R_ROWS_PER_ITEM)
    float* out;                 // (N, H, W, 64) fp32
    float* partial;             // optional (N, px_blocks * row_chunks * 2, 3, 64)
};

__global__ void __launch_bounds__(R_THREADS, 1)
conv_rows_kernel(const __grid_constant__ CUtensorMap map_a_hi, const __grid_constant__ CUtensorMap map_a_lo,
                 const __grid_constant__ CUtensorMap map_w_hi, const __grid_constant__ CUtensorMap map_w_lo, const RowsArgs a) {
    pdl_trigger();
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~static_cast<uintptr_t>(1023));
    float* comb = reinterpret_cast<float*>(smem + R_OFF_COMB);
    uint64_t* bars = reinterpret_cast<uint64_t*>(smem + R_OFF_BARS);
    float* counts = reinterpret_cast<float*>(smem + R_OFF_BARS + 128);   // valid pixels per consumer warp and item
    const uint32_t wfull = smem_u32(bars);                 // all 9 taps loaded
    const uint32_t rfull0 = wfull + 8;                     // ring slot filled
    const uint32_t rempty0 = rfull0 + 8 * R_RING;          // ring slot free

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int items_img = a.px_blocks * a.row_chunks;
    const int num_work = a.N * items_img * 2;              // (item, rank)

    if (warp == 0 && lane == 0) {
        tma_prefetch_desc(&map_a_hi); tma_prefetch_desc(&map_a_lo);
        tma_prefetch_desc(&map_w_hi); tma_prefetch_desc(&map_w_lo);
    }
    if (warp == 1 && lane == 0) {
        mbar_init(wfull, 1);
        for (int s = 0; s < R_RING; ++s) {
            mbar_init(rfull0 + 8 * s, 1);
            mbar_init(rempty0 + 8 * s, 1);
        }
        fence_barrier_init();
    }
    __syncthreads();
    const uint32_t ring0 = smem_u32(smem), wsm0 = smem_u32(smem + R_OFF_W);

    if (warp < 4) {
        if (warp == 0 && lane == 0) {
            // ------------------------------------------------------------ TMA producer
            // the filter is a constant of the forward: loaded before the dependency wait
            mbar_arrive_expect_tx(wfull, 9 * R_W_TAP);
            for (int tap = 0; tap < 9; ++tap) {
                tma_load_2d(wsm0 + tap * R_W_TAP, &map_w_hi, wfull, tap * 64, 0);
                tma_load_2d(wsm0 + tap * R_W_TAP + R_W_HALF, &map_w_lo, wfull, tap * 64, 0);
            }
            pdl_wait();                                   // the activation comes from the previous kernel
            uint32_t ld = 0;                              // rows loaded so far: slot = ld % R_RING
            for (int work = blockIdx.x; work < num_work; work += gridDim.x) {
                const int item = work >> 1, rank = work & 1;
                const int img = item / items_img, rem = item - img * items_img;
                const int px = rem / a.row_chunks, y0 = (rem - px * a.row_chunks) * R_ROWS_PER_ITEM;
                const int y1 = min(a.H, y0 + R_ROWS_PER_ITEM);
                for (int strip = 0; strip < 2; ++strip) {
                    const int xs = px * 256 + rank * 128 + strip * R_STRIP;
                    if (xs >= a.W) continue;              // strip outside the image: nothing to compute
                    for (int yy = y0 - 1; yy <= y1; ++yy, ++ld) {
                        const uint32_t slot = ld % R_RING, phase = (ld / R_RING) & 1;
                        mbar_wait(rempty0 + 8 * slot, phase ^ 1);
                        const uint32_t fb = rfull0 + 8 * slot;
                        mbar_arrive_expect_tx(fb, 2 * R_ROW_TX);
                        tma_load_4d(ring0 + slot * 2 * R_ROW_BYTES, &map_a_hi, fb, 0, xs - 1, yy, img);
                        tma_load_4d(ring0 + slot * 2 * R_ROW_BYTES + R_ROW_BYTES, &map_a_lo, fb, 0, xs - 1, yy, img);
                    }
                }
            }
        }
    } else {
        // ------------------------------------------------------------ consumer warpgroup: MMA + epilogue
        pdl_wait();
        const int w4 = warp & 3;
        const bool releaser = (threadIdx.x & 127) == 0;
        mbar_wait(wfull, 0);
        uint32_t base_ld = 0, waited = 0;                 // first ring index of the strip; rows already waited for
        float acc[32];
        for (int work = blockIdx.x; work < num_work; work += gridDim.x) {
            const int item = work >> 1, rank = work & 1;
            const int img = item / items_img, rem = item - img * items_img;
            const int px = rem / a.row_chunks, chunk = rem - px * a.row_chunks;
            const int y0 = chunk * R_ROWS_PER_ITEM, ntiles = min(a.H, y0 + R_ROWS_PER_ITEM) - y0;
            // statistics of this thread's columns 8j + 2(lane%4), +1 over its tcount pixels of the item: sums of the
            // deviations from the first value it sees (a pixel of the same 8-row block, so sums of squares stay small)
            float shift[8][2], ssum[8][2], ssq[8][2], tcount = 0.f;
#pragma unroll
            for (int j = 0; j < 8; ++j) { ssum[j][0] = ssum[j][1] = 0.f; ssq[j][0] = ssq[j][1] = 0.f; }
            for (int strip = 0; strip < 2; ++strip) {
                const int xs = px * 256 + rank * 128 + strip * R_STRIP;
                if (xs >= a.W) continue;
                for (int j = 0; j < ntiles; ++j) {
                    wgmma_fence();
#pragma unroll
                    for (int dr = 0; dr < 3; ++dr) {
                        // rows arrive in order; the taps of filter row dr need ring index base + j + dr
                        while (waited <= base_ld + j + dr) {
                            mbar_wait(rfull0 + 8 * (waited % R_RING), (waited / R_RING) & 1);
                            ++waited;
                        }
                        const uint32_t row = ring0 + ((base_ld + j + dr) % R_RING) * 2 * R_ROW_BYTES;
#pragma unroll
                        for (int ds = 0; ds < 3; ++ds) {
                            const uint32_t wt = wsm0 + (dr * 3 + ds) * R_W_TAP;
                            // start address on pixel ds of the row buffer: the tensor core applies the 128-byte swizzle to
                            // ABSOLUTE shared-memory address bits (as TMA did when it wrote the row), so a start that is a
                            // whole number of 128-byte rows into the 1 KB pattern needs nothing else -- descriptor base offset 0
                            const uint64_t a_hi = wgmma_desc_sw128(row + ds * 128);
                            const uint64_t a_lo = wgmma_desc_sw128(row + R_ROW_BYTES + ds * 128);
                            const uint64_t w_hi = wgmma_desc_sw128(wt), w_lo = wgmma_desc_sw128(wt + R_W_HALF);
#pragma unroll
                            for (int k = 0; k < BK / MMA_K; ++k) {
                                const uint64_t adv = static_cast<uint64_t>((k * MMA_K * 2) >> 4);
                                wgmma_n64(acc, a_hi + adv, w_hi + adv, (dr | ds | k) != 0);
                                wgmma_n64(acc, a_lo + adv, w_hi + adv, 1);
                                wgmma_n64(acc, a_hi + adv, w_lo + adv, 1);
                            }
                        }
                    }
                    wgmma_commit();
                    wgmma_wait<0>();
                    wgmma_acc_ready(acc);
                    if (releaser) {
                        mbar_arrive(rempty0 + 8 * ((base_ld + j) % R_RING));          // input row y-1: last use was this tile
                        if (j == ntiles - 1) {                                          // the strip's last two rows
                            mbar_arrive(rempty0 + 8 * ((base_ld + j + 1) % R_RING));
                            mbar_arrive(rempty0 + 8 * ((base_ld + j + 2) % R_RING));
                        }
                    }
#pragma unroll
                    for (int h = 0; h < 2; ++h) {
                        const int x = xs + w4 * 16 + (lane >> 2) + 8 * h;
                        if (x < a.W) {
                            float* orow = a.out + ((static_cast<size_t>(img) * a.H + (y0 + j)) * a.W + x) * 64 + 2 * (lane & 3);
                            if (tcount == 0.f) {
#pragma unroll
                                for (int c = 0; c < 8; ++c) { shift[c][0] = acc[4 * c + 2 * h]; shift[c][1] = acc[4 * c + 2 * h + 1]; }
                            }
                            tcount += 1.f;
#pragma unroll
                            for (int c = 0; c < 8; ++c) {
                                const float2 o = make_float2(acc[4 * c + 2 * h], acc[4 * c + 2 * h + 1]);
                                *reinterpret_cast<float2*>(orow + 8 * c) = o;
                                const float dx = o.x - shift[c][0], dy = o.y - shift[c][1];
                                ssum[c][0] += dx; ssum[c][1] += dy;
                                ssq[c][0] = fmaf(dx, dx, ssq[c][0]); ssq[c][1] = fmaf(dy, dy, ssq[c][1]);
                            }
                        }
                    }
                }
                base_ld += ntiles + 2;
            }
            if (a.partial) {
                // (count, mean, M2) per thread, merged over the 8 lanes that hold the same columns (lane 0..3 keep the
                // result, always merged in the same order), then over the four warps in a fixed order
                float* mine = comb + w4 * 128;               // [column][mean, M2]
                const float inv = tcount > 0.f ? 1.f / tcount : 0.f;
                float n = tcount;
#pragma unroll
                for (int w = 4; w <= 16; w <<= 1) {
                    const float nb = __shfl_xor_sync(0xffffffffu, n, w);
                    const float f = n + nb > 0.f ? nb / (n + nb) : 0.f, g = n * f;
#pragma unroll
                    for (int c = 0; c < 8; ++c) {
#pragma unroll
                        for (int e = 0; e < 2; ++e) {
                            if (w == 4) {                    // the thread's own (mean, M2) from its shifted sums
                                const float s = ssum[c][e];
                                ssum[c][e] = tcount > 0.f ? fmaf(s, inv, shift[c][e]) : 0.f;
                                ssq[c][e] = fmaxf(ssq[c][e] - s * s * inv, 0.f);
                            }
                            const float mb = __shfl_xor_sync(0xffffffffu, ssum[c][e], w);
                            const float m2b = __shfl_xor_sync(0xffffffffu, ssq[c][e], w);
                            chan_merge(f, g, ssum[c][e], ssq[c][e], mb, m2b);
                        }
                    }
                    n += nb;
                }
                if (lane < 4) {
#pragma unroll
                    for (int c = 0; c < 8; ++c) {
#pragma unroll
                        for (int e = 0; e < 2; ++e) {
                            const int col = 8 * c + 2 * lane + e;
                            mine[col * 2] = ssum[c][e]; mine[col * 2 + 1] = ssq[c][e];
                        }
                    }
                }
                if (lane == 0) counts[w4] = n;
                asm volatile("bar.sync 1, 128;" ::: "memory");
                const int col = threadIdx.x - 128;
                if (col < 64) {
                    float n = 0.f, mean = 0.f, m2 = 0.f;
#pragma unroll
                    for (int w = 0; w < 4; ++w) {
                        if (counts[w] > 0.f) {
                            chan_merge_n(n, mean, m2, counts[w], comb[w * 128 + col * 2], comb[w * 128 + col * 2 + 1]);
                            n += counts[w];
                        }
                    }
                    float* p = a.partial + ((static_cast<size_t>(img) * items_img + rem) * 2 + rank) * 192;
                    p[col] = mean;
                    p[64 + col] = m2;
                    p[128 + col] = n;
                }
                asm volatile("bar.sync 1, 128;" ::: "memory");  // comb is rewritten by the next item
            }
        }
    }
}

}  // namespace pips

using namespace pips;

extern "C" int pips_conv_rows_chunks(int H, int W) {
    if (H <= 0 || W <= 0) return 0;
    return ((W + 255) / 256) * ((H + R_ROWS_PER_ITEM - 1) / R_ROWS_PER_ITEM) * 2;
}

// x_hi/x_lo: (N, H, W, 64) bf16; w_hi/w_lo: (64, 9*64) bf16, k = (r*3 + s)*64 + ci; out: (N, H, W, 64) fp32;
// partial (optional): (N, pips_conv_rows_chunks(H, W), 3, 64) fp32 per-chunk (mean, M2, count) of `out` per channel.
extern "C" int pips_conv_rows(const void* x_hi, const void* x_lo, int N, int H, int W, const void* w_hi, const void* w_lo,
                              float* out, float* partial, void* stream) {
    if (!x_hi || !x_lo || !w_hi || !w_lo || !out) return fail("pips_conv_rows: null pointer");
    if (N <= 0 || H <= 0 || W <= 0) return fail("pips_conv_rows: empty input");
    RowsArgs a;
    a.N = N; a.H = H; a.W = W; a.px_blocks = (W + 255) / 256; a.row_chunks = (H + R_ROWS_PER_ITEM - 1) / R_ROWS_PER_ITEM;
    a.out = out; a.partial = partial;

    CUtensorMap ma_hi, ma_lo, mw_hi, mw_lo;
    {
        cuuint64_t gdim[4] = {64, static_cast<cuuint64_t>(W), static_cast<cuuint64_t>(H), static_cast<cuuint64_t>(N)};
        cuuint64_t gstr[3] = {64 * 2, static_cast<cuuint64_t>(W) * 64 * 2, static_cast<cuuint64_t>(H) * W * 64 * 2};
        cuuint32_t box[4] = {64, R_BOX_PX, 1, 1};
        cuuint32_t estr[4] = {1, 1, 1, 1};
        if (!encode_tiled_pair(&ma_hi, &ma_lo, x_hi, x_lo, 4, gdim, gstr, box, estr, CU_TENSOR_MAP_SWIZZLE_128B))
            return fail("pips_conv_rows: activation tensor map failed");
    }
    {
        cuuint64_t gdim[2] = {9 * 64, 64};
        cuuint64_t gstr[1] = {9 * 64 * 2};
        cuuint32_t box[2] = {64, 64};
        cuuint32_t estr[2] = {1, 1};
        if (!encode_tiled_pair(&mw_hi, &mw_lo, w_hi, w_lo, 2, gdim, gstr, box, estr, CU_TENSOR_MAP_SWIZZLE_128B))
            return fail("pips_conv_rows: weight tensor map failed");
    }
    const int work = 2 * N * a.px_blocks * a.row_chunks;
    const int grid = work < sm_count() ? work : sm_count();
    return launch_kernel<conv_rows_kernel>("pips_conv_rows", true, grid, R_THREADS, R_SMEM_BYTES, static_cast<cudaStream_t>(stream), ma_hi,
                                           ma_lo, mw_hi, mw_lo, a);
}
