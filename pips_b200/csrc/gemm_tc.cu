// Mixer dense layers on the Hopper tensor cores (wgmma, accumulators in registers).
//
//   C[M,N] = epilogue( A[M,K] . W[N,K]^T + bias[N] )
//
// A (activations) and W (nn.Linear weight, (out,in) == N x K, K-major) are bf16.  In the
// "bf16x3" precision mode both operands are carried as a (hi, lo) bf16 pair with
// v ~= hi + lo, and the product is evaluated as A_hi.W_hi + A_lo.W_hi + A_hi.W_lo with fp32
// accumulation (relative error ~2^-16 per product instead of 2^-8), which is what the
// 1e-3 px parity target of the refinement loop needs (reference: fp32 nn.Linear,
// nets/pips.py:104-107,:115,:122).
//
// Structure (one CTA per SM, persistent over 128 x BN output tiles; BN = 256 for large problems, 128 / 64 when
// 256-wide tiles would leave most SMs without a tile -- few particles: the demo clip, chained windows):
//   warp 0       TMA producer  : cp.async.bulk.tensor 64B-swizzled 32-wide K-blocks of A and W -> smem ring
//   warps 1..3   epilogue warps (BN = 256): bias / GELU + (hi, lo) split / residual of the tiles handed over to them
//   warps 4..7   consumer warpgroup 0: rows 0..63 of the tile   } wgmma m64nBNk16 straight from the ring, then the
//   warps 8..11  consumer warpgroup 1: rows 64..127             } epilogue or the handoff (below)
// The ring is 3 (x3, BN = 256) to 8 stages deep, so a slot's TMA has several K-blocks of MMAs to land in.
//
// Epilogue, BN = 256: a consumer writes its 64 x 256 accumulator into a shared-memory handoff buffer (one warpgroup's
// half; the two take turns, guarded by mbarriers) as 32-column fp32 chunks in the 128-byte-swizzled layout of the fp32
// store box, and goes straight on to the next tile's MMAs.  The epilogue warps add the bias chunk by chunk -- in place,
// then a TMA store (a TMA add-reduce for the residual); or for GELU they write the bf16 hi and lo boxes over the chunk's
// fp32 values -- so the GELU runs under the next tile's MMAs.  The epilogue warps are the producer warpgroup's idle
// warps.  A fourth, dedicated warpgroup (512 threads, registers split with setmaxnreg) measured slower: the 128-register
// launch bound of a 512-thread CTA is below what ptxas needs to compile one m64n256k16 wgmma (C7602, "register target
// of 154"), so its consumers must issue two m64n128k16 per term and read A twice; FC2 and gemm_in lost 4-9 %.
// BN = 128 / 64: bias / GELU + (hi, lo) split in the consumers' registers, then 32-column chunks of the warpgroup's 64
// rows go through a double-buffered staging area in shared memory to one TMA store per chunk.  No thread waits on
// global memory.  TMA clips the boxes at M and N, which covers partial tiles.
//
// CLUSTER = 2 ("pair" tiles, 256 x 256 per cluster): the two CTAs of a cluster take the two 128-row halves of the tile
// and share its W tile -- each loads one 128-row half of W and TMA-multicasts it into both shared memories, which
// halves the W traffic from L2.  A ring slot is then released by the consumers of BOTH CTAs.
#include <stdlib.h>

#include <string>

#include "gemm_common.cuh"

namespace pips {

constexpr int BM = 128;
constexpr int KB = 32;                                 // K-block of the ring: 32 bf16 = one 64-byte swizzle row
constexpr int GEMM_THREADS = 384;                      // producer warpgroup + 2 consumer warpgroups
constexpr uint32_t A_TILE_BYTES = BM * KB * 2;         // 8 KB
constexpr int EPI_COLS = 32;                           // epilogue chunk: 32 columns of a warpgroup's 64 rows
constexpr uint32_t EPI_BUF_BYTES = 64 * EPI_COLS * 4;  // 8 KB: an fp32 chunk, or a bf16 hi chunk + a bf16 lo chunk
constexpr uint32_t EPI_STAGING_BYTES = 2 * 2 * EPI_BUF_BYTES;   // in-consumer epilogue: two buffers per consumer warpgroup
constexpr int EPI_THREADS = 96;                        // epilogue warps: warps 1..3 of the producer warpgroup

// kHandoff: the 256-wide inference tiles, whose consumers hand their accumulators to epilogue warps through a buffer
// of one 64 x BN fp32 half (a buffer for both halves leaves room for only 2 ring stages, and measured slower).
// Otherwise (128 / 64-wide tiles, aux, weight gradient): the consumers run the epilogue from registers.
template <int TERMS, int BN, bool INFERENCE = false>
struct GemmCfg {
    static constexpr bool kHandoff = INFERENCE && BN == 256;
    static constexpr uint32_t kWTileBytes = BN * KB * 2;                  // 16 / 8 / 4 KB
    static constexpr int kOperandCopies = TERMS == 3 ? 2 : 1;             // hi (+ lo)
    static constexpr uint32_t kStageBytes = kOperandCopies * (A_TILE_BYTES + kWTileBytes);
    static constexpr uint32_t kHalfBytes = 64 * BN * 4;                   // one consumer warpgroup's fp32 accumulator
    static constexpr uint32_t kEpiBytes = kHandoff ? kHalfBytes : EPI_STAGING_BYTES;
    static constexpr uint32_t kFixedBytes = 1024 /*align*/ + kEpiBytes + 256 /*barriers*/;
    static constexpr int kFit = static_cast<int>((227u * 1024u - kFixedBytes) / kStageBytes);
    static constexpr int kStages = kFit > 8 ? 8 : kFit;
    static constexpr uint32_t kSmemBytes = kStages * kStageBytes + kFixedBytes;
    static_assert(kStages >= 3 && kSmemBytes <= 227u * 1024u, "ring + epilogue buffer must fit in 227 KB");
};

struct GemmArgs {
    int M, N, K;                 // valid rows / cols, K multiple of 64
    const float* bias;           // [N]
    int epilogue;                // PIPS_EPI_*
    float* out_f32;              // BIAS / BIAS_RESID target (row stride ldo)
    int ldo;
    __nv_bfloat16* out_hi;       // BIAS_GELU / _PRE / GELU_GRAD target (row stride ldh); out_lo may be null
    __nv_bfloat16* out_lo;
    int ldh;
    int num_tiles;               // output tiles of the launched variant (set by its launcher)
    // the fields below are read by the aux and weight-gradient variants only
    float* aux;                  // BIAS_GELU_PRE: pre-activation out; GELU_GRAD: pre-activation in (row stride ld_aux)
    int ld_aux;
    int kb_per_split;            // weight-gradient variant: K-blocks (32 rows of M) per split of M
};

__host__ __device__ __forceinline__ bool bf16_epilogue(int epi) {
    return epi == PIPS_EPI_BIAS_GELU || epi == PIPS_EPI_BIAS_GELU_PRE || epi == PIPS_EPI_GELU_GRAD;
}

struct GemmMaps {
    CUtensorMap a_hi, a_lo, w_hi, w_lo;    // operands: {KB, rows} boxes, 64-byte swizzle
    CUtensorMap out_f32;                   // BIAS / BIAS_RESID target: {32, 64} fp32 boxes, 128-byte swizzle
    CUtensorMap out_hi, out_lo;            // BIAS_GELU targets: {32, 64} bf16 boxes, 64-byte swizzle
};

template <int BN>
__device__ __forceinline__ void gemm_mma(float (&d)[BN / 2], uint64_t a_desc, uint64_t b_desc, uint32_t accumulate) {
    if constexpr (BN == 256) wgmma_n256(d, a_desc, b_desc, accumulate);
    else wgmma_tile<BN>(d, a_desc, b_desc, accumulate);
}

// Offset of byte `byte` of row `row` in a staging chunk with PITCH-byte rows, swizzled the way TMA reads it with a
// swizzle span of PITCH (128 B: the 16-byte unit is XORed with row % 8; 64 B: with (row / 2) % 4).  The swizzle also
// spreads the 8 rows that a warp writes at once over distinct banks.
template <int PITCH>
__device__ __forceinline__ uint32_t staged(int row, int byte) {
    const uint32_t o = static_cast<uint32_t>(row * PITCH + byte);
    return o ^ (((o >> 7) & (PITCH / 16 - 1)) << 4);
}

// Columns of the output that its tensor map covers.  A TMA store writes whole 16-byte units of a row, so an fp32 map N
// wide would also write the up to 3 columns past N that share the last unit (the pad columns of a row of delta at odd S,
// PIPS_DELTA_LD); the fp32 map stops at N rounded down to a multiple of 4, and the epilogue threads store the last N % 4
// columns themselves (store_tail).
__host__ __device__ __forceinline__ int tma_cols(const GemmArgs& args) {
    return bf16_epilogue(args.epilogue) ? args.N : (args.N & ~3);
}

// fp32 value v of (row, col) when col is one of the last N % 4 columns, which the output map does not cover
__device__ __forceinline__ void store_tail(const GemmArgs& args, int row, int col, float v) {
    if (row < args.M && col >= (args.N & ~3) && col < args.N) {
        float* o = args.out_f32 + static_cast<size_t>(row) * args.ldo + col;
        *o = args.epilogue == PIPS_EPI_BIAS_RESID ? *o + v : v;                  // as the reduce-add: the bits of (acc + b) + x
    }
}

// Epilogue of a warpgroup's 64 x BN accumulator (wgmma fragment layout, ptx.cuh).  `row0` is the first of the
// warpgroup's rows, `n0` the tile's first column, `staging` its two EPI_BUF_BYTES buffers; `chunk` counts the chunks
// this warpgroup has staged so far (it picks the buffer and tells when a buffer has had a store issued from it).
// AUX: the pre-activation epilogues (BIAS_GELU_PRE, GELU_GRAD) -- a separate instantiation, so the plain ones keep
// their registers.
template <int BN, bool AUX = false>
__device__ __forceinline__ void epilogue_tma(const GemmMaps& maps, const GemmArgs& args, const float (&acc)[BN / 2], int row0,
                                             int n0, uint32_t staging, uint32_t& chunk, int wg) {
    if (row0 >= args.M) return;                                           // whole warpgroup past M: nothing to store
    const int lane = threadIdx.x & 31;
    const int r = ((threadIdx.x >> 5) & 3) * 16 + (lane >> 2);           // fragment rows r, r + 8 of the 64
    const int cq = 2 * (lane & 3);                                        // fragment columns cq, cq + 1 of each 8
    const bool issuer = (threadIdx.x & 127) == 0;
    const bool gelu = AUX ? bf16_epilogue(args.epilogue) : args.epilogue == PIPS_EPI_BIAS_GELU;
#pragma unroll
    for (int c = 0; c < BN / EPI_COLS; ++c) {
        const int col0 = n0 + c * EPI_COLS;
        if (col0 >= args.N) break;
        const uint32_t buf = staging + (chunk & 1) * EPI_BUF_BYTES;
        if (issuer && chunk >= 2) bulk_wait_read<1>();                   // the store issued from buf two chunks ago has read it
        named_bar_sync(1 + wg, 128);
#pragma unroll
        for (int jj = 0; jj < EPI_COLS / 8; ++jj) {
            const int j = c * (EPI_COLS / 8) + jj;
            const int col = col0 + 8 * jj + cq;
            const float2 b = make_float2(col < args.N ? __ldg(args.bias + col) : 0.f, col + 1 < args.N ? __ldg(args.bias + col + 1) : 0.f);
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const float2 f = add2(make_float2(acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1]), b);
                if (gelu) {
                    float2 g;
                    if constexpr (AUX) {
                        // the aux epilogues require N % 8 == 0, so col < N covers col + 1
                        const int row = row0 + r + 8 * h;
                        const bool inside = row < args.M && col < args.N;
                        float* aux = args.aux + static_cast<size_t>(row) * args.ld_aux + col;
                        if (args.epilogue == PIPS_EPI_GELU_GRAD) {
                            const float2 pre = inside ? __ldg(reinterpret_cast<const float2*>(aux)) : make_float2(0.f, 0.f);
                            g = mul2(f, make_float2(gelu_grad_exact(pre.x), gelu_grad_exact(pre.y)));
                        } else {
                            g = gelu_fast2_abs(f);
                            if (inside) *reinterpret_cast<float2*>(aux) = f;
                        }
                    } else {
                        g = gelu_fast2_abs(f);
                    }
                    const uint32_t hw = cvt_bf16x2(g.x, g.y);
                    const uint32_t o = staged<EPI_COLS * 2>(r + 8 * h, (8 * jj + cq) * 2);
                    st_shared_u32(buf + o, hw);
                    if (args.out_lo) {
                        const float2 lo = fma2(make_float2(__uint_as_float(hw << 16), __uint_as_float(hw & 0xffff0000u)), bcast2(-1.0f), g);   // g - hi, one rounding
                        st_shared_u32(buf + EPI_BUF_BYTES / 2 + o, cvt_bf16x2(lo.x, lo.y));
                    }
                } else {
                    st_shared_f32x2(buf + staged<EPI_COLS * 4>(r + 8 * h, (8 * jj + cq) * 4), f);
                    if (col + 1 >= (args.N & ~3)) {
                        store_tail(args, row0 + r + 8 * h, col, f.x);
                        store_tail(args, row0 + r + 8 * h, col + 1, f.y);
                    }
                }
            }
        }
        fence_proxy_async_smem();                                         // make the writes visible to the TMA unit
        named_bar_sync(1 + wg, 128);
        if (issuer && col0 < tma_cols(args)) {
            if (gelu) {
                tma_store_2d(&maps.out_hi, buf, col0, row0);
                if (args.out_lo) tma_store_2d(&maps.out_lo, buf + EPI_BUF_BYTES / 2, col0, row0);
            } else if (args.epilogue == PIPS_EPI_BIAS_RESID) {
                tma_reduce_add_2d(&maps.out_f32, buf, col0, row0);       // x + (acc + b): the bits of (acc + b) + x
            } else {
                tma_store_2d(&maps.out_f32, buf, col0, row0);
            }
            bulk_commit();
        }
        ++chunk;
    }
}

// The epilogue warps' work on one consumer warpgroup's 64 x BN accumulator, handed off at `buf` as BN / 32 chunks
// of 64 rows x 32 fp32 columns (EPI_BUF_BYTES each, 128-byte swizzle: the layout the fp32 store box reads).  Per chunk:
// add the bias in place and store / add-reduce the chunk, or for BIAS_GELU write GELU's (hi, lo) split over the chunk's
// fp32 values as a 64-byte-swizzled bf16 hi box and lo box and store those.  Run by EPI_THREADS threads; thread t takes
// the 16-byte units t + EPI_THREADS i of a chunk: rows t / 8 + EPI_ROWS i, columns 4 (t % 8) .. + 3, so its four bias
// values serve every row.  Each value meets the operations of the in-consumer epilogue in the same order: the same bits.
template <int BN>
__device__ __forceinline__ void epilogue_handoff(const GemmMaps& maps, const GemmArgs& args, uint32_t buf, int row0, int n0) {
    constexpr int EPI_ROWS = EPI_THREADS / 8;                             // rows per pass over the threads
    constexpr int PASSES = (64 + EPI_ROWS - 1) / EPI_ROWS;
    const int t = threadIdx.x - 32;
    const int u = t & 7;
    const bool issuer = t == 0;
    const bool gelu = args.epilogue == PIPS_EPI_BIAS_GELU;
#pragma unroll 1
    for (int c = 0; c < BN / EPI_COLS; ++c) {
        const int col0 = n0 + c * EPI_COLS;
        if (col0 >= args.N) break;
        const uint32_t chunk = buf + c * EPI_BUF_BYTES;
        const int col = col0 + 4 * u;
        const float2 b01 = make_float2(col < args.N ? __ldg(args.bias + col) : 0.f, col + 1 < args.N ? __ldg(args.bias + col + 1) : 0.f);
        const float2 b23 = make_float2(col + 2 < args.N ? __ldg(args.bias + col + 2) : 0.f, col + 3 < args.N ? __ldg(args.bias + col + 3) : 0.f);
        float4 v[PASSES];
#pragma unroll
        for (int i = 0; i < PASSES; ++i)
            if ((t >> 3) + EPI_ROWS * i < 64) v[i] = ld_shared_f32x4(chunk + staged<EPI_COLS * 4>((t >> 3) + EPI_ROWS * i, 16 * u));
        if (gelu) {
            named_bar_sync(1, EPI_THREADS);                              // the chunk is read: its bf16 boxes go over it
#pragma unroll
            for (int i = 0; i < PASSES; ++i) {
                if ((t >> 3) + EPI_ROWS * i >= 64) break;
                const float2 g01 = gelu_fast2_abs(add2(make_float2(v[i].x, v[i].y), b01));
                const float2 g23 = gelu_fast2_abs(add2(make_float2(v[i].z, v[i].w), b23));
                const uint32_t h01 = cvt_bf16x2(g01.x, g01.y), h23 = cvt_bf16x2(g23.x, g23.y);
                const uint32_t o = staged<EPI_COLS * 2>((t >> 3) + EPI_ROWS * i, 8 * u);
                st_shared_u32x2(chunk + o, h01, h23);
                if (args.out_lo) {
                    // g - hi, one rounding
                    const float2 l01 = fma2(make_float2(__uint_as_float(h01 << 16), __uint_as_float(h01 & 0xffff0000u)), bcast2(-1.0f), g01);
                    const float2 l23 = fma2(make_float2(__uint_as_float(h23 << 16), __uint_as_float(h23 & 0xffff0000u)), bcast2(-1.0f), g23);
                    st_shared_u32x2(chunk + EPI_BUF_BYTES / 2 + o, cvt_bf16x2(l01.x, l01.y), cvt_bf16x2(l23.x, l23.y));
                }
            }
        } else {
#pragma unroll
            for (int i = 0; i < PASSES; ++i) {
                if ((t >> 3) + EPI_ROWS * i >= 64) break;
                const float2 f01 = add2(make_float2(v[i].x, v[i].y), b01), f23 = add2(make_float2(v[i].z, v[i].w), b23);
                st_shared_f32x4(chunk + staged<EPI_COLS * 4>((t >> 3) + EPI_ROWS * i, 16 * u), make_float4(f01.x, f01.y, f23.x, f23.y));
                if (col + 3 >= (args.N & ~3)) {
                    const int row = row0 + (t >> 3) + EPI_ROWS * i;
                    store_tail(args, row, col, f01.x);
                    store_tail(args, row, col + 1, f01.y);
                    store_tail(args, row, col + 2, f23.x);
                    store_tail(args, row, col + 3, f23.y);
                }
            }
        }
        fence_proxy_async_smem();                                         // make the writes visible to the TMA unit
        named_bar_sync(1, EPI_THREADS);
        if (issuer && col0 < tma_cols(args)) {
            if (gelu) {
                tma_store_2d(&maps.out_hi, chunk, col0, row0);
                if (args.out_lo) tma_store_2d(&maps.out_lo, chunk + EPI_BUF_BYTES / 2, col0, row0);
            } else if (args.epilogue == PIPS_EPI_BIAS_RESID) {
                tma_reduce_add_2d(&maps.out_f32, chunk, col0, row0);     // x + (acc + b): the bits of (acc + b) + x
            } else {
                tma_store_2d(&maps.out_f32, chunk, col0, row0);
            }
            bulk_commit();
        }
    }
}

// Weight-gradient epilogue: the warpgroup's 64 x 128 fp32 partial sum of one split of M goes straight from registers to
// its slice of the output (rows n, columns k, row stride args.ldo); rows >= N and columns >= K are not stored.
__device__ __forceinline__ void epilogue_wgrad(const GemmArgs& args, const float (&acc)[64], float* out, int row0, int k0) {
    const int lane = threadIdx.x & 31;
    const int r = ((threadIdx.x >> 5) & 3) * 16 + (lane >> 2);
    const int cq = 2 * (lane & 3);
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        const int n = row0 + r + 8 * h;
        if (n >= args.N) continue;
        float* o = out + static_cast<size_t>(n) * args.ldo;
#pragma unroll
        for (int j = 0; j < 16; ++j) {
            const int k = k0 + 8 * j + cq;                                // K % 8 == 0: k < K covers k + 1
            if (k < args.K) *reinterpret_cast<float2*>(o + k) = make_float2(acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1]);
        }
    }
}

// WGRAD = false: C = epi(A . W^T + bias), K-major operands (above).
// WGRAD = true:  the weight gradient dW[N,K] = sum_m G[m,n] X[m,k] (maps a_* over G, w_* over X; both row-major with m as
// the row, so both are read MN-major).  A ring stage holds 32 rows of m: the 128 n of the tile as four {32 n, 32 m}
// boxes and the 128 k as four more, each box one stack of MN-major SW64 atoms.  A tile is (n block, k block, split of M);
// each split's partial sum goes to its own slice of args.out_f32 (N*K floats apart) and is summed in a fixed order later.
template <int TERMS, int BN, int CLUSTER, bool WGRAD = false, bool AUX = false>
__device__ __forceinline__ void gemm_tc_body(const GemmMaps& maps, const GemmArgs& args) {
    using Cfg = GemmCfg<TERMS, BN, !WGRAD && !AUX>;
    constexpr bool HANDOFF = Cfg::kHandoff;
    constexpr int kStages = Cfg::kStages;
    constexpr uint32_t W_TILE_BYTES = Cfg::kWTileBytes;
    constexpr uint32_t BOX_BYTES = 32 * KB * 2;                    // WGRAD: one {32, 32} box, 2 KB
    static_assert(CLUSTER == 1 || BN == 256, "cluster tiles are 256 columns wide");
    static_assert(!WGRAD || (BN == 128 && CLUSTER == 1 && TERMS == 3), "the weight-gradient variant is bf16x3, 128 x 128");
    // the 128-byte-swizzled epilogue buffers need 1024-byte alignment (the 64-byte-swizzled ring needs 512)
    uint8_t* smem = aligned_smem();
    uint8_t* staging = smem + kStages * Cfg::kStageBytes;
    Ring ring(smem, Cfg::kStageBytes, kStages, reinterpret_cast<uint64_t*>(staging + Cfg::kEpiBytes), kStages);
    // HANDOFF: the consumer warpgroups take turns in the handoff buffer, 0 then 1 on every tile.  ho_full: a consumer has
    // filled it (128 arrivals).  ho_empty + 8 wg: the epilogue warps' store issuer has drained the other warpgroup's
    // turn before wg's, and its stores have read the buffer.  A barrier per warpgroup, so that a warpgroup that runs a
    // whole tile ahead of the epilogue cannot take a phase meant for the other one.
    const uint32_t ho_full = smem_u32(staging + Cfg::kEpiBytes) + 16 * kStages, ho_empty = ho_full + 8;

    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;
    const uint32_t rank = CLUSTER == 2 ? cluster_ctarank() : 0;
    const int worker = blockIdx.x / CLUSTER, num_workers = gridDim.x / CLUSTER;     // a CTA, or a cluster of two
    pdl_trigger();

    constexpr int TM = BM * CLUSTER;
    // C = A . W^T: tiles (m block, n block), all of K.  WGRAD: tiles (n block, k block, split of M), the split's K-blocks.
    const int tiles_n = WGRAD ? (args.K + BN - 1) / BN : (args.N + BN - 1) / BN;
    const int total_kb = WGRAD ? (args.M + KB - 1) / KB : args.K / KB;
    const int splits = WGRAD ? (total_kb + args.kb_per_split - 1) / args.kb_per_split : 1;
    // tile t -> first output row (m, or n), first output column (n, or k), K-block range
    auto tile_coords = [&](int t, int& row0, int& col0, int& kb0, int& kb1) {
        if constexpr (WGRAD) {
            const int s = t % splits;
            t /= splits;
            kb0 = s * args.kb_per_split;
            kb1 = min(total_kb, kb0 + args.kb_per_split);
        } else {
            kb0 = 0;
            kb1 = total_kb;
        }
        row0 = (t / tiles_n) * TM + static_cast<int>(rank) * BM;
        col0 = (t % tiles_n) * BN;
    };

    if (warp == 0 && lane == 0) {
        tma_prefetch_desc(&maps.a_hi);
        tma_prefetch_desc(&maps.w_hi);
        if (TERMS == 3) {
            tma_prefetch_desc(&maps.a_lo);
            tma_prefetch_desc(&maps.w_lo);
        }
        if (WGRAD) {
        } else if (AUX ? bf16_epilogue(args.epilogue) : args.epilogue == PIPS_EPI_BIAS_GELU) {
            tma_prefetch_desc(&maps.out_hi);
            if (args.out_lo) tma_prefetch_desc(&maps.out_lo);
        } else {
            tma_prefetch_desc(&maps.out_f32);
        }
    }
    if (warp == 1 && lane == 0) {
        if constexpr (HANDOFF) {
            mbar_init(ho_full, 128);
            mbar_init(ho_empty, 1);
            mbar_init(ho_empty + 8, 1);
        }
        ring.init(2 * CLUSTER);                             // one arrival per consumer warpgroup that reads the slot's W
    }
    if (CLUSTER == 2) cluster_sync_all();                   // the peer's barriers exist before anything is sent to them
    else __syncthreads();
    pdl_wait();                                             // operands and the residual stream come from the previous kernel

    // Register budget per warpgroup: the producer warpgroup needs few, the consumers hold the accumulator.  The HANDOFF
    // kernels keep the launch's 168 per thread everywhere: their producer warpgroup also runs the epilogue warps, and
    // the consumers' 128-float accumulator with the mainloop's state fits in 168.
    if (warp < 4) {
        if constexpr (!HANDOFF) asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");
        if (warp == 0 && lane == 0) {
            // ------------------------------------------------------------ TMA producer
            for (int t = worker; t < args.num_tiles; t += num_workers) {
                int m0, n0, kb0, kb1;
                tile_coords(t, m0, n0, kb0, kb1);
                for (int kb = kb0; kb < kb1; ++kb) {
                    ring.produce([&](uint32_t base, uint32_t fb) {
                        const int k0 = kb * KB;
                        if constexpr (WGRAD) {             // m0: first n of the tile, n0: first k, k0: first m
#pragma unroll
                            for (int i = 0; i < 4; ++i) {
                                tma_load_2d(base + i * BOX_BYTES, &maps.a_hi, fb, m0 + 32 * i, k0);
                                tma_load_2d(base + A_TILE_BYTES + i * BOX_BYTES, &maps.w_hi, fb, n0 + 32 * i, k0);
                                tma_load_2d(base + A_TILE_BYTES + W_TILE_BYTES + i * BOX_BYTES, &maps.a_lo, fb, m0 + 32 * i, k0);
                                tma_load_2d(base + 2 * A_TILE_BYTES + W_TILE_BYTES + i * BOX_BYTES, &maps.w_lo, fb, n0 + 32 * i, k0);
                            }
                        } else {
                            tma_load_2d(base, &maps.a_hi, fb, k0, m0);
                            if (TERMS == 3) tma_load_2d(base + A_TILE_BYTES + W_TILE_BYTES, &maps.a_lo, fb, k0, m0);
                            if (CLUSTER == 2) {
                                // this CTA's half of the W tile (box = 128 rows), into both CTAs
                                const uint32_t half = rank * (W_TILE_BYTES / 2);
                                tma_load_2d_multicast(base + A_TILE_BYTES + half, &maps.w_hi, fb, k0, n0 + static_cast<int>(rank) * (BN / 2), 3);
                                if (TERMS == 3)
                                    tma_load_2d_multicast(base + 2 * A_TILE_BYTES + W_TILE_BYTES + half, &maps.w_lo, fb, k0,
                                                          n0 + static_cast<int>(rank) * (BN / 2), 3);
                            } else {
                                tma_load_2d(base + A_TILE_BYTES, &maps.w_hi, fb, k0, n0);
                                if (TERMS == 3) tma_load_2d(base + 2 * A_TILE_BYTES + W_TILE_BYTES, &maps.w_lo, fb, k0, n0);
                            }
                        }
                    });
                }
            }
        } else if (HANDOFF && warp > 0) {
            // -------------------------------------------------------- epilogue warps: the consumers' halves in turn
            const bool issuer = threadIdx.x == 32;
            uint32_t turn = 0;                              // turns taken; turn 2 i + wg: warpgroup wg on tile i
            for (int t = worker; t < args.num_tiles; t += num_workers) {
                int m0, n0, kb0, kb1;
                tile_coords(t, m0, n0, kb0, kb1);
                for (int wg = 0; wg < 2; ++wg, ++turn) {
                    mbar_wait(ho_full, turn & 1);
                    if (m0 + wg * 64 < args.M)              // else the whole half is past M: nothing to store
                        epilogue_handoff<BN>(maps, args, smem_u32(staging), m0 + wg * 64, n0);
                    if (issuer) {
                        bulk_wait_read<0>();                // the stores have read the buffer: the other warpgroup may fill it
                        mbar_arrive(ho_empty + 8 * (wg ^ 1));
                    }
                }
            }
            if (issuer) bulk_wait<0>();                     // the last stores have finished writing
        }
    } else {
        if constexpr (!HANDOFF) asm volatile("setmaxnreg.inc.sync.aligned.u32 232;");
        // ------------------------------------------------------------ consumers: MMA (+ epilogue), 64 rows each
        const int wg = (warp - 4) >> 2;
        const bool releaser = (threadIdx.x & 127) == 0;
        const uint32_t my_staging = smem_u32(staging) + wg * 2 * EPI_BUF_BYTES;   // in-consumer epilogue
        uint32_t chunk = 0;
        uint32_t turn = wg;                                  // HANDOFF: this warpgroup's next turn in the handoff buffer
        float acc[BN / 2];
        auto release = [&](int slot) {
            if (releaser) {
                ring.release(slot);
                if (CLUSTER == 2) mbar_arrive_cluster(ring.empty(slot), rank ^ 1);
            }
        };
        for (int t = worker; t < args.num_tiles; t += num_workers) {
            int m0, n0, kb0, kb1;
            tile_coords(t, m0, n0, kb0, kb1);
            int prev = -1;                                   // ring slot whose MMAs are still in flight
            for (int kb = kb0; kb < kb1; ++kb) {
                const uint32_t base = ring.wait();
                if constexpr (WGRAD) {
                    wgmma_fence();
                    // the warpgroup's 64 n are the boxes 2wg, 2wg + 1; a K=16 step is 16 rows of m = 1 KB into every box
                    const uint32_t a_hi = base + wg * 2 * BOX_BYTES, w_hi = base + A_TILE_BYTES;
                    const uint32_t a_lo = a_hi + A_TILE_BYTES + W_TILE_BYTES, w_lo = w_hi + A_TILE_BYTES + W_TILE_BYTES;
                    auto mma = [&](uint64_t a, uint64_t w, uint32_t accumulate) {
                        wgmma_n128_tt(*reinterpret_cast<float(*)[64]>(&acc[0]), a, w, accumulate);
                    };
#pragma unroll
                    for (int k = 0; k < KB / MMA_K; ++k) {
                        mma_bf16x3(mma, wgmma_desc_sw64_mn(a_hi + k * 1024, BOX_BYTES),
                                   wgmma_desc_sw64_mn(a_lo + k * 1024, BOX_BYTES), wgmma_desc_sw64_mn(w_hi + k * 1024, BOX_BYTES),
                                   wgmma_desc_sw64_mn(w_lo + k * 1024, BOX_BYTES), (kb != kb0) | k);
                    }
                } else {
                    const uint64_t a_hi = wgmma_desc_sw64(base + wg * (A_TILE_BYTES / 2));
                    const uint64_t w_hi = wgmma_desc_sw64(base + A_TILE_BYTES);
                    const uint64_t a_lo = wgmma_desc_sw64(base + A_TILE_BYTES + W_TILE_BYTES + wg * (A_TILE_BYTES / 2));
                    const uint64_t w_lo = wgmma_desc_sw64(base + 2 * A_TILE_BYTES + W_TILE_BYTES);
                    wgmma_fence();
#pragma unroll
                    for (int k = 0; k < KB / MMA_K; ++k) {
                        const uint64_t adv = static_cast<uint64_t>((k * MMA_K * 2) >> 4);   // 32 B per K=16 step
                        auto mma = [&](uint64_t a, uint64_t w, uint32_t accumulate) {
                            gemm_mma<BN>(acc, a + adv, w + adv, accumulate);
                        };
                        if (TERMS == 3) mma_bf16x3(mma, a_hi, a_lo, w_hi, w_lo, (kb | k) != 0);
                        else mma(a_hi, w_hi, (kb | k) != 0);
                    }
                }
                wgmma_commit();
                if (prev >= 0) {
                    wgmma_wait<1>();                         // the previous slot's MMAs have retired: slot reusable
                    release(prev);
                }
                prev = static_cast<int>(ring.stage);
                ring.advance();
            }
            wgmma_wait<0>();
            wgmma_acc_ready(acc);
            release(prev);
            if constexpr (WGRAD) {
                const int split = t % splits;
                float* out = args.out_f32 + static_cast<size_t>(split) * args.N * args.ldo;
                epilogue_wgrad(args, *reinterpret_cast<const float(*)[64]>(&acc[0]), out, m0 + wg * 64, n0);
            } else if constexpr (!HANDOFF) {
                epilogue_tma<BN, AUX>(maps, args, acc, m0 + wg * 64, n0, my_staging, chunk, wg);
            } else {
                // hand the accumulator to the epilogue warps as BN / 32 fp32 chunks and go on to the next tile
                // turn 2 i + wg waits for the (i + wg)-th drain on ho_empty + 8 wg (warpgroup 0's first turn: none)
                mbar_wait(ho_empty + 8 * wg, ((turn >> 1) + wg + 1) & 1);
                const uint32_t buf = smem_u32(staging);
                const int r = ((threadIdx.x >> 5) & 3) * 16 + (lane >> 2);   // fragment rows r, r + 8 of the 64
                const int cq = 2 * (lane & 3);                                // fragment columns cq, cq + 1 of each 8
#pragma unroll
                for (int j = 0; j < BN / 8; ++j) {
#pragma unroll
                    for (int h = 0; h < 2; ++h)
                        st_shared_f32x2(buf + (j / 4) * EPI_BUF_BYTES + staged<EPI_COLS * 4>(r + 8 * h, (8 * (j % 4) + cq) * 4),
                                        make_float2(acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1]));
                }
                mbar_arrive(ho_full);
                turn += 2;
            }
        }
        if (!HANDOFF && releaser) bulk_wait<0>();            // the last stores have finished reading shared memory and writing
    }
    if (CLUSTER == 2) cluster_sync_all();                   // nobody leaves while the peer may still signal or write to us
}

template <int TERMS, int BN>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
gemm_tc_kernel(const __grid_constant__ GemmMaps maps, const GemmArgs args) {
    gemm_tc_body<TERMS, BN, 1>(maps, args);
}

template <int TERMS>
__global__ void __cluster_dims__(2, 1, 1) __launch_bounds__(GEMM_THREADS, 1)
gemm_tc_pair_kernel(const __grid_constant__ GemmMaps maps, const GemmArgs args) {
    gemm_tc_body<TERMS, 256, 2>(maps, args);
}

__global__ void __launch_bounds__(GEMM_THREADS, 1)
gemm_tc_aux_kernel(const __grid_constant__ GemmMaps maps, const GemmArgs args) {
    gemm_tc_body<3, 128, 1, false, true>(maps, args);
}

__global__ void __launch_bounds__(GEMM_THREADS, 1)
wgrad_kernel(const __grid_constant__ GemmMaps maps, const GemmArgs args) {
    gemm_tc_body<3, 128, 1, true>(maps, args);
}

// Rows of M per split of the weight-gradient GEMM.  The layer shapes give 20..64 output tiles of 128 x 128, too few for the
// SMs; splitting M fills them.  A constant, so the partial sums -- and the bits -- depend on the shape only.
constexpr int WG_SPLIT_ROWS = 2048;

// ---------------------------------------------------------------------------------- host side

// the (hi, lo) operand maps; map_lo = nullptr: the hi map only
static bool make_operand_maps(CUtensorMap* map_hi, CUtensorMap* map_lo, const void* hi, const void* lo, int rows, int K,
                              int ld_elems, int box_rows) {
    // global tensor (innermost first): {K, rows}, row stride ld_elems*2 bytes; box {32, box_rows}, 64B swizzle
    cuuint64_t gdim[2] = {static_cast<cuuint64_t>(K), static_cast<cuuint64_t>(rows)};
    cuuint64_t gstride[1] = {static_cast<cuuint64_t>(ld_elems) * 2};
    cuuint32_t box[2] = {static_cast<cuuint32_t>(KB), static_cast<cuuint32_t>(box_rows)};
    cuuint32_t estr[2] = {1, 1};
    if (!map_lo)
        return encode_tiled(map_hi, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(hi), gdim, gstride, box, estr,
                            CU_TENSOR_MAP_SWIZZLE_64B);
    return encode_tiled_pair(map_hi, map_lo, hi, lo, 2, gdim, gstride, box, estr, CU_TENSOR_MAP_SWIZZLE_64B);
}

// Output tensor {tma_cols, M} with row stride `ld` elements; box {EPI_COLS, 64} (one warpgroup's chunk), swizzled like
// the staging buffer.  The bounds are the problem's, so TMA drops the rows and columns of a tile beyond M and tma_cols.
static bool make_output_map(CUtensorMap* map, void* ptr, const GemmArgs& args, int ld, bool f32) {
    const int cols = tma_cols(args) > 0 ? tma_cols(args) : args.N;        // N < 4: the map is never stored through
    cuuint64_t gdim[2] = {static_cast<cuuint64_t>(cols), static_cast<cuuint64_t>(args.M)};
    cuuint64_t gstride[1] = {static_cast<cuuint64_t>(ld) * (f32 ? 4 : 2)};
    cuuint32_t box[2] = {static_cast<cuuint32_t>(EPI_COLS), 64};
    cuuint32_t estr[2] = {1, 1};
    return encode_tiled(map, f32 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, ptr, gdim, gstride, box,
                        estr, f32 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_64B);
}

// every map of the problem (bf16: the lo maps are copies of the hi ones); W boxes are `w_box_rows` rows (the tile width, or
// its half in the pair kernel)
static const char* make_maps(GemmMaps* m, bool x3, const void* a_hi, const void* a_lo, int lda, int a_rows, const void* w_hi,
                             const void* w_lo, int ldw, int w_rows, int w_box_rows, const GemmArgs& args) {
    *m = GemmMaps{};
    if (!make_operand_maps(&m->a_hi, x3 ? &m->a_lo : nullptr, a_hi, a_lo, a_rows, args.K, lda, BM)) return "tensor map (A) failed";
    if (!make_operand_maps(&m->w_hi, x3 ? &m->w_lo : nullptr, w_hi, w_lo, w_rows, args.K, ldw, w_box_rows))
        return "tensor map (W) failed";
    if (!x3) {
        m->a_lo = m->a_hi;
        m->w_lo = m->w_hi;
    }
    if (bf16_epilogue(args.epilogue)) {
        if (!make_output_map(&m->out_hi, args.out_hi, args, args.ldh, false)) return "tensor map (out hi) failed";
        if (args.out_lo && !make_output_map(&m->out_lo, args.out_lo, args, args.ldh, false)) return "tensor map (out lo) failed";
    } else if (!make_output_map(&m->out_f32, args.out_f32, args, args.ldo, true)) {
        return "tensor map (out) failed: out_f32 must be 16-byte aligned";
    }
    return nullptr;
}

// 0: automatic, 1: pair kernel, 64/128/256: single-CTA kernel with that tile width
static int forced_tile() {
    const char* e = getenv("PIPS_B200_GEMM_TILE");
    if (!e || !e[0]) return 0;
    if (e[0] == 'p') return 1;
    const int v = atoi(e);
    return (v == 64 || v == 128 || v == 256) ? v : 0;
}

int launch_single(int bn, bool x3, const void* a_hi, const void* a_lo, int lda, int a_rows, const void* w_hi, const void* w_lo,
                  int ldw, int w_rows, const GemmArgs& args, cudaStream_t st);

int launch_pair(bool x3, const void* a_hi, const void* a_lo, int lda, int a_rows, const void* w_hi, const void* w_lo, int ldw,
                int w_rows, const GemmArgs& args, cudaStream_t st);

int launch_aux(const void* a_hi, const void* a_lo, int lda, int a_rows, const void* w_hi, const void* w_lo, int ldw, int w_rows,
               const GemmArgs& args, cudaStream_t st);

static bool use_pair_kernel() {
    static int v = -1;
    if (v < 0) {
        const char* e = getenv("PIPS_B200_GEMM_PAIR");
        v = (e && e[0] == '0') ? 0 : 1;
    }
    return v == 1;
}

}  // namespace pips

using namespace pips;

extern "C" int pips_gemm_tc(const void* a_hi, const void* a_lo, int lda, int a_rows,
                            const void* w_hi, const void* w_lo, int ldw, int w_rows,
                            int M, int N, int K, const float* bias, int epilogue,
                            float* out_f32, int ldo, void* out_hi, void* out_lo, int ldh,
                            void* stream) {
    return pips_gemm_tc_aux(a_hi, a_lo, lda, a_rows, w_hi, w_lo, ldw, w_rows, M, N, K, bias, epilogue, out_f32, ldo, out_hi,
                            out_lo, ldh, nullptr, 0, stream);
}

extern "C" int pips_gemm_tc_aux(const void* a_hi, const void* a_lo, int lda, int a_rows,
                                const void* w_hi, const void* w_lo, int ldw, int w_rows,
                                int M, int N, int K, const float* bias, int epilogue,
                                float* out_f32, int ldo, void* out_hi, void* out_lo, int ldh,
                                float* aux, int ld_aux, void* stream) {
    if (K % BK != 0 || K <= 0) return fail("pips_gemm_tc: K must be a positive multiple of 64");
    if (M <= 0 || N <= 0) return fail("pips_gemm_tc: empty problem");
    if (a_rows < M || w_rows < N) return fail("pips_gemm_tc: operand allocations smaller than the problem");
    if ((lda % 8) || (ldw % 8)) return fail("pips_gemm_tc: leading dimensions must be multiples of 8 elements (16 B)");
    if (!bias) return fail("pips_gemm_tc: bias is required");
    const bool x3 = a_lo != nullptr && w_lo != nullptr;
    if ((a_lo != nullptr) != (w_lo != nullptr)) return fail("pips_gemm_tc: need both or neither lo operands");
    if (bf16_epilogue(epilogue)) {
        if (!out_hi || (ldh % 8)) return fail("pips_gemm_tc: GELU epilogue needs out_hi with ldh % 8 == 0");
        if (epilogue != PIPS_EPI_BIAS_GELU) {
            if (!aux || (reinterpret_cast<uintptr_t>(aux) & 7) || ld_aux < N || (ld_aux % 2) || (N % 8))
                return fail("pips_gemm_tc: the pre-activation epilogues need an 8-byte aligned aux with ld_aux >= N, "
                            "ld_aux % 2 == 0, and N % 8 == 0");
            if (!x3) return fail("pips_gemm_tc: the pre-activation epilogues are bf16x3 only (a_lo and w_lo required)");
        }
    } else if (epilogue == PIPS_EPI_BIAS || epilogue == PIPS_EPI_BIAS_RESID) {
        if (!out_f32 || (ldo % 4)) return fail("pips_gemm_tc: fp32 epilogue needs out_f32 with ldo % 4 == 0");
    } else {
        return fail("pips_gemm_tc: unknown epilogue");
    }
    GemmArgs args = {};
    args.M = M; args.N = N; args.K = K; args.bias = bias; args.epilogue = epilogue;
    args.out_f32 = out_f32; args.ldo = ldo;
    args.out_hi = static_cast<__nv_bfloat16*>(out_hi); args.out_lo = static_cast<__nv_bfloat16*>(out_lo); args.ldh = ldh;
    args.aux = aux; args.ld_aux = ld_aux;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    // Tile shape.  Every variant accumulates each output element over K in the same order (same MMA K-steps, same
    // hi/lo term order), so the choice changes the schedule, not the bits (tests/test_kernels_gpu.py).
    //   pair  256x256 per cluster of two CTAs (W multicast): least operand traffic; needs enough pair tiles to fill the GPU
    //   128 x {256,128,64} single CTA: when 256-wide tiles would leave most SMs idle (few particles)
    if (epilogue == PIPS_EPI_BIAS_GELU_PRE || epilogue == PIPS_EPI_GELU_GRAD)
        return launch_aux(a_hi, a_lo, lda, a_rows, w_hi, w_lo, ldw, w_rows, args, st);
    const int force = forced_tile();                  // PIPS_B200_GEMM_TILE = pair | 256 | 128 | 64 (tests, profiling)
    const bool pair_ok = use_pair_kernel() && M > 128 && (a_rows % 256) == 0 && (w_rows % 256) == 0;
    const int pair_tiles = ((M + 255) / 256) * ((N + 255) / 256);
    const int sms = sm_count();
    int bn = 256;
    bool pair = pair_ok && pair_tiles * 2 >= (sms * 3) / 4;          // at least 3/4 of the SMs get a tile
    if (!pair) {
        const int tm = (M + BM - 1) / BM;
        while (bn > 64 && tm * ((N + bn - 1) / bn) < (sms * 3) / 4) bn >>= 1;
    }
    if (force == 1) pair = pair_ok;
    else if (force > 1) { pair = false; bn = force; }
    if ((w_rows % bn) != 0) { bn = 256; pair = pair && pair_ok; }   // TMA boxes must stay inside the weight allocation
    if (pair)
        return launch_pair(x3, a_hi, a_lo, lda, a_rows, w_hi, w_lo, ldw, w_rows, args, st);
    return launch_single(bn, x3, a_hi, a_lo, lda, a_rows, w_hi, w_lo, ldw, w_rows, args, st);
}

namespace pips {
int colsum_launch(const float* g, const void* g_hi, const void* g_lo, size_t ld, int M, int N, float* scratch, float* out,
                  cudaStream_t st);   // mixer_grad.cu
}  // namespace pips

extern "C" size_t pips_wgrad_scratch_floats(int M, int N, int K) {
    if (M <= 0 || N <= 0 || K <= 0) return 0;
    const size_t splits = (static_cast<size_t>(M) + WG_SPLIT_ROWS - 1) / WG_SPLIT_ROWS;
    return splits > 1 ? splits * N * K : 0;
}

extern "C" int pips_wgrad(const void* g_hi, const void* g_lo, int ldg, const void* x_hi, const void* x_lo, int ldx, int M, int N,
                          int K, float* scratch, float* dw, void* stream) {
    if (!g_hi || !g_lo || !x_hi || !x_lo || !dw) return fail("pips_wgrad: null pointer");
    if (M <= 0 || N <= 0 || K <= 0) return fail("pips_wgrad: empty problem");
    if ((N % 8) || (K % 8) || ldg < N || ldx < K || (ldg % 8) || (ldx % 8))
        return fail("pips_wgrad: N and K must be multiples of 8, ldg >= N and ldx >= K multiples of 8");
    if ((reinterpret_cast<uintptr_t>(g_hi) | reinterpret_cast<uintptr_t>(g_lo) | reinterpret_cast<uintptr_t>(x_hi)
         | reinterpret_cast<uintptr_t>(x_lo) | reinterpret_cast<uintptr_t>(dw) | reinterpret_cast<uintptr_t>(scratch)) & 15)
        return fail("pips_wgrad: operands, scratch and dw must be 16-byte aligned");
    const int splits = (M + WG_SPLIT_ROWS - 1) / WG_SPLIT_ROWS;
    if (static_cast<long long>(N) * K > 0x7fffffffLL || splits > 256) return fail("pips_wgrad: problem too large");
    if (splits > 1 && !scratch) return fail("pips_wgrad: scratch of pips_wgrad_scratch_floats(M, N, K) floats is required");
    GemmMaps maps = {};
    if (!make_operand_maps(&maps.a_hi, &maps.a_lo, g_hi, g_lo, M, N, ldg, 32) ||
        !make_operand_maps(&maps.w_hi, &maps.w_lo, x_hi, x_lo, M, K, ldx, 32))
        return fail("pips_wgrad: tensor map failed");
    GemmArgs a = {};
    a.M = M; a.N = N; a.K = K; a.epilogue = PIPS_EPI_BIAS;
    a.out_f32 = splits > 1 ? scratch : dw; a.ldo = K;
    a.kb_per_split = WG_SPLIT_ROWS / KB;
    a.num_tiles = ((N + BM - 1) / BM) * ((K + 127) / 128) * splits;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const int grid = a.num_tiles < sm_count() ? a.num_tiles : sm_count();
    if (const int err = launch_kernel<wgrad_kernel>("pips_wgrad", true, grid, GEMM_THREADS, GemmCfg<3, 128>::kSmemBytes, st, maps, a))
        return err;
    if (splits == 1) return 0;
    // the splits' partial sums, in split order
    const size_t nk = static_cast<size_t>(N) * K;
    return colsum_launch(scratch, nullptr, nullptr, nk, splits, static_cast<int>(nk), nullptr, dw, st);
}

namespace pips {

template <int TERMS, int BN>
static int launch_variant(const GemmMaps& maps, const GemmArgs& args, cudaStream_t st) {
    GemmArgs a = args;
    a.num_tiles = ((args.M + BM - 1) / BM) * ((args.N + BN - 1) / BN);
    const int grid = a.num_tiles < sm_count() ? a.num_tiles : sm_count();
    using Cfg = GemmCfg<TERMS, BN, true>;
    return launch_kernel<gemm_tc_kernel<TERMS, BN>>("pips_gemm_tc", true, grid, GEMM_THREADS, Cfg::kSmemBytes, st, maps, a);
}

template <int TERMS>
static int launch_pair_variant(const GemmMaps& maps, const GemmArgs& args, cudaStream_t st) {
    GemmArgs a = args;
    a.num_tiles = ((args.M + 255) / 256) * ((args.N + 255) / 256);
    const int max_pairs = sm_count() / 2;
    const int pairs = a.num_tiles < max_pairs ? a.num_tiles : max_pairs;
    using Cfg = GemmCfg<TERMS, 256, true>;
    return launch_kernel<gemm_tc_pair_kernel<TERMS>>("pips_gemm_tc (pair)", true, 2 * pairs, GEMM_THREADS, Cfg::kSmemBytes, st,
                                                     maps, a);
}

int launch_pair(bool x3, const void* a_hi, const void* a_lo, int lda, int a_rows, const void* w_hi, const void* w_lo, int ldw,
                int w_rows, const GemmArgs& args, cudaStream_t st) {
    GemmMaps maps;                                           // every operand box is 128 rows: a CTA's rows of A, its half of the W tile
    if (const char* err = make_maps(&maps, x3, a_hi, a_lo, lda, a_rows, w_hi, w_lo, ldw, w_rows, 128, args)) {
        return fail((std::string("pips_gemm_tc (pair): ") + err).c_str());
    }
    return x3 ? launch_pair_variant<3>(maps, args, st) : launch_pair_variant<1>(maps, args, st);
}

// the pre-activation epilogues: bf16x3, 128 x 128 tiles (the FC1 / FC2 backward shapes have thousands of them)
int launch_aux(const void* a_hi, const void* a_lo, int lda, int a_rows, const void* w_hi, const void* w_lo, int ldw, int w_rows,
               const GemmArgs& args, cudaStream_t st) {
    GemmMaps maps;
    if (const char* err = make_maps(&maps, true, a_hi, a_lo, lda, a_rows, w_hi, w_lo, ldw, w_rows, 128, args)) {
        return fail((std::string("pips_gemm_tc: ") + err).c_str());
    }
    GemmArgs a = args;
    a.num_tiles = ((args.M + BM - 1) / BM) * ((args.N + 127) / 128);
    const int grid = a.num_tiles < sm_count() ? a.num_tiles : sm_count();
    return launch_kernel<gemm_tc_aux_kernel>("pips_gemm_tc (aux)", true, grid, GEMM_THREADS, GemmCfg<3, 128>::kSmemBytes, st, maps, a);
}

int launch_single(int bn, bool x3, const void* a_hi, const void* a_lo, int lda, int a_rows, const void* w_hi, const void* w_lo,
                  int ldw, int w_rows, const GemmArgs& args, cudaStream_t st) {
    GemmMaps maps;
    if (const char* err = make_maps(&maps, x3, a_hi, a_lo, lda, a_rows, w_hi, w_lo, ldw, w_rows, bn, args)) {
        return fail((std::string("pips_gemm_tc: ") + err).c_str());
    }
    if (x3) return bn == 256 ? launch_variant<3, 256>(maps, args, st)
                 : bn == 128 ? launch_variant<3, 128>(maps, args, st)
                             : launch_variant<3, 64>(maps, args, st);
    return bn == 256 ? launch_variant<1, 256>(maps, args, st)
         : bn == 128 ? launch_variant<1, 128>(maps, args, st)
                     : launch_variant<1, 64>(maps, args, st);
}

}  // namespace pips
