// 2-D convolution of the feature encoder as an implicit GEMM on the Hopper tensor cores (wgmma).
//
//   out[n, oy, ox, co] = sum_{r,s,ci} in[n, oy*st + r - pad, ox*st + s - pad, ci] * w[co, r, s, ci]   (+ bias[co])
//
// for the 3x3 / 1x1, stride 1 / 2 convolutions of BasicEncoder's residual stages and head
// (nets/pips.py:135-136, :170, :221-223).  Activations are channels-last bf16 (hi, lo) pairs (v ~= hi + lo)
// written by pips_inorm_apply / pips_resize_pair, weights are packed (Cout_pad, taps*Cp) bf16 (hi, lo), and
// every product is evaluated as hi*hi + lo*hi + hi*lo with fp32 accumulation -- the same bf16x3
// scheme as the mixer GEMMs (gemm_tc.cu), whose pipeline this kernel reuses (TMA producer warp, two consumer
// warpgroups of 64 pixels each):
//   GEMM-M  = output pixels, one CTA = TH rows x TW columns = 128 pixels; CTAs 2p and 2p+1 ("ranks" of pair p)
//             take two adjacent tiles, the unit of the statistics layout below
//   GEMM-N  = output channels (64 / 128 / 256)
//   GEMM-K  = taps x input channels; one K-chunk = 64 channels of one filter tap
// The A tile of a K-chunk is ONE 4-D TMA box {64 ch, TW px, TH rows, 1 image} of the input at the tap's
// offset (element strides = conv stride; out-of-bounds = zero padding), so no im2col buffer exists anywhere.
#include "gemm_common.cuh"

namespace pips {

constexpr int C_THREADS = 384;
constexpr uint32_t C_A_BYTES = 128 * BK * 2;          // 128 pixels x 64 channels bf16
constexpr int C_MAX_STAGES = 8;
constexpr uint32_t C_RING_BYTES = 200 * 1024;         // smem ring: stage = A_hi | A_lo | W_hi | W_lo, 2*(16 KB + BN*128 B)
constexpr uint32_t C_COMB_BYTES = 8 * 8 * 64 * 4;      // statistics exchange: 8 consumer warps x 256 columns x (mean, M2)
constexpr uint32_t C_SMEM_BYTES = C_RING_BYTES + C_COMB_BYTES + 1024 + 256;   // + alignment, barriers and 8 warp counts

struct ConvArgs {
    int N, Ho, Wo, Cout;        // output (NHWC fp32, row stride Cout)
    int Cp;                     // padded input channels per tap (multiple of 64)
    int R, S, sy, sx, py, px;   // filter taps, conv stride (rows, cols), zero padding (rows, cols)
    int TW, TH;                 // pixel tile: TW * TH == 128
    int tiles_x, tiles_y;       // tiles per image
    int BN;                     // GEMM-N tile == padded Cout: 64, 128 or 256
    int stages;                 // ring depth: 3 (BN = 256) .. 8 (BN = 64)
    const float* bias;          // [Cout] or null
    float* out;
    // Work items: the tiles of ONE image in groups of G consecutive pair tiles (pt_img pair tiles per image, groups_img
    // groups).  A group is the unit of the InstanceNorm partial statistics (nets/pips.py:154-157): with `partial` set, the
    // epilogue accumulates (mean, M2, count) per output channel over the group's valid pixels and every CTA writes one
    // row partial[(img * groups_img + g) * 2 + rank][3][Cout] -- a layout fixed by the image geometry alone (never by the
    // batch), merged in fp64 by pips_inorm_finalize.
    int G, groups_img, pt_img;
    float* partial;             // optional
};

template <int BN>
__global__ void __launch_bounds__(C_THREADS, 1)
conv_tc_kernel(const __grid_constant__ CUtensorMap map_a_hi, const __grid_constant__ CUtensorMap map_a_lo,
               const __grid_constant__ CUtensorMap map_w_hi, const __grid_constant__ CUtensorMap map_w_lo, const ConvArgs a) {
    pdl_trigger();
    uint8_t* smem = aligned_smem();
    float* comb = reinterpret_cast<float*>(smem + C_RING_BYTES);
    uint64_t* bars = reinterpret_cast<uint64_t*>(smem + C_RING_BYTES + C_COMB_BYTES);
    float* counts = reinterpret_cast<float*>(bars + 2 * C_MAX_STAGES);      // valid pixels per consumer warp and item

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int rank = blockIdx.x & 1;
    const int pair = blockIdx.x >> 1, num_pairs = gridDim.x >> 1;

    const int tiles_img = a.tiles_x * a.tiles_y;
    const int num_items = a.N * a.groups_img;
    const int chunks = a.Cp / BK;
    const int num_kb = a.R * a.S * chunks;
    constexpr uint32_t W_BYTES = BN * BK * 2;
    constexpr uint32_t C_STAGE_BYTES = 2 * (C_A_BYTES + W_BYTES);             // hi + lo; multiple of 1 KB
    constexpr uint32_t off_w_hi = 2 * C_A_BYTES, off_w_lo = 2 * C_A_BYTES + W_BYTES;
    Ring ring(smem, C_STAGE_BYTES, a.stages, bars, C_MAX_STAGES);

    if (warp == 0 && lane == 0) {
        tma_prefetch_desc(&map_a_hi); tma_prefetch_desc(&map_a_lo);
        tma_prefetch_desc(&map_w_hi); tma_prefetch_desc(&map_w_lo);
    }
    if (warp == 1 && lane == 0) ring.init(2);
    __syncthreads();
    pdl_wait();                                         // the activation operand comes from the previous kernel

    if (warp < 4) {
        asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");
        if (warp == 0 && lane == 0) {
            // ------------------------------------------------------------ TMA producer
            for (int item = pair; item < num_items; item += num_pairs) {
                const int img = item / a.groups_img, p0 = (item - img * a.groups_img) * a.G, p1 = min(a.pt_img, p0 + a.G);
                for (int ptl = p0; ptl < p1; ++ptl) {
                    const int rem = 2 * ptl + rank;     // tile inside the image; == tiles_img: a tile past the
                                                        // last one (odd tile count), computed but never stored
                    const int oy0 = (rem / a.tiles_x) * a.TH, ox0 = (rem % a.tiles_x) * a.TW;
                    int kb = 0;
                    for (int r = 0; r < a.R; ++r) {
                        for (int s = 0; s < a.S; ++s) {
                            const int ix = ox0 * a.sx + s - a.px, iy = oy0 * a.sy + r - a.py;
                            for (int c = 0; c < chunks; ++c, ++kb) {
                                ring.produce([&](uint32_t base, uint32_t fb) {
                                    tma_load_4d(base, &map_a_hi, fb, c * BK, ix, iy, img);
                                    tma_load_4d(base + C_A_BYTES, &map_a_lo, fb, c * BK, ix, iy, img);
                                    tma_load_2d(base + off_w_hi, &map_w_hi, fb, kb * BK, 0);
                                    tma_load_2d(base + off_w_lo, &map_w_lo, fb, kb * BK, 0);
                                });
                            }
                        }
                    }
                }
            }
        }
    } else {
        asm volatile("setmaxnreg.inc.sync.aligned.u32 232;");
        // ------------------------------------------------------------ consumers: MMA + epilogue, 64 pixels each
        const int wg = (warp - 4) >> 2, w4 = warp & 3;
        const bool releaser = (threadIdx.x & 127) == 0;
        constexpr int NJ = BN / 8;                            // 8-column blocks of the accumulator
        float acc[BN / 2];
        for (int item = pair; item < num_items; item += num_pairs) {
            const int img = item / a.groups_img, grp = item - img * a.groups_img;
            const int p0 = grp * a.G, p1 = min(a.pt_img, p0 + a.G);
            // per-warp statistics of the item: mine[column] = (mean, M2) over the warp's wcount valid pixels
            float* mine = comb + (warp - 4) * (BN * 2);
            float wcount = 0.f;
            if (a.partial) {
                for (int i = lane; i < BN * 2; i += 32) mine[i] = 0.f;
                __syncwarp();
            }
            for (int ptl = p0; ptl < p1; ++ptl) {
                int prev = -1;
                for (int kb = 0; kb < num_kb; ++kb) {
                    const uint32_t base = ring.wait();
                    const uint64_t a_hi = wgmma_desc_sw128(base + wg * (C_A_BYTES / 2));
                    const uint64_t a_lo = wgmma_desc_sw128(base + C_A_BYTES + wg * (C_A_BYTES / 2));
                    const uint64_t w_hi = wgmma_desc_sw128(base + off_w_hi);
                    const uint64_t w_lo = wgmma_desc_sw128(base + off_w_lo);
                    wgmma_fence();
#pragma unroll
                    for (int k = 0; k < BK / MMA_K; ++k) {
                        const uint64_t adv = static_cast<uint64_t>((k * MMA_K * 2) >> 4);
                        auto mma = [&](uint64_t a_desc, uint64_t w_desc, uint32_t accumulate) {
                            wgmma_tile<BN>(acc, a_desc + adv, w_desc + adv, accumulate);
                        };
                        mma_bf16x3(mma, a_hi, a_lo, w_hi, w_lo, (kb | k) != 0);
                    }
                    wgmma_commit();
                    if (prev >= 0) {
                        wgmma_wait<1>();
                        if (releaser) ring.release(prev);
                    }
                    prev = static_cast<int>(ring.stage);
                    ring.advance();
                }
                wgmma_wait<0>();
                wgmma_acc_ready(acc);
                if (releaser) ring.release(prev);

                const int rem = 2 * ptl + rank;
                const int i0 = wg * 64 + w4 * 16 + (lane >> 2);             // pixel index inside the tile (and i0 + 8)
                bool ok[2];
                float* orow[2];
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    const int i = i0 + 8 * h;
                    const int oy = (rem / a.tiles_x) * a.TH + i / a.TW, ox = (rem % a.tiles_x) * a.TW + i % a.TW;
                    ok[h] = rem < tiles_img && oy < a.Ho && ox < a.Wo;
                    orow[h] = a.out + ((static_cast<size_t>(img) * a.Ho + oy) * a.Wo + ox) * a.Cout;
                }
                // valid pixels among the warp's 16 (each pixel is held by the 4 lanes of a lane / 4 group)
                const int n16 = (__popc(__ballot_sync(0xffffffffu, ok[0])) + __popc(__ballot_sync(0xffffffffu, ok[1]))) >> 2;
                const float inv16 = n16 > 0 ? 1.f / n16 : 0.f;
                const float mf = n16 * (1.f / (wcount + n16)), mg = wcount * mf;    // merge weights, the same for every column
#pragma unroll
                for (int j = 0; j < NJ; ++j) {
                    const int col = 8 * j + 2 * (lane & 3);
                    const bool cok = col < a.Cout;                    // Cout is a multiple of 4: column pairs are whole
                    float2 b = make_float2(0.f, 0.f);
                    if (a.bias && cok) b = __ldg(reinterpret_cast<const float2*>(a.bias + col));
                    float2 o[2], s = make_float2(0.f, 0.f);
#pragma unroll
                    for (int h = 0; h < 2; ++h) {
                        o[h] = make_float2(acc[4 * j + 2 * h] + b.x, acc[4 * j + 2 * h + 1] + b.y);
                        if (ok[h] && cok) {
                            *reinterpret_cast<float2*>(orow[h] + col) = o[h];
                            s.x += o[h].x; s.y += o[h].y;
                        }
                    }
                    if (a.partial && n16 > 0) {
                        // (mean, M2) over the warp's valid pixels, two passes in registers, merged into the warp's
                        // running statistics of the item; lanes with equal lane % 4 hold the same columns
#pragma unroll
                        for (int w = 4; w <= 16; w <<= 1) { s.x += __shfl_xor_sync(0xffffffffu, s.x, w); s.y += __shfl_xor_sync(0xffffffffu, s.y, w); }
                        const float2 m = make_float2(s.x * inv16, s.y * inv16);
                        float2 q = make_float2(0.f, 0.f);
#pragma unroll
                        for (int h = 0; h < 2; ++h) {
                            if (ok[h]) {
                                const float dx = o[h].x - m.x, dy = o[h].y - m.y;
                                q.x = fmaf(dx, dx, q.x); q.y = fmaf(dy, dy, q.y);
                            }
                        }
#pragma unroll
                        for (int w = 4; w <= 16; w <<= 1) { q.x += __shfl_xor_sync(0xffffffffu, q.x, w); q.y += __shfl_xor_sync(0xffffffffu, q.y, w); }
                        if (lane < 4 && cok) {
                            chan_merge(mf, mg, mine[col * 2], mine[col * 2 + 1], m.x, q.x);
                            chan_merge(mf, mg, mine[col * 2 + 2], mine[col * 2 + 3], m.y, q.y);
                        }
                    }
                }
                wcount += static_cast<float>(n16);
            }
            if (a.partial) {
                // the 8 consumer warps' statistics merged in a fixed order
                if (lane == 0) counts[warp - 4] = wcount;
                asm volatile("bar.sync 1, 256;" ::: "memory");
                float* p = a.partial + ((static_cast<size_t>(img) * a.groups_img + grp) * 2 + rank) * 3 * a.Cout;
                for (int col = threadIdx.x - 128; col < a.Cout; col += 256) {
                    float n = 0.f, mean = 0.f, m2 = 0.f;
#pragma unroll
                    for (int w = 0; w < 8; ++w) {
                        if (counts[w] > 0.f) {
                            chan_merge_n(n, mean, m2, counts[w], comb[w * (BN * 2) + col * 2], comb[w * (BN * 2) + col * 2 + 1]);
                            n += counts[w];
                        }
                    }
                    p[col] = mean;
                    p[a.Cout + col] = m2;
                    p[2 * a.Cout + col] = n;
                }
                asm volatile("bar.sync 1, 256;" ::: "memory");    // comb is rewritten by the next item
            }
        }
    }
}

}  // namespace pips

using namespace pips;

// x_hi/x_lo: (N, H, W, Cp) bf16; w_hi/w_lo: (BN, R*S*Cp) bf16 with BN = Cout rounded up to 64/128/256 (zero rows);
// out: (N, Ho, Wo, Cout) fp32.
// tile shape and work-item grouping from the output geometry alone (the partial-statistics layout depends on it)
static void conv_geometry(int Ho, int Wo, int sx, ConvArgs& a) {
    // widest power-of-two tile row that does not exceed the output width (<= 128), the rest in rows
    int tw = 128;
    while (tw > 8 && tw > Wo) tw >>= 1;
    if (sx == 2 && (tw - 1) * 2 + 1 > 256) tw = 64;
    a.TW = tw; a.TH = 128 / tw;
    a.tiles_x = (Wo + a.TW - 1) / a.TW; a.tiles_y = (Ho + a.TH - 1) / a.TH;
    a.pt_img = (a.tiles_x * a.tiles_y + 1) / 2;               // pair tiles per image
    a.G = (a.pt_img + 31) / 32;                               // at most 32 groups (64 partial rows) per image
    a.groups_img = (a.pt_img + a.G - 1) / a.G;
}

template <int BN>
static int conv_tc_launch(const CUtensorMap& ma_hi, const CUtensorMap& ma_lo, const CUtensorMap& mw_hi, const CUtensorMap& mw_lo,
                          const ConvArgs& a, void* stream) {
    const int items = a.N * a.groups_img;
    const int max_pairs = sm_count() / 2;
    const int pairs = items < max_pairs ? items : max_pairs;
    return launch_kernel<conv_tc_kernel<BN>>("pips_conv_tc", true, 2 * pairs, C_THREADS, C_SMEM_BYTES, static_cast<cudaStream_t>(stream),
                                             ma_hi, ma_lo, mw_hi, mw_lo, a);
}

static int conv_tc_impl(const void* x_hi, const void* x_lo, int N, int H, int W, int Cp, const void* w_hi, const void* w_lo,
                        int Cout, int R, int S, int sy, int sx, int py, int px, const float* bias, float* out, float* partial,
                        void* stream) {
    if (!x_hi || !x_lo || !w_hi || !w_lo || !out) return fail("pips_conv_tc: null pointer");
    if (N <= 0 || H <= 0 || W <= 0 || Cp <= 0 || (Cp % BK)) return fail("pips_conv_tc: Cp must be a positive multiple of 64");
    if (Cout <= 0 || Cout > 256 || (Cout % 4)) return fail("pips_conv_tc: Cout must be a multiple of 4, at most 256");
    if (R <= 0 || S <= 0 || R > 7 || S > 7 || (sy != 1 && sy != 2) || (sx != 1 && sx != 2) || py < 0 || px < 0)
        return fail("pips_conv_tc: unsupported filter geometry");
    const int Ho = (H + 2 * py - R) / sy + 1, Wo = (W + 2 * px - S) / sx + 1;
    if (Ho <= 0 || Wo <= 0) return fail("pips_conv_tc: empty output");
    ConvArgs a;
    a.N = N; a.Ho = Ho; a.Wo = Wo; a.Cout = Cout; a.Cp = Cp; a.R = R; a.S = S; a.sy = sy; a.sx = sx; a.py = py; a.px = px;
    a.BN = Cout <= 64 ? 64 : (Cout <= 128 ? 128 : 256);
    {
        const uint32_t stage = 2 * (C_A_BYTES + static_cast<uint32_t>(a.BN) * BK * 2);
        int st = static_cast<int>(C_RING_BYTES / stage);
        a.stages = st > C_MAX_STAGES ? C_MAX_STAGES : st;      // BN 256: 2 x 96 KB, 128: 3 x 64 KB, 64: 4 x 48 KB
    }
    conv_geometry(Ho, Wo, sx, a);
    a.bias = bias; a.out = out; a.partial = partial;

    CUtensorMap ma_hi, ma_lo, mw_hi, mw_lo;
    {
        cuuint64_t gdim[4] = {static_cast<cuuint64_t>(Cp), static_cast<cuuint64_t>(W), static_cast<cuuint64_t>(H), static_cast<cuuint64_t>(N)};
        cuuint64_t gstr[3] = {static_cast<cuuint64_t>(Cp) * 2, static_cast<cuuint64_t>(W) * Cp * 2, static_cast<cuuint64_t>(H) * W * Cp * 2};
        cuuint32_t box[4] = {static_cast<cuuint32_t>(BK), static_cast<cuuint32_t>((a.TW - 1) * sx + 1),
                             static_cast<cuuint32_t>((a.TH - 1) * sy + 1), 1};
        cuuint32_t estr[4] = {1, static_cast<cuuint32_t>(sx), static_cast<cuuint32_t>(sy), 1};
        if (!encode_tiled_pair(&ma_hi, &ma_lo, x_hi, x_lo, 4, gdim, gstr, box, estr, CU_TENSOR_MAP_SWIZZLE_128B))
            return fail("pips_conv_tc: activation tensor map failed");
    }
    {
        const int K = R * S * Cp;
        cuuint64_t gdim[2] = {static_cast<cuuint64_t>(K), static_cast<cuuint64_t>(a.BN)};
        cuuint64_t gstr[1] = {static_cast<cuuint64_t>(K) * 2};
        cuuint32_t box[2] = {static_cast<cuuint32_t>(BK), static_cast<cuuint32_t>(a.BN)};
        cuuint32_t estr[2] = {1, 1};
        if (!encode_tiled_pair(&mw_hi, &mw_lo, w_hi, w_lo, 2, gdim, gstr, box, estr, CU_TENSOR_MAP_SWIZZLE_128B))
            return fail("pips_conv_tc: weight tensor map failed");
    }
    return a.BN == 64 ? conv_tc_launch<64>(ma_hi, ma_lo, mw_hi, mw_lo, a, stream)
         : a.BN == 128 ? conv_tc_launch<128>(ma_hi, ma_lo, mw_hi, mw_lo, a, stream)
                       : conv_tc_launch<256>(ma_hi, ma_lo, mw_hi, mw_lo, a, stream);
}

extern "C" int pips_conv_tc(const void* x_hi, const void* x_lo, int N, int H, int W, int Cp, const void* w_hi, const void* w_lo,
                            int Cout, int R, int S, int stride, int pad, const float* bias, float* out, void* stream) {
    return conv_tc_impl(x_hi, x_lo, N, H, W, Cp, w_hi, w_lo, Cout, R, S, stride, stride, pad, pad, bias, out, nullptr, stream);
}

// Anisotropic form (separate row / column stride and padding): the 7x7 stem runs as a 7x1 convolution over the
// column-unfolded image written by pips_stem_pack.
extern "C" int pips_conv_tc_aniso(const void* x_hi, const void* x_lo, int N, int H, int W, int Cp, const void* w_hi, const void* w_lo,
                                  int Cout, int R, int S, int stride_y, int stride_x, int pad_y, int pad_x, const float* bias,
                                  float* out, void* stream) {
    return conv_tc_impl(x_hi, x_lo, N, H, W, Cp, w_hi, w_lo, Cout, R, S, stride_y, stride_x, pad_y, pad_x, bias, out, nullptr, stream);
}

// Number of partial-statistics rows per image pips_conv_tc_stats writes for this geometry (0: invalid geometry).
extern "C" int pips_conv_tc_chunks(int H, int W, int R, int S, int stride_y, int stride_x, int pad_y, int pad_x) {
    if (H <= 0 || W <= 0 || R <= 0 || S <= 0 || stride_y <= 0 || stride_x <= 0) return 0;
    const int Ho = (H + 2 * pad_y - R) / stride_y + 1, Wo = (W + 2 * pad_x - S) / stride_x + 1;
    if (Ho <= 0 || Wo <= 0) return 0;
    ConvArgs a;
    conv_geometry(Ho, Wo, stride_x, a);
    return a.groups_img * 2;
}

// pips_conv_tc_aniso that also accumulates the InstanceNorm partial statistics of its output in the epilogue:
// partial (N, pips_conv_tc_chunks(...), 3, Cout) fp32 = per chunk (mean, M2, count) per channel, for pips_inorm_finalize.
extern "C" int pips_conv_tc_stats(const void* x_hi, const void* x_lo, int N, int H, int W, int Cp, const void* w_hi, const void* w_lo,
                                  int Cout, int R, int S, int stride_y, int stride_x, int pad_y, int pad_x, const float* bias,
                                  float* out, float* partial, void* stream) {
    if (!partial) return fail("pips_conv_tc_stats: null partial buffer");
    return conv_tc_impl(x_hi, x_lo, N, H, W, Cp, w_hi, w_lo, Cout, R, S, stride_y, stride_x, pad_y, pad_x, bias, out, partial, stream);
}
