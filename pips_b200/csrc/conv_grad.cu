// Weight gradient of the feature encoder's convolutions on the Hopper tensor cores (wgmma), bf16x3:
//
//   dW[co, (r*S + s)*Cp + ci] = sum_{n, oy, ox} dY[n, oy, ox, co] * X[n, oy*sy + r - py, ox*sx + s - px, ci]
//
// An implicit GEMM with the pixels as the contraction index, on the pipeline of the dense weight-gradient GEMM
// (gemm_tc.cu, pips_wgrad): a TMA producer warp, the shared ring (gemm_common.cuh), two consumer warpgroups of 64 output
// channels each, both operands MN-major with 64-byte swizzle.  A ring stage holds one tile of 32 output pixels (TH rows x
// TW columns of one image): the 128 co of the tile as four {32 co, TW, TH, 1} boxes of dY, and the 128 k of the tile as
// four {32 ci, TW, TH, 1} boxes of X, each at its filter tap's offset with the element strides set to the conv stride --
// the same 4-D box conv_tc loads for that tap.  Boxes outside the image are filled with zero by TMA, so padding needs
// no code and no im2col buffer exists.  With dy_step = 2 the dY boxes read every other pixel of a zero-dilated
// gradient (the layout the strided convolutions' input gradient needs), so the same buffer serves both.
//
// It is a kernel of its own, not a variant of gemm_tc_body's weight-gradient path: there the producer's box coordinates
// are not kept in uniform registers, so each of a stage's 16 4-D loads goes through an elected-lane loop of register
// moves, and with 6 MMAs per 32-pixel stage the producer sets the pace (16 % slower on layer1).  Here they are uniform.
//
// A work item is (128 co, 128 k, chunk of pixel tiles).  The chunk size depends on the geometry only; every chunk
// writes its own partial dW, and the chunks are added in order by the column-sum kernel: no atomics, the same bits
// on any number of SMs.
#include "gemm_common.cuh"

namespace pips {

constexpr int CW_THREADS = 384;
constexpr int CW_PIX = 32;                                  // pixels per ring stage
constexpr uint32_t CW_BOX = 32 * CW_PIX * 2;                // {32 channels, 32 pixels} bf16: 2 KB
constexpr uint32_t CW_TILE = 4 * CW_BOX;                    // 128 channels
constexpr uint32_t CW_STAGE = 4 * CW_TILE;                  // dY hi | X hi | dY lo | X lo: 32 KB
constexpr int CW_STAGES = 6;
constexpr uint32_t CW_SMEM = CW_STAGES * CW_STAGE + 1024 + 256;
constexpr int CW_TARGET_ITEMS = 1024;                       // work items a problem is split into (about 8 per SM)
constexpr int CW_MAX_SPLITS = 256;                          // one pass of the column-sum kernel adds them

struct ConvWgradArgs {
    int Cout, K, Cp, S;                 // dW is (Cout, K), K = R*S*Cp
    int sy, sx, py, px, step;           // conv stride and padding, dY pixel step (2: zero-dilated dY)
    int TW, TH, tiles_x, tiles_img;     // pixel tiles of the output
    int tiles;                          // N * tiles_img
    int k_blocks, splits, chunk;        // 128-wide k blocks, chunks of `chunk` pixel tiles
    int num_items;
    float* out;                         // (splits, Cout, K) partials, or dW when splits == 1
};

__global__ void __launch_bounds__(CW_THREADS, 1)
conv_wgrad_kernel(const __grid_constant__ CUtensorMap map_dy_hi, const __grid_constant__ CUtensorMap map_dy_lo,
                  const __grid_constant__ CUtensorMap map_x_hi, const __grid_constant__ CUtensorMap map_x_lo,
                  const ConvWgradArgs a) {
    pdl_trigger();
    uint8_t* smem = aligned_smem();
    Ring ring(smem, CW_STAGE, CW_STAGES, reinterpret_cast<uint64_t*>(smem + CW_STAGES * CW_STAGE), CW_STAGES);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

    if (warp == 0 && lane == 0) {
        tma_prefetch_desc(&map_dy_hi); tma_prefetch_desc(&map_dy_lo);
        tma_prefetch_desc(&map_x_hi); tma_prefetch_desc(&map_x_lo);
    }
    if (warp == 1 && lane == 0) ring.init(2);              // one arrival per consumer warpgroup
    __syncthreads();
    pdl_wait();

    // item -> (first co, first k, pixel-tile range)
    auto coords = [&](int t, int& n0, int& k0, int& q0, int& q1, int& split) {
        split = t % a.splits;
        t /= a.splits;
        k0 = (t % a.k_blocks) * 128;
        n0 = (t / a.k_blocks) * 128;
        q0 = split * a.chunk;
        q1 = min(a.tiles, q0 + a.chunk);
    };

    if (warp < 4) {
        asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");
        if (warp == 0 && lane == 0) {
            // ------------------------------------------------------------ TMA producer
            for (int t = blockIdx.x; t < a.num_items; t += gridDim.x) {
                int n0, k0, q0, q1, split;
                coords(t, n0, k0, q0, q1, split);
                // the tap and channel of each 32-wide k box (k past K: a channel past Cp, i.e. a box of zeros)
                int bc[4], bx[4], by[4];
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                    const int k = k0 + 32 * i;
                    const int tap = k < a.K ? k / a.Cp : 0;
                    const int r = tap / a.S, s = tap - r * a.S;
                    bc[i] = k < a.K ? k - tap * a.Cp : a.Cp;
                    bx[i] = s - a.px;
                    by[i] = r - a.py;
                }
                for (int q = q0; q < q1; ++q) {
                    const int img = q / a.tiles_img;
                    const int rem = q - img * a.tiles_img;
                    const int oy0 = (rem / a.tiles_x) * a.TH, ox0 = (rem % a.tiles_x) * a.TW;
                    ring.produce([&](uint32_t base, uint32_t fb) {
#pragma unroll
                        for (int i = 0; i < 4; ++i) {
                            const int x = ox0 * a.sx + bx[i], y = oy0 * a.sy + by[i];
                            tma_load_4d(base + i * CW_BOX, &map_dy_hi, fb, n0 + 32 * i, ox0 * a.step, oy0 * a.step, img);
                            tma_load_4d(base + CW_TILE + i * CW_BOX, &map_x_hi, fb, bc[i], x, y, img);
                            tma_load_4d(base + 2 * CW_TILE + i * CW_BOX, &map_dy_lo, fb, n0 + 32 * i, ox0 * a.step, oy0 * a.step, img);
                            tma_load_4d(base + 3 * CW_TILE + i * CW_BOX, &map_x_lo, fb, bc[i], x, y, img);
                        }
                    });
                }
            }
        }
    } else {
        asm volatile("setmaxnreg.inc.sync.aligned.u32 232;");
        // ------------------------------------------------------------ consumers: 64 co x 128 k each
        const int wg = (warp - 4) >> 2;
        const bool releaser = (threadIdx.x & 127) == 0;
        float acc[64];
        auto mma = [&](uint64_t a_desc, uint64_t x_desc, uint32_t accumulate) { wgmma_n128_tt(acc, a_desc, x_desc, accumulate); };
        for (int t = blockIdx.x; t < a.num_items; t += gridDim.x) {
            int n0, k0, q0, q1, split;
            coords(t, n0, k0, q0, q1, split);
            int prev = -1;
            for (int q = q0; q < q1; ++q) {
                const uint32_t base = ring.wait();
                const uint32_t a_hi = base + wg * 2 * CW_BOX, x_hi = base + CW_TILE;
                const uint32_t a_lo = a_hi + 2 * CW_TILE, x_lo = x_hi + 2 * CW_TILE;
                wgmma_fence();
#pragma unroll
                for (int k = 0; k < CW_PIX / MMA_K; ++k) {
                    mma_bf16x3(mma, wgmma_desc_sw64_mn(a_hi + k * 1024, CW_BOX), wgmma_desc_sw64_mn(a_lo + k * 1024, CW_BOX),
                               wgmma_desc_sw64_mn(x_hi + k * 1024, CW_BOX), wgmma_desc_sw64_mn(x_lo + k * 1024, CW_BOX), (q != q0) | k);
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
            // the warpgroup's 64 x 128 partial sum straight from registers to its slice of the output
            float* out = a.out + static_cast<size_t>(split) * a.Cout * a.K;
            const int r = (warp & 3) * 16 + (lane >> 2);
            const int cq = 2 * (lane & 3);
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int n = n0 + wg * 64 + r + 8 * h;
                if (n >= a.Cout) continue;
                float* o = out + static_cast<size_t>(n) * a.K;
#pragma unroll
                for (int j = 0; j < 16; ++j) {
                    const int k = k0 + 8 * j + cq;                    // K % 64 == 0: k < K covers k + 1
                    if (k < a.K) *reinterpret_cast<float2*>(o + k) = make_float2(acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1]);
                }
            }
        }
    }
}

int colsum_launch(const float* g, const void* g_hi, const void* g_lo, size_t ld, int M, int N, float* scratch, float* out,
                  cudaStream_t st);   // mixer_grad.cu

}  // namespace pips

using namespace pips;

// pixel tiles and chunking from the geometry alone (the partial sums, and so the bits, depend on it)
static bool wgrad_geometry(int N, int Ho, int Wo, int Cout, int K, ConvWgradArgs& a) {
    if (N <= 0 || Ho <= 0 || Wo <= 0 || Cout <= 0 || K <= 0) return false;
    a.TW = Wo >= 32 ? 32 : (Wo >= 16 ? 16 : 8);
    a.TH = CW_PIX / a.TW;
    a.tiles_x = (Wo + a.TW - 1) / a.TW;
    a.tiles_img = a.tiles_x * ((Ho + a.TH - 1) / a.TH);
    const long long tiles = static_cast<long long>(N) * a.tiles_img;
    if (tiles > 0x7fffffffLL) return false;
    a.Cout = Cout; a.K = K;
    a.k_blocks = (K + 127) / 128;
    const int blocks = a.k_blocks * ((Cout + 127) / 128);
    int splits = (CW_TARGET_ITEMS + blocks - 1) / blocks;
    if (splits > CW_MAX_SPLITS) splits = CW_MAX_SPLITS;
    if (splits > tiles) splits = static_cast<int>(tiles);
    a.tiles = static_cast<int>(tiles);
    a.chunk = static_cast<int>((tiles + splits - 1) / splits);
    a.splits = static_cast<int>((tiles + a.chunk - 1) / a.chunk);
    a.num_items = blocks * a.splits;
    return true;
}

extern "C" size_t pips_conv_wgrad_scratch_floats(int N, int Ho, int Wo, int Cout, int K) {
    ConvWgradArgs a;
    if (!wgrad_geometry(N, Ho, Wo, Cout, K, a)) return 0;
    return a.splits > 1 ? static_cast<size_t>(a.splits) * Cout * K : 0;
}

extern "C" int pips_conv_wgrad(const void* dy_hi, const void* dy_lo, int ldy, int dy_step, const void* x_hi, const void* x_lo,
                               int N, int H, int W, int Cp, int Cout, int R, int S, int stride_y, int stride_x, int pad_y,
                               int pad_x, float* scratch, float* dw, void* stream) {
    if (!dy_hi || !dy_lo || !x_hi || !x_lo || !dw) return fail("pips_conv_wgrad: null pointer");
    if (N <= 0 || H <= 0 || W <= 0 || Cp <= 0 || (Cp % 64)) return fail("pips_conv_wgrad: Cp must be a positive multiple of 64");
    if (Cout <= 0 || ldy < Cout || (ldy % 8)) return fail("pips_conv_wgrad: ldy must be >= Cout and a multiple of 8");
    if (R <= 0 || S <= 0 || R > 7 || S > 7 || (stride_y != 1 && stride_y != 2) || (stride_x != 1 && stride_x != 2) || pad_y < 0 || pad_x < 0)
        return fail("pips_conv_wgrad: unsupported filter geometry");
    if (dy_step != 1 && !(dy_step == 2 && stride_y == 2 && stride_x == 2))
        return fail("pips_conv_wgrad: dy_step must be 1, or 2 for a stride-2 convolution");
    const int Ho = (H + 2 * pad_y - R) / stride_y + 1, Wo = (W + 2 * pad_x - S) / stride_x + 1;
    if (Ho <= 0 || Wo <= 0) return fail("pips_conv_wgrad: empty output");
    if ((reinterpret_cast<uintptr_t>(dy_hi) | reinterpret_cast<uintptr_t>(dy_lo) | reinterpret_cast<uintptr_t>(x_hi)
         | reinterpret_cast<uintptr_t>(x_lo) | reinterpret_cast<uintptr_t>(dw) | reinterpret_cast<uintptr_t>(scratch)) & 15)
        return fail("pips_conv_wgrad: operands, scratch and dw must be 16-byte aligned");
    const int K = R * S * Cp;
    if (static_cast<long long>(Cout) * K > 0x7fffffffLL) return fail("pips_conv_wgrad: problem too large");
    ConvWgradArgs a;
    if (!wgrad_geometry(N, Ho, Wo, Cout, K, a)) return fail("pips_conv_wgrad: problem too large");
    if (a.splits > 1 && !scratch) return fail("pips_conv_wgrad: scratch of pips_conv_wgrad_scratch_floats(...) floats is required");
    a.Cp = Cp; a.S = S; a.sy = stride_y; a.sx = stride_x; a.py = pad_y; a.px = pad_x; a.step = dy_step;
    a.out = a.splits > 1 ? scratch : dw;

    CUtensorMap mdy_hi, mdy_lo, mx_hi, mx_lo;
    {
        // dY: (N, Hd, Wd, ldy); a zero-dilated dY lives on the input's grid
        const int Hd = dy_step == 1 ? Ho : H, Wd = dy_step == 1 ? Wo : W;
        cuuint64_t gdim[4] = {static_cast<cuuint64_t>(ldy), static_cast<cuuint64_t>(Wd), static_cast<cuuint64_t>(Hd), static_cast<cuuint64_t>(N)};
        cuuint64_t gstr[3] = {static_cast<cuuint64_t>(ldy) * 2, static_cast<cuuint64_t>(Wd) * ldy * 2, static_cast<cuuint64_t>(Hd) * Wd * ldy * 2};
        cuuint32_t box[4] = {32, static_cast<cuuint32_t>((a.TW - 1) * dy_step + 1), static_cast<cuuint32_t>((a.TH - 1) * dy_step + 1), 1};
        cuuint32_t estr[4] = {1, static_cast<cuuint32_t>(dy_step), static_cast<cuuint32_t>(dy_step), 1};
        if (!encode_tiled_pair(&mdy_hi, &mdy_lo, dy_hi, dy_lo, 4, gdim, gstr, box, estr, CU_TENSOR_MAP_SWIZZLE_64B))
            return fail("pips_conv_wgrad: gradient tensor map failed");
    }
    {
        cuuint64_t gdim[4] = {static_cast<cuuint64_t>(Cp), static_cast<cuuint64_t>(W), static_cast<cuuint64_t>(H), static_cast<cuuint64_t>(N)};
        cuuint64_t gstr[3] = {static_cast<cuuint64_t>(Cp) * 2, static_cast<cuuint64_t>(W) * Cp * 2, static_cast<cuuint64_t>(H) * W * Cp * 2};
        cuuint32_t box[4] = {32, static_cast<cuuint32_t>((a.TW - 1) * stride_x + 1), static_cast<cuuint32_t>((a.TH - 1) * stride_y + 1), 1};
        cuuint32_t estr[4] = {1, static_cast<cuuint32_t>(stride_x), static_cast<cuuint32_t>(stride_y), 1};
        if (!encode_tiled_pair(&mx_hi, &mx_lo, x_hi, x_lo, 4, gdim, gstr, box, estr, CU_TENSOR_MAP_SWIZZLE_64B))
            return fail("pips_conv_wgrad: activation tensor map failed");
    }
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const int grid = a.num_items < sm_count() ? a.num_items : sm_count();
    if (const int err = launch_kernel<conv_wgrad_kernel>("pips_conv_wgrad", true, grid, CW_THREADS, CW_SMEM, st, mdy_hi, mdy_lo, mx_hi,
                                                         mx_lo, a))
        return err;
    if (a.splits == 1) return 0;
    const size_t nk = static_cast<size_t>(Cout) * K;
    return colsum_launch(scratch, nullptr, nullptr, nk, a.splits, static_cast<int>(nk), nullptr, dw, st);
}
