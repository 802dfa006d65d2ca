// Channels-last element-wise stages of the feature encoder (fnet, nets/pips.py:131-281), fused so that
// between two convolutions every activation is read once and written once:
//   pips_inorm_stats     InstanceNorm2d statistics per (frame, channel) over H*W          (:154-157, :200-201)
//   pips_inorm_apply     normalise (+ReLU) (+residual, itself optionally normalised) (+ReLU) and emit the
//                        plain fp32 activation and/or the [hi | lo | hi] TF32-split operand of the next conv
//   pips_resize_split3   F.interpolate(bilinear, align_corners=True) of a stage output into its channel slice
//                        of the 416-channel concat, already split                          (:269-273)
// The convolutions themselves stay on cuDNN (TF32 tensor cores, 3-term split => fp32-class accuracy);
// fnet is upstream of the refinement hot path (SURVEY.md section 8a row a13).
#include "common.cuh"

namespace pips {

__device__ __forceinline__ float tf32_hi(float v) { return __uint_as_float(__float_as_uint(v) & 0xffffe000u); }

// ---------------------------------------------------------------------------------------- statistics
// Partial statistics: per (image, chunk) three rows of C floats, (mean, M2, count) of the chunk's pixels (chan_merge).
// grid (chunks, N); block 256 threads = (C/4 float4 lanes) x rows; every thread runs Welford's update over its pixels
// in fp32, rows are merged through smem in a fixed order, chunks by the finalize kernel in fp64: deterministic.
__device__ __forceinline__ void welford(float n, float v, float& mean, float& m2) {
    const float d = v - mean;
    mean += d / n;
    m2 = fmaf(d, v - mean, m2);
}

__global__ void __launch_bounds__(256)
inorm_partial_kernel(const float* __restrict__ y, int HW, int C, int chunk_px, float* __restrict__ partial) {
    extern __shared__ float sm[];                       // [rows][2][C]: (mean, M2)
    pdl_trigger();
    pdl_wait();
    const int c4n = C >> 2;
    const int lane_c = threadIdx.x % c4n, row = threadIdx.x / c4n, rows = blockDim.x / c4n;
    const int n = blockIdx.y, chunk = blockIdx.x;
    const int p0 = chunk * chunk_px, p1 = min(HW, p0 + chunk_px);
    if (row < rows) {
        float4 m = make_float4(0.f, 0.f, 0.f, 0.f), q = m;
        float cnt = 0.f;
        const float4* base = reinterpret_cast<const float4*>(y + (static_cast<size_t>(n) * HW) * C) + lane_c;
        for (int p = p0 + row; p < p1; p += rows) {
            const float4 v = base[static_cast<size_t>(p) * c4n];
            cnt += 1.f;
            welford(cnt, v.x, m.x, q.x); welford(cnt, v.y, m.y, q.y); welford(cnt, v.z, m.z, q.z); welford(cnt, v.w, m.w, q.w);
        }
        float* d = sm + (row * 2) * C + lane_c * 4;
        d[0] = m.x; d[1] = m.y; d[2] = m.z; d[3] = m.w;
        d[C + 0] = q.x; d[C + 1] = q.y; d[C + 2] = q.z; d[C + 3] = q.w;
    }
    __syncthreads();
    float* out = partial + (static_cast<size_t>(n) * gridDim.x + chunk) * 3 * C;
    for (int c = threadIdx.x; c < C; c += blockDim.x) {
        float cnt = 0.f, mean = 0.f, m2 = 0.f;
        for (int r = 0; r < rows; ++r) {
            const float nr = static_cast<float>(p1 - p0 - r > 0 ? (p1 - p0 - r + rows - 1) / rows : 0);   // pixels of row r
            if (nr > 0.f) { chan_merge_n(cnt, mean, m2, nr, sm[r * 2 * C + c], sm[r * 2 * C + C + c]); cnt += nr; }
        }
        out[c] = mean; out[C + c] = m2; out[2 * C + c] = cnt;
    }
}

// (mean, rstd) per (image, channel) from the chunks' (mean, M2, count), merged in fp64
__global__ void inorm_finalize_kernel(const float* __restrict__ partial, int chunks, int HW, int C, float* __restrict__ stats) {
    const int n = blockIdx.x;
    pdl_trigger();
    pdl_wait();
    const float* pn = partial + static_cast<size_t>(n) * chunks * 3 * C;
    for (int c = threadIdx.x; c < C; c += blockDim.x) {
        double s = 0.0;
        for (int k = 0; k < chunks; ++k) s += static_cast<double>(pn[k * 3 * C + 2 * C + c]) * pn[k * 3 * C + c];
        const double mean = s / HW;
        double m2 = 0.0;
        for (int k = 0; k < chunks; ++k) {
            const double d = static_cast<double>(pn[k * 3 * C + c]) - mean;
            m2 += pn[k * 3 * C + C + c] + pn[k * 3 * C + 2 * C + c] * d * d;
        }
        const double var = m2 / HW;                     // biased variance, as InstanceNorm uses for normalisation
        stats[(static_cast<size_t>(n) * 2) * C + c] = static_cast<float>(mean);
        stats[(static_cast<size_t>(n) * 2 + 1) * C + c] = static_cast<float>(1.0 / sqrt(var + 1e-5));
    }
}

// ---------------------------------------------------------------------------------------- apply
struct ApplyArgs {
    const float* y; const float* stats_y;               // stats NULL => y used as is
    const float* r; const float* stats_r;               // optional residual (+ optional normalisation)
    int relu_main, relu_out;
    float* out_plain; float* out_split; int split_ld;   // split_ld = channels of the split tensor (>= 3*C)
    __nv_bfloat16* out_hi; __nv_bfloat16* out_lo; int pair_ld;   // bf16 (hi, lo) operand of pips_conv_tc, row stride pair_ld >= C
    int HW, C;
};

__global__ void __launch_bounds__(256)
inorm_apply_kernel(const ApplyArgs a, size_t total4) {
    pdl_trigger();
    pdl_wait();
    const int c4n = a.C >> 2;
    // with a bf16 pair output the loop also covers the pair's padding channels [C, pair_ld) and writes them as zero
    // (they are K padding of the next convolution): no separate fill pass over the operand
    const int c4p = a.out_hi ? a.pair_ld >> 2 : c4n;
    for (size_t j = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; j < total4; j += static_cast<size_t>(gridDim.x) * blockDim.x) {
        const int c4 = static_cast<int>(j % c4p);
        const size_t pix = j / c4p;                      // n*HW + p
        if (c4 >= c4n) {
            const size_t o = pix * a.pair_ld + c4 * 4;
            *reinterpret_cast<uint2*>(a.out_hi + o) = make_uint2(0u, 0u);
            *reinterpret_cast<uint2*>(a.out_lo + o) = make_uint2(0u, 0u);
            continue;
        }
        const size_t i = pix * c4n + c4;
        const int n = static_cast<int>(pix / a.HW);
        float4 v = reinterpret_cast<const float4*>(a.y)[i];
        if (a.stats_y) {
            const float4 m = reinterpret_cast<const float4*>(a.stats_y + static_cast<size_t>(n) * 2 * a.C)[c4];
            const float4 s = reinterpret_cast<const float4*>(a.stats_y + (static_cast<size_t>(n) * 2 + 1) * a.C)[c4];
            v.x = (v.x - m.x) * s.x; v.y = (v.y - m.y) * s.y; v.z = (v.z - m.z) * s.z; v.w = (v.w - m.w) * s.w;
        }
        if (a.relu_main) { v.x = fmaxf(v.x, 0.f); v.y = fmaxf(v.y, 0.f); v.z = fmaxf(v.z, 0.f); v.w = fmaxf(v.w, 0.f); }
        if (a.r) {
            float4 w = reinterpret_cast<const float4*>(a.r)[i];
            if (a.stats_r) {
                const float4 m = reinterpret_cast<const float4*>(a.stats_r + static_cast<size_t>(n) * 2 * a.C)[c4];
                const float4 s = reinterpret_cast<const float4*>(a.stats_r + (static_cast<size_t>(n) * 2 + 1) * a.C)[c4];
                w.x = (w.x - m.x) * s.x; w.y = (w.y - m.y) * s.y; w.z = (w.z - m.z) * s.z; w.w = (w.w - m.w) * s.w;
            }
            v.x += w.x; v.y += w.y; v.z += w.z; v.w += w.w;
        }
        if (a.relu_out) { v.x = fmaxf(v.x, 0.f); v.y = fmaxf(v.y, 0.f); v.z = fmaxf(v.z, 0.f); v.w = fmaxf(v.w, 0.f); }
        if (a.out_plain) reinterpret_cast<float4*>(a.out_plain)[i] = v;
        if (a.out_split) {
            const float4 h = make_float4(tf32_hi(v.x), tf32_hi(v.y), tf32_hi(v.z), tf32_hi(v.w));
            const float4 l = make_float4(v.x - h.x, v.y - h.y, v.z - h.z, v.w - h.w);
            float* d = a.out_split + pix * a.split_ld + c4 * 4;
            *reinterpret_cast<float4*>(d) = h;
            *reinterpret_cast<float4*>(d + a.C) = l;
            *reinterpret_cast<float4*>(d + 2 * a.C) = h;
        }
        if (a.out_hi) {
            __nv_bfloat16 h[4], l[4];
            split_bf16(v.x, h[0], l[0]); split_bf16(v.y, h[1], l[1]); split_bf16(v.z, h[2], l[2]); split_bf16(v.w, h[3], l[3]);
            const size_t o = pix * a.pair_ld + c4 * 4;
            *reinterpret_cast<uint2*>(a.out_hi + o) = make_uint2(pack_bf16(h[0], h[1]), pack_bf16(h[2], h[3]));
            *reinterpret_cast<uint2*>(a.out_lo + o) = make_uint2(pack_bf16(l[0], l[1]), pack_bf16(l[2], l[3]));
        }
    }
}

// ---------------------------------------------------------------------------------------- resize into the concat
__global__ void __launch_bounds__(256)
resize_split3_kernel(const float* __restrict__ src, int Hs, int Ws, int C, float* __restrict__ dst, __nv_bfloat16* __restrict__ dst_hi,
                     __nv_bfloat16* __restrict__ dst_lo, int Ho, int Wo, int Ctot, int c_off, size_t total4) {
    // bf16 pair output: when fewer than 64 channels remain after this slice they are the concat's K padding (rows are padded
    // to a multiple of 64) -- this call writes them as zero, so the concat needs no fill pass
    pdl_trigger();
    pdl_wait();
    const int tail = (!dst && Ctot - (c_off + C) < 64) ? Ctot - (c_off + C) : 0;
    const int c4n = (C + tail) >> 2, c4v = C >> 2;
    // at::native area_pixel_compute_scale(align_corners=true): (in - 1) / (out - 1), 0 when out == 1
    const float sh = Ho > 1 ? static_cast<float>(Hs - 1) / static_cast<float>(Ho - 1) : 0.f;
    const float sw = Wo > 1 ? static_cast<float>(Ws - 1) / static_cast<float>(Wo - 1) : 0.f;
    for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < total4; i += static_cast<size_t>(gridDim.x) * blockDim.x) {
        const int c4 = static_cast<int>(i % c4n);
        size_t p = i / c4n;
        const int ox = static_cast<int>(p % Wo); p /= Wo;
        const int oy = static_cast<int>(p % Ho);
        const int n = static_cast<int>(p / Ho);
        if (c4 >= c4v) {
            const size_t o = ((static_cast<size_t>(n) * Ho + oy) * Wo + ox) * static_cast<size_t>(Ctot) + c_off + c4 * 4;
            *reinterpret_cast<uint2*>(dst_hi + o) = make_uint2(0u, 0u);
            *reinterpret_cast<uint2*>(dst_lo + o) = make_uint2(0u, 0u);
            continue;
        }
        const float fy = sh * oy, fx = sw * ox;
        const int y0 = static_cast<int>(fy), x0 = static_cast<int>(fx);
        const int yp = y0 < Hs - 1 ? 1 : 0, xp = x0 < Ws - 1 ? 1 : 0;
        const float ly = fy - y0, lx = fx - x0, hy = 1.f - ly, hx = 1.f - lx;
        const float4* b = reinterpret_cast<const float4*>(src + ((static_cast<size_t>(n) * Hs + y0) * Ws + x0) * C) + c4;
        const float4 v00 = b[0], v01 = b[static_cast<size_t>(xp) * c4v];
        const float4 v10 = b[static_cast<size_t>(yp) * Ws * c4v], v11 = b[(static_cast<size_t>(yp) * Ws + xp) * c4v];
        float4 v;
        v.x = hy * (hx * v00.x + lx * v01.x) + ly * (hx * v10.x + lx * v11.x);
        v.y = hy * (hx * v00.y + lx * v01.y) + ly * (hx * v10.y + lx * v11.y);
        v.z = hy * (hx * v00.z + lx * v01.z) + ly * (hx * v10.z + lx * v11.z);
        v.w = hy * (hx * v00.w + lx * v01.w) + ly * (hx * v10.w + lx * v11.w);
        if (dst) {
            const float4 h = make_float4(tf32_hi(v.x), tf32_hi(v.y), tf32_hi(v.z), tf32_hi(v.w));
            const float4 l = make_float4(v.x - h.x, v.y - h.y, v.z - h.z, v.w - h.w);
            float* d = dst + ((static_cast<size_t>(n) * Ho + oy) * Wo + ox) * (3 * static_cast<size_t>(Ctot)) + c_off + c4 * 4;
            *reinterpret_cast<float4*>(d) = h;
            *reinterpret_cast<float4*>(d + Ctot) = l;
            *reinterpret_cast<float4*>(d + 2 * Ctot) = h;
        } else {                                        // bf16 (hi, lo) pair, row stride Ctot
            __nv_bfloat16 h[4], l[4];
            split_bf16(v.x, h[0], l[0]); split_bf16(v.y, h[1], l[1]); split_bf16(v.z, h[2], l[2]); split_bf16(v.w, h[3], l[3]);
            const size_t o = ((static_cast<size_t>(n) * Ho + oy) * Wo + ox) * static_cast<size_t>(Ctot) + c_off + c4 * 4;
            *reinterpret_cast<uint2*>(dst_hi + o) = make_uint2(pack_bf16(h[0], h[1]), pack_bf16(h[2], h[3]));
            *reinterpret_cast<uint2*>(dst_lo + o) = make_uint2(pack_bf16(l[0], l[1]), pack_bf16(l[2], l[3]));
        }
    }
}

// ---------------------------------------------------------------------------------------- stem input
// nets/pips.py:436 (2*(rgb/255)-1) fused with the unfolding of the 7x7 / stride-2 stem (:206) into a plain stride-1
// convolution with 4 row taps over 64-channel pixels.  Output pixel (j, ox) of the unfolded tensor holds, for the TWO
// input rows y = 2j-3 and y = 2j-2, the 7 column taps x 3 colours at x = 2*ox + s - 3 (zero outside the image):
//   channels [ 0,32): row 2j-3, k = s*3 + colour (21 used)      channels [32,64): row 2j-2, same order
// Output row oy of the stem needs input rows 2oy-3 .. 2oy+3 = row pairs j = oy .. oy+3 (the 8th row, 2oy+4, meets a zero
// filter row), i.e. a 4x1 convolution with stride 1 and no padding over the (Ho+3) x Wo unfolded image: K = 4 x 64 = 256.
// (Round 1 unfolded only the columns: one 64-channel pixel per input row, 7 row taps at stride 2 -- K = 448 and twice
// the bytes; the unfolded tensor is the largest activation of the whole encoder.)
template <typename T>
__global__ void __launch_bounds__(256)
stem_pack_kernel(const T* __restrict__ rgb, int H, int W, int Wo, int J, __nv_bfloat16* __restrict__ out_hi,
                 __nv_bfloat16* __restrict__ out_lo, size_t total) {
    // one thread per (n, j, ox, group of 4 channels); 16 groups per pixel: 8 per input row, groups 5 (partly), 6, 7 are padding
    pdl_trigger();
    pdl_wait();
    for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < total; i += static_cast<size_t>(gridDim.x) * blockDim.x) {
        const int g = static_cast<int>(i & 15);
        size_t p = i >> 4;
        const int ox = static_cast<int>(p % Wo); p /= Wo;
        const int j = static_cast<int>(p % J);
        const size_t n = p / J;
        const int y = 2 * j - 3 + (g >> 3);
        __nv_bfloat16 h[4], l[4];
#pragma unroll
        for (int e = 0; e < 4; ++e) {
            const int k = (g & 7) * 4 + e;               // k = s*3 + colour
            float v = 0.f;
            if (k < 21 && y >= 0 && y < H) {
                const int s = k / 3, c = k - 3 * s;
                const int x = 2 * ox + s - 3;
                if (x >= 0 && x < W) {
                    const float raw = static_cast<float>(rgb[((n * 3 + c) * H + y) * static_cast<size_t>(W) + x]);
                    v = 2.0f * (raw / 255.0f) - 1.0f;
                }
            }
            split_bf16(v, h[e], l[e]);
        }
        *reinterpret_cast<uint2*>(out_hi + i * 4) = make_uint2(pack_bf16(h[0], h[1]), pack_bf16(h[2], h[3]));
        *reinterpret_cast<uint2*>(out_lo + i * 4) = make_uint2(pack_bf16(l[0], l[1]), pack_bf16(l[2], l[3]));
    }
}

}  // namespace pips

using namespace pips;

static unsigned grid_for(size_t total) {
    size_t b = (total + 255) / 256;
    const size_t cap = static_cast<size_t>(sm_count()) * 16;
    return static_cast<unsigned>(b < cap ? (b ? b : 1) : cap);
}

extern "C" int pips_inorm_stats(const float* y, int N, int HW, int C, float* partial, int chunks, float* stats, void* stream) {
    if (!y || !partial || !stats) return fail("pips_inorm_stats: null pointer");
    if (N <= 0 || HW <= 0 || C <= 0 || (C % 4) || C > 1024 || chunks <= 0) return fail("pips_inorm_stats: bad shape (C % 4 == 0, C <= 1024)");
    const int c4n = C / 4;
    if (c4n > 256) return fail("pips_inorm_stats: C too large");
    const int rows = 256 / c4n;
    const int chunk_px = (HW + chunks - 1) / chunks;
    const size_t smem = static_cast<size_t>(rows) * 2 * C * sizeof(float);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    cudaError_t e = launch_pdl(inorm_partial_kernel, dim3(chunks, N), dim3(256), smem, st, y, HW, C, chunk_px, partial);
    if (e == cudaSuccess) e = cudaGetLastError();
    if (e != cudaSuccess) return fail_cuda("pips_inorm_stats: partial", e);
    e = launch_pdl(inorm_finalize_kernel, dim3(N), dim3(256), 0, st, static_cast<const float*>(partial), chunks, HW, C, stats);
    if (e == cudaSuccess) e = cudaGetLastError();
    return e == cudaSuccess ? 0 : fail_cuda("pips_inorm_stats: finalize", e);
}

// statistics from per-chunk partials some other kernel produced (pips_conv_rows accumulates them in its epilogue)
extern "C" int pips_inorm_finalize(const float* partial, int N, int chunks, int HW, int C, float* stats, void* stream) {
    if (!partial || !stats) return fail("pips_inorm_finalize: null pointer");
    if (N <= 0 || HW <= 0 || C <= 0 || chunks <= 0) return fail("pips_inorm_finalize: bad shape");
    cudaError_t e = launch_pdl(inorm_finalize_kernel, dim3(N), dim3(256), 0, static_cast<cudaStream_t>(stream), partial, chunks, HW, C, stats);
    if (e == cudaSuccess) e = cudaGetLastError();
    return e == cudaSuccess ? 0 : fail_cuda("pips_inorm_finalize", e);
}

static int inorm_apply_impl(const float* y, const float* stats_y, const float* r, const float* stats_r, int relu_main, int relu_out,
                            float* out_plain, float* out_split, int split_ld, void* out_hi, void* out_lo, int pair_ld, int N, int HW,
                            int C, void* stream) {
    if (!y || (!out_plain && !out_split && !out_hi)) return fail("pips_inorm_apply: null pointer");
    if (N <= 0 || HW <= 0 || C <= 0 || (C % 4)) return fail("pips_inorm_apply: bad shape (C % 4 == 0)");
    if (out_split && (split_ld < 3 * C || (split_ld % 4))) return fail("pips_inorm_apply: split_ld must be >= 3*C and a multiple of 4");
    if (out_hi && (!out_lo || pair_ld < C || (pair_ld % 4))) return fail("pips_inorm_apply: pair output needs out_lo and pair_ld >= C, % 4 == 0");
    ApplyArgs a;
    a.y = y; a.stats_y = stats_y; a.r = r; a.stats_r = stats_r; a.relu_main = relu_main; a.relu_out = relu_out;
    a.out_plain = out_plain; a.out_split = out_split; a.split_ld = split_ld; a.HW = HW; a.C = C;
    a.out_hi = static_cast<__nv_bfloat16*>(out_hi); a.out_lo = static_cast<__nv_bfloat16*>(out_lo); a.pair_ld = pair_ld;
    const size_t total4 = static_cast<size_t>(N) * HW * ((out_hi ? pair_ld : C) / 4);
    cudaError_t e = launch_pdl(inorm_apply_kernel, dim3(grid_for(total4)), dim3(256), 0, static_cast<cudaStream_t>(stream), a, total4);
    if (e == cudaSuccess) e = cudaGetLastError();
    return e == cudaSuccess ? 0 : fail_cuda("pips_inorm_apply", e);
}

extern "C" int pips_inorm_apply(const float* y, const float* stats_y, const float* r, const float* stats_r, int relu_main,
                                int relu_out, float* out_plain, float* out_split, int split_ld, int N, int HW, int C, void* stream) {
    return inorm_apply_impl(y, stats_y, r, stats_r, relu_main, relu_out, out_plain, out_split, split_ld, nullptr, nullptr, 0, N, HW, C,
                            stream);
}

extern "C" int pips_inorm_apply_pair(const float* y, const float* stats_y, const float* r, const float* stats_r, int relu_main,
                                     int relu_out, float* out_plain, void* out_hi, void* out_lo, int pair_ld, int N, int HW, int C,
                                     void* stream) {
    if (!out_hi) return fail("pips_inorm_apply_pair: null pointer");
    return inorm_apply_impl(y, stats_y, r, stats_r, relu_main, relu_out, out_plain, nullptr, 0, out_hi, out_lo, pair_ld, N, HW, C, stream);
}

static int resize_impl(const float* src, int N, int Hs, int Ws, int C, float* dst, void* dst_hi, void* dst_lo, int Ho, int Wo, int Ctot,
                       int c_off, void* stream) {
    if (!src || (!dst && (!dst_hi || !dst_lo))) return fail("pips_resize: null pointer");
    if (N <= 0 || Hs <= 0 || Ws <= 0 || Ho <= 0 || Wo <= 0 || (C % 4) || (Ctot % 4) || (c_off % 4) || c_off + C > Ctot)
        return fail("pips_resize: bad shape");
    const int tail = (!dst && Ctot - (c_off + C) < 64) ? Ctot - (c_off + C) : 0;
    const size_t total4 = static_cast<size_t>(N) * Ho * Wo * ((C + tail) / 4);
    cudaError_t e = launch_pdl(resize_split3_kernel, dim3(grid_for(total4)), dim3(256), 0, static_cast<cudaStream_t>(stream), src, Hs, Ws, C, dst,
                               static_cast<__nv_bfloat16*>(dst_hi), static_cast<__nv_bfloat16*>(dst_lo), Ho, Wo, Ctot, c_off, total4);
    if (e == cudaSuccess) e = cudaGetLastError();
    return e == cudaSuccess ? 0 : fail_cuda("pips_resize", e);
}

extern "C" int pips_resize_split3(const float* src, int N, int Hs, int Ws, int C, float* dst, int Ho, int Wo, int Ctot, int c_off,
                                  void* stream) {
    if (!dst) return fail("pips_resize_split3: null pointer");
    return resize_impl(src, N, Hs, Ws, C, dst, nullptr, nullptr, Ho, Wo, Ctot, c_off, stream);
}

extern "C" int pips_resize_pair(const float* src, int N, int Hs, int Ws, int C, void* dst_hi, void* dst_lo, int Ho, int Wo, int Ctot,
                                int c_off, void* stream) {
    return resize_impl(src, N, Hs, Ws, C, nullptr, dst_hi, dst_lo, Ho, Wo, Ctot, c_off, stream);
}

// rgb: (N, 3, H, W) fp32 (dtype 0) or bf16 (dtype 1), values 0..255; out_hi/out_lo: (N, Ho + 3, Wo, 64) with
// Ho = (H - 1) / 2 + 1, Wo = (W - 1) / 2 + 1
extern "C" int pips_stem_pack(const void* rgb, int dtype, int N, int H, int W, void* out_hi, void* out_lo, void* stream) {
    if (!rgb || !out_hi || !out_lo) return fail("pips_stem_pack: null pointer");
    if (N <= 0 || H <= 0 || W <= 0) return fail("pips_stem_pack: empty image");
    if (dtype != 0 && dtype != 1) return fail("pips_stem_pack: dtype must be 0 (fp32) or 1 (bf16)");
    const int Wo = (W - 1) / 2 + 1, J = (H - 1) / 2 + 1 + 3;
    const size_t total = static_cast<size_t>(N) * J * Wo * 16;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    cudaError_t e0;
    if (dtype == 0)
        e0 = launch_pdl(stem_pack_kernel<float>, dim3(grid_for(total)), dim3(256), 0, st, static_cast<const float*>(rgb), H, W, Wo, J,
                        static_cast<__nv_bfloat16*>(out_hi), static_cast<__nv_bfloat16*>(out_lo), total);
    else
        e0 = launch_pdl(stem_pack_kernel<__nv_bfloat16>, dim3(grid_for(total)), dim3(256), 0, st, static_cast<const __nv_bfloat16*>(rgb), H, W, Wo, J,
                        static_cast<__nv_bfloat16*>(out_hi), static_cast<__nv_bfloat16*>(out_lo), total);
    if (e0 != cudaSuccess) return fail_cuda("pips_stem_pack", e0);
    cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? 0 : fail_cuda("pips_stem_pack", e);
}
