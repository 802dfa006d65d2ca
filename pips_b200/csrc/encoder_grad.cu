// CUDA-core parts of the feature encoder's backward (the convolutions' gradients are wgmma kernels: conv_grad.cu for
// the weights, pips_conv_tc over a flipped weight for the inputs):
//   pips_inorm_grad    InstanceNorm backward fused with the ReLU masks of pips_inorm_apply and the residual sum
//   pips_resize_grad   adjoint of pips_resize_pair (bilinear, align_corners=True) as a gather
// Per-(image, channel) sums use partials in a layout fixed by the image geometry, merged in fp64: deterministic.
#include "common.cuh"

namespace pips {

constexpr int IG_MAX_CHUNKS = 64;

struct InormGradArgs {
    const float* y; const float* stats;             // the normalised input and its (mean, rstd)
    const float* r; const float* stats_r;           // optional residual of the forward (+ its statistics)
    int relu_main, relu_out;
    const float* g0; const float* g1; const float* g2;   // upstream gradients of the forward's output, summed
    int HW, C;
};

// The forward's arithmetic (inorm_apply_kernel) for one float4: x_hat of y and the two ReLU masks.  g enters as the
// sum of the upstream gradients; on return `skip` is g masked by the output ReLU (the gradient of the residual
// branch) and g additionally masked by the main ReLU.
__device__ __forceinline__ void ig_load(const InormGradArgs& a, size_t i, int n, int c4, float4& xh, float4& g, float4& skip) {
    const float4 m = reinterpret_cast<const float4*>(a.stats + static_cast<size_t>(n) * 2 * a.C)[c4];
    const float4 s = reinterpret_cast<const float4*>(a.stats + (static_cast<size_t>(n) * 2 + 1) * a.C)[c4];
    const float4 y = reinterpret_cast<const float4*>(a.y)[i];
    xh = make_float4((y.x - m.x) * s.x, (y.y - m.y) * s.y, (y.z - m.z) * s.z, (y.w - m.w) * s.w);
    g = reinterpret_cast<const float4*>(a.g0)[i];
    if (a.g1) { const float4 b = reinterpret_cast<const float4*>(a.g1)[i]; g.x += b.x; g.y += b.y; g.z += b.z; g.w += b.w; }
    if (a.g2) { const float4 b = reinterpret_cast<const float4*>(a.g2)[i]; g.x += b.x; g.y += b.y; g.z += b.z; g.w += b.w; }
    if (a.relu_out) {
        float4 v = xh;
        if (a.relu_main) { v.x = fmaxf(v.x, 0.f); v.y = fmaxf(v.y, 0.f); v.z = fmaxf(v.z, 0.f); v.w = fmaxf(v.w, 0.f); }
        if (a.r) {
            float4 w = reinterpret_cast<const float4*>(a.r)[i];
            if (a.stats_r) {
                const float4 mr = reinterpret_cast<const float4*>(a.stats_r + static_cast<size_t>(n) * 2 * a.C)[c4];
                const float4 sr = reinterpret_cast<const float4*>(a.stats_r + (static_cast<size_t>(n) * 2 + 1) * a.C)[c4];
                w.x = (w.x - mr.x) * sr.x; w.y = (w.y - mr.y) * sr.y; w.z = (w.z - mr.z) * sr.z; w.w = (w.w - mr.w) * sr.w;
            }
            v.x += w.x; v.y += w.y; v.z += w.z; v.w += w.w;
        }
        if (!(v.x > 0.f)) g.x = 0.f;
        if (!(v.y > 0.f)) g.y = 0.f;
        if (!(v.z > 0.f)) g.z = 0.f;
        if (!(v.w > 0.f)) g.w = 0.f;
    }
    skip = g;
    if (a.relu_main) {
        if (!(xh.x > 0.f)) g.x = 0.f;
        if (!(xh.y > 0.f)) g.y = 0.f;
        if (!(xh.z > 0.f)) g.z = 0.f;
        if (!(xh.w > 0.f)) g.w = 0.f;
    }
}

// partial[(n * chunks + chunk) * 2 + {0, 1}][C] (fp64): sum of g and of g * x_hat over the chunk's pixels
__global__ void __launch_bounds__(256)
inorm_grad_partial_kernel(const InormGradArgs a, int chunk_px, double* __restrict__ partial) {
    extern __shared__ float sm[];                       // [rows][2][C]
    pdl_trigger();
    pdl_wait();
    const int c4n = a.C >> 2;
    const int lane_c = threadIdx.x % c4n, row = threadIdx.x / c4n, rows = blockDim.x / c4n;
    const int n = blockIdx.y, chunk = blockIdx.x;
    const int p0 = chunk * chunk_px, p1 = min(a.HW, p0 + chunk_px);
    if (row < rows) {
        float4 sg = make_float4(0.f, 0.f, 0.f, 0.f), sx = sg;
        for (int p = p0 + row; p < p1; p += rows) {
            const size_t i = (static_cast<size_t>(n) * a.HW + p) * c4n + lane_c;
            float4 xh, g, skip;
            ig_load(a, i, n, lane_c, xh, g, skip);
            sg.x += g.x; sg.y += g.y; sg.z += g.z; sg.w += g.w;
            sx.x = fmaf(g.x, xh.x, sx.x); sx.y = fmaf(g.y, xh.y, sx.y); sx.z = fmaf(g.z, xh.z, sx.z); sx.w = fmaf(g.w, xh.w, sx.w);
        }
        float* d = sm + (row * 2) * a.C + lane_c * 4;
        d[0] = sg.x; d[1] = sg.y; d[2] = sg.z; d[3] = sg.w;
        d[a.C + 0] = sx.x; d[a.C + 1] = sx.y; d[a.C + 2] = sx.z; d[a.C + 3] = sx.w;
    }
    __syncthreads();
    double* out = partial + (static_cast<size_t>(n) * gridDim.x + chunk) * 2 * a.C;
    for (int c = threadIdx.x; c < a.C; c += blockDim.x) {
        double s0 = 0.0, s1 = 0.0;
        for (int r = 0; r < rows; ++r) { s0 += sm[r * 2 * a.C + c]; s1 += sm[r * 2 * a.C + a.C + c]; }
        out[c] = s0;
        out[a.C + c] = s1;
    }
}

// (mean g, mean g * x_hat) per (image, channel), the chunks added in order in fp64
__global__ void inorm_grad_finalize_kernel(const double* __restrict__ partial, int chunks, int HW, int C, float* __restrict__ means) {
    pdl_trigger();
    pdl_wait();
    const int n = blockIdx.x;
    const double* pn = partial + static_cast<size_t>(n) * chunks * 2 * C;
    for (int c = threadIdx.x; c < C; c += blockDim.x) {
        double s0 = 0.0, s1 = 0.0;
        for (int k = 0; k < chunks; ++k) { s0 += pn[k * 2 * C + c]; s1 += pn[k * 2 * C + C + c]; }
        means[(static_cast<size_t>(n) * 2) * C + c] = static_cast<float>(s0 / HW);
        means[(static_cast<size_t>(n) * 2 + 1) * C + c] = static_cast<float>(s1 / HW);
    }
}

// dy = rstd * (g - mean(g) - x_hat * mean(g x_hat)) as a bf16 (hi, lo) pair of row stride pair_ld (channels [C, pair_ld)
// zero), on the (H, W) grid or zero-dilated on a (Hd, Wd) grid (pixel (y, x) at (2y, 2x), zeros elsewhere);
// optionally the skip gradient in fp32.
__global__ void __launch_bounds__(256)
inorm_grad_apply_kernel(const InormGradArgs a, const float* __restrict__ means, int W, int Hd, int Wd, int dil,
                        __nv_bfloat16* __restrict__ dy_hi, __nv_bfloat16* __restrict__ dy_lo, int pair_ld,
                        float* __restrict__ g_out, size_t total4) {
    pdl_trigger();
    pdl_wait();
    const int c4n = a.C >> 2, c4p = pair_ld >> 2;
    for (size_t j = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; j < total4; j += static_cast<size_t>(gridDim.x) * blockDim.x) {
        const int c4 = static_cast<int>(j % c4p);
        const size_t pix = j / c4p;                     // n * Hd * Wd + pixel of the output grid
        const int n = static_cast<int>(pix / (static_cast<size_t>(Hd) * Wd));
        const int q = static_cast<int>(pix - static_cast<size_t>(n) * Hd * Wd);
        const int yd = q / Wd, xd = q - yd * Wd;
        const bool src = c4 < c4n && (!dil || ((yd & 1) == 0 && (xd & 1) == 0));
        uint2 h = make_uint2(0u, 0u), l = h;
        if (src) {
            const int p = dil ? (yd >> 1) * W + (xd >> 1) : q;
            const size_t i = (static_cast<size_t>(n) * a.HW + p) * c4n + c4;
            float4 xh, g, skip;
            ig_load(a, i, n, c4, xh, g, skip);
            if (g_out) reinterpret_cast<float4*>(g_out)[i] = skip;
            const float4 mg = reinterpret_cast<const float4*>(means + static_cast<size_t>(n) * 2 * a.C)[c4];
            const float4 mx = reinterpret_cast<const float4*>(means + (static_cast<size_t>(n) * 2 + 1) * a.C)[c4];
            const float4 s = reinterpret_cast<const float4*>(a.stats + (static_cast<size_t>(n) * 2 + 1) * a.C)[c4];
            const float v0 = s.x * (g.x - mg.x - xh.x * mx.x), v1 = s.y * (g.y - mg.y - xh.y * mx.y);
            const float v2 = s.z * (g.z - mg.z - xh.z * mx.z), v3 = s.w * (g.w - mg.w - xh.w * mx.w);
            __nv_bfloat16 hh[4], ll[4];
            split_bf16(v0, hh[0], ll[0]); split_bf16(v1, hh[1], ll[1]); split_bf16(v2, hh[2], ll[2]); split_bf16(v3, hh[3], ll[3]);
            h = make_uint2(pack_bf16(hh[0], hh[1]), pack_bf16(hh[2], hh[3]));
            l = make_uint2(pack_bf16(ll[0], ll[1]), pack_bf16(ll[2], ll[3]));
        }
        const size_t o = pix * pair_ld + c4 * 4;
        *reinterpret_cast<uint2*>(dy_hi + o) = h;
        *reinterpret_cast<uint2*>(dy_lo + o) = l;
    }
}

// ---------------------------------------------------------------------------------------- resize adjoint
// The taps of destination row `o` on source rows, exactly as resize_split3_kernel computes them: weight of source row s.
__device__ __forceinline__ float tap_weight(float sc, int o, int s, int n_src) {
    const float f = sc * o;
    const int i0 = static_cast<int>(f);
    const int ip = i0 < n_src - 1 ? 1 : 0;
    const float l = f - i0;
    return (i0 == s ? 1.f - l : 0.f) + (i0 + ip == s ? l : 0.f);
}

// destination rows whose taps can touch source row s: a superset, checked exactly by tap_weight
__device__ __forceinline__ void tap_range(float sc, int s, int n_dst, int& lo, int& hi) {
    if (sc == 0.f) { lo = 0; hi = n_dst - 1; return; }
    lo = max(0, static_cast<int>(floorf((s - 1) / sc)) - 1);
    hi = min(n_dst - 1, static_cast<int>(ceilf((s + 1) / sc)) + 1);
}

__global__ void __launch_bounds__(256)
resize_grad_kernel(const float* __restrict__ g, int ldg, int c_off, int Ho, int Wo, float* __restrict__ out, int Hs, int Ws, int C,
                   size_t total4) {
    pdl_trigger();
    pdl_wait();
    const int c4n = C >> 2;
    const float sh = Ho > 1 ? static_cast<float>(Hs - 1) / static_cast<float>(Ho - 1) : 0.f;
    const float sw = Wo > 1 ? static_cast<float>(Ws - 1) / static_cast<float>(Wo - 1) : 0.f;
    for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < total4; i += static_cast<size_t>(gridDim.x) * blockDim.x) {
        const int c4 = static_cast<int>(i % c4n);
        size_t p = i / c4n;
        const int sx = static_cast<int>(p % Ws); p /= Ws;
        const int sy = static_cast<int>(p % Hs);
        const int n = static_cast<int>(p / Hs);
        int y_lo, y_hi, x_lo, x_hi;
        tap_range(sh, sy, Ho, y_lo, y_hi);
        tap_range(sw, sx, Wo, x_lo, x_hi);
        float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
        for (int oy = y_lo; oy <= y_hi; ++oy) {
            const float wy = tap_weight(sh, oy, sy, Hs);
            if (wy == 0.f) continue;
            float4 row = make_float4(0.f, 0.f, 0.f, 0.f);
            for (int ox = x_lo; ox <= x_hi; ++ox) {
                const float wx = tap_weight(sw, ox, sx, Ws);
                if (wx == 0.f) continue;
                const float4 v = *reinterpret_cast<const float4*>(g + ((static_cast<size_t>(n) * Ho + oy) * Wo + ox) * ldg + c_off + c4 * 4);
                row.x = fmaf(wx, v.x, row.x); row.y = fmaf(wx, v.y, row.y); row.z = fmaf(wx, v.z, row.z); row.w = fmaf(wx, v.w, row.w);
            }
            acc.x = fmaf(wy, row.x, acc.x); acc.y = fmaf(wy, row.y, acc.y); acc.z = fmaf(wy, row.z, acc.z); acc.w = fmaf(wy, row.w, acc.w);
        }
        reinterpret_cast<float4*>(out)[i] = acc;
    }
}

}  // namespace pips

using namespace pips;

static unsigned ig_grid(size_t total) {
    size_t b = (total + 255) / 256;
    const size_t cap = static_cast<size_t>(sm_count()) * 16;
    return static_cast<unsigned>(b < cap ? (b ? b : 1) : cap);
}

static int ig_chunks(int HW) {
    const int c = HW / 256;
    return c < 1 ? 1 : (c > IG_MAX_CHUNKS ? IG_MAX_CHUNKS : c);
}

extern "C" size_t pips_inorm_grad_scratch_floats(int N, int HW, int C) {
    if (N <= 0 || HW <= 0 || C <= 0) return 0;
    // fp64 partials (2 floats each) + the (N, 2, C) means
    return static_cast<size_t>(N) * ig_chunks(HW) * 2 * C * 2 + static_cast<size_t>(N) * 2 * C;
}

extern "C" int pips_inorm_grad(const float* y, const float* stats, const float* r, const float* stats_r, int relu_main, int relu_out,
                               const float* g0, const float* g1, const float* g2, int N, int H, int W, int C, float* scratch,
                               void* dy_hi, void* dy_lo, int pair_ld, int dil_h, int dil_w, float* g_out, void* stream) {
    if (!y || !stats || !g0 || !scratch || !dy_hi || !dy_lo) return fail("pips_inorm_grad: null pointer");
    if (N <= 0 || H <= 0 || W <= 0 || C <= 0 || (C % 4) || C > 1024) return fail("pips_inorm_grad: bad shape (C % 4 == 0, C <= 1024)");
    if (pair_ld < C || (pair_ld % 4)) return fail("pips_inorm_grad: pair_ld must be >= C and a multiple of 4");
    if (stats_r && !r) return fail("pips_inorm_grad: stats_r without r");
    if (r && !relu_out) return fail("pips_inorm_grad: a residual only changes the output ReLU's mask (relu_out)");
    const bool dil = dil_h != 0 || dil_w != 0;
    if (dil && ((dil_h + 1) / 2 != H || (dil_w + 1) / 2 != W || dil_h <= 0 || dil_w <= 0))
        return fail("pips_inorm_grad: the dilated grid must be (2H or 2H-1, 2W or 2W-1)");
    const int HW = H * W;
    const int chunks = ig_chunks(HW);
    InormGradArgs a;
    a.y = y; a.stats = stats; a.r = r; a.stats_r = stats_r; a.relu_main = relu_main; a.relu_out = relu_out;
    a.g0 = g0; a.g1 = g1; a.g2 = g2; a.HW = HW; a.C = C;
    double* partial = reinterpret_cast<double*>(scratch);
    if (reinterpret_cast<uintptr_t>(scratch) & 15) return fail("pips_inorm_grad: scratch must be 16-byte aligned");
    float* means = scratch + static_cast<size_t>(N) * chunks * 2 * C * 2;
    const int c4n = C / 4;
    const int rows = 256 / c4n;
    const size_t smem = static_cast<size_t>(rows) * 2 * C * sizeof(float);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    cudaError_t e = launch_pdl(inorm_grad_partial_kernel, dim3(chunks, N), dim3(256), smem, st, a, (HW + chunks - 1) / chunks, partial);
    if (e == cudaSuccess) e = cudaGetLastError();
    if (e != cudaSuccess) return fail_cuda("pips_inorm_grad: partial", e);
    e = launch_pdl(inorm_grad_finalize_kernel, dim3(N), dim3(256), 0, st, static_cast<const double*>(partial), chunks, HW, C, means);
    if (e == cudaSuccess) e = cudaGetLastError();
    if (e != cudaSuccess) return fail_cuda("pips_inorm_grad: finalize", e);
    const int Hd = dil ? dil_h : H, Wd = dil ? dil_w : W;
    const size_t total4 = static_cast<size_t>(N) * Hd * Wd * (pair_ld / 4);
    e = launch_pdl(inorm_grad_apply_kernel, dim3(ig_grid(total4)), dim3(256), 0, st, a, static_cast<const float*>(means), W, Hd, Wd,
                   dil ? 1 : 0, static_cast<__nv_bfloat16*>(dy_hi), static_cast<__nv_bfloat16*>(dy_lo), pair_ld, g_out, total4);
    if (e == cudaSuccess) e = cudaGetLastError();
    return e == cudaSuccess ? 0 : fail_cuda("pips_inorm_grad: apply", e);
}

extern "C" int pips_resize_grad(const float* g, int ldg, int c_off, int N, int Ho, int Wo, float* out, int Hs, int Ws, int C,
                                void* stream) {
    if (!g || !out) return fail("pips_resize_grad: null pointer");
    if (N <= 0 || Ho <= 0 || Wo <= 0 || Hs <= 0 || Ws <= 0 || C <= 0 || (C % 4) || (ldg % 4) || (c_off % 4) || c_off < 0 || c_off + C > ldg)
        return fail("pips_resize_grad: bad shape (C, ldg, c_off multiples of 4, c_off + C <= ldg)");
    const size_t total4 = static_cast<size_t>(N) * Hs * Ws * (C / 4);
    cudaError_t e = launch_pdl(resize_grad_kernel, dim3(ig_grid(total4)), dim3(256), 0, static_cast<cudaStream_t>(stream), g, ldg, c_off,
                               Ho, Wo, out, Hs, Ws, C, total4);
    if (e == cudaSuccess) e = cudaGetLastError();
    return e == cudaSuccess ? 0 : fail_cuda("pips_resize_grad", e);
}
