// CUDA-core parts of the DeltaBlock mixer's backward (the dense layers' gradients are wgmma GEMMs, gemm_tc.cu):
//   pips_tokenmix_grad   LN2 backward -> token-mixing MLP backward -> LN1 backward, one sequence (8 x 512) per step
//   pips_ln_pool_grad    mean over S + final LayerNorm backward
//   pips_colsum          fixed-order column sums: bias gradients, and the reduction of every per-CTA partial row
// Parameter gradients are summed without atomics: each CTA owns a partial row, and pips_colsum adds the rows in order.
#include "mixer_common.cuh"

namespace pips {

constexpr int CS_ROWS = 256;          // rows per split of a column sum
constexpr int TG_SEQS = 8;            // sequences per CTA of the backward kernels: the partial rows stay few
constexpr int TG_PARAMS = 2600;       // ln1_w ln1_b tok_w1 tok_b1 tok_w2 tok_b2 ln2_w ln2_b
constexpr int LP_PARAMS = 1024;       // ln_w ln_b

// out[y * N + n] = sum of rows [y * rows_per, min(M, (y + 1) * rows_per)) of column n; fp32 g or the pair hi + lo
__global__ void __launch_bounds__(256)
colsum_kernel(const float* __restrict__ g, const __nv_bfloat16* __restrict__ hi, const __nv_bfloat16* __restrict__ lo, size_t ld,
              int M, int N, int rows_per, float* __restrict__ out) {
    const int n = blockIdx.x * 256 + threadIdx.x;
    if (n >= N) return;
    const int r0 = blockIdx.y * rows_per;
    const int r1 = min(M, r0 + rows_per);
    float a = 0.0f;
    for (int m = r0; m < r1; ++m) {
        const size_t i = static_cast<size_t>(m) * ld + n;
        a += g ? g[i] : __bfloat162float(hi[i]) + (lo ? __bfloat162float(lo[i]) : 0.0f);
    }
    out[static_cast<size_t>(blockIdx.y) * N + n] = a;
}

size_t colsum_scratch(int M, int N) {
    const int splits = (M + CS_ROWS - 1) / CS_ROWS;
    return splits > 1 ? static_cast<size_t>(splits) * N : 0;
}

int colsum_launch(const float* g, const void* g_hi, const void* g_lo, size_t ld, int M, int N, float* scratch, float* out,
                  cudaStream_t st) {
    const int splits = (M + CS_ROWS - 1) / CS_ROWS;
    const dim3 grid((N + 255) / 256, splits);
    colsum_kernel<<<grid, 256, 0, st>>>(g, static_cast<const __nv_bfloat16*>(g_hi), static_cast<const __nv_bfloat16*>(g_lo), ld, M, N,
                                         CS_ROWS, splits > 1 ? scratch : out);
    if (splits > 1) colsum_kernel<<<dim3((N + 255) / 256, 1), 256, 0, st>>>(scratch, nullptr, nullptr, N, splits, N, splits, out);
    cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? 0 : fail_cuda("pips_colsum", e);
}

namespace {

// row statistics of layernorm8 (mixer_common.cuh), the same arithmetic: mean and 1/sqrt(var + 1e-5) of the 8 rows
__device__ __forceinline__ void ln_stats8(const float (&x)[8][4], float (&m)[8], float (&r)[8], float (*red)[8]) {
    float q[8];
#pragma unroll
    for (int s = 0; s < 8; ++s) m[s] = (x[s][0] + x[s][1]) + (x[s][2] + x[s][3]);
    block_sum8(m, red);
#pragma unroll
    for (int s = 0; s < 8; ++s) {
        m[s] *= (1.0f / 512.0f);
        const float d0 = x[s][0] - m[s], d1 = x[s][1] - m[s], d2 = x[s][2] - m[s], d3 = x[s][3] - m[s];
        q[s] = (d0 * d0 + d1 * d1) + (d2 * d2 + d3 * d3);
    }
    block_sum8(q, red);
#pragma unroll
    for (int s = 0; s < 8; ++s) r[s] = rsqrtf(q[s] * (1.0f / 512.0f) + 1e-5f);
}

// LayerNorm backward of the 8 rows: dx += r (g dy - mean(g dy) - xh mean(g dy xh)), xh = (x - m) r; dgam += dy xh, dbet += dy
__device__ __forceinline__ void ln_backward8(const float (&x)[8][4], const float (&m)[8], const float (&r)[8], const float (&dy)[8][4],
                                             const float4 gam, float (&dgam)[4], float (&dbet)[4], float (&dx)[8][4], float (*red)[8]) {
    const float g[4] = {gam.x, gam.y, gam.z, gam.w};
    float a[8], b[8], xh[8][4];
#pragma unroll
    for (int s = 0; s < 8; ++s) {
        a[s] = b[s] = 0.0f;
#pragma unroll
        for (int c = 0; c < 4; ++c) {
            xh[s][c] = (x[s][c] - m[s]) * r[s];
            const float gd = dy[s][c] * g[c];
            dgam[c] = fmaf(dy[s][c], xh[s][c], dgam[c]);
            dbet[c] += dy[s][c];
            a[s] += gd;
            b[s] = fmaf(gd, xh[s][c], b[s]);
        }
    }
    block_sum8(a, red);
    block_sum8(b, red);
#pragma unroll
    for (int s = 0; s < 8; ++s) {
        const float ma = a[s] * (1.0f / 512.0f), mb = b[s] * (1.0f / 512.0f);
#pragma unroll
        for (int c = 0; c < 4; ++c) dx[s][c] += r[s] * (dy[s][c] * g[c] - ma - xh[s][c] * mb);
    }
}

__device__ __forceinline__ void load_rows(const float* p, size_t base, float (&v)[8][4]) {
#pragma unroll
    for (int s = 0; s < 8; ++s) {
        const float4 t = *reinterpret_cast<const float4*>(p + base + s * 512);
        v[s][0] = t.x; v[s][1] = t.y; v[s][2] = t.z; v[s][3] = t.w;
    }
}

// warp sum of 16 values at once: after the halving butterfly, lane L holds the sum over the warp of value
// 8 b4 + 4 b3 + 2 b2 + b1 (b_i = bit i of L); 16 shuffles instead of 80.  Each sum is formed in one fixed order.
__device__ __forceinline__ float warp_sum16(const float (&v)[16], int lane) {
    float w[8], x[4], y[2];
    const bool u4 = lane & 16, u3 = lane & 8, u2 = lane & 4, u1 = lane & 2;
#pragma unroll
    for (int i = 0; i < 8; ++i) w[i] = (u4 ? v[i + 8] : v[i]) + __shfl_xor_sync(0xffffffffu, u4 ? v[i] : v[i + 8], 16);
#pragma unroll
    for (int i = 0; i < 4; ++i) x[i] = (u3 ? w[i + 4] : w[i]) + __shfl_xor_sync(0xffffffffu, u3 ? w[i] : w[i + 4], 8);
#pragma unroll
    for (int i = 0; i < 2; ++i) y[i] = (u2 ? x[i + 2] : x[i]) + __shfl_xor_sync(0xffffffffu, u2 ? x[i] : x[i + 2], 4);
    const float z = (u1 ? y[1] : y[0]) + __shfl_xor_sync(0xffffffffu, u1 ? y[0] : y[1], 2);
    return z + __shfl_xor_sync(0xffffffffu, z, 1);
}

// One CTA of 128 threads runs TG_SEQS sequences one after the other; thread t owns channels 4t..4t+3 of the 8 rows.
// Token mixing is independent per channel: u = LN1(x_in) (8 values), h_j = b1_j + sum_s w1[j,s] u_s, a_j = gelu(h_j),
// z_s = b2_s + sum_j w2[s,j] a_j.  With dz = dL/dx_mid:
//   dw2[s,j] += dz_s a_j   db2 += dz   dh_j = gelu'(h_j) sum_s w2[s,j] dz_s   dw1[j,s] += dh_j u_s   db1 += dh   du_s = sum_j w1[j,s] dh_j
// The hidden layer is recomputed in registers, one j at a time.  The per-channel products are summed over the warp
// (warp_sum16) and accumulated in shared memory per warp; the CTA's partial row is written at the end.
// Registers: the per-thread rows xv, dz, u, du ([8][4] each) and v[16] put this kernel at 255 registers with 16 bytes
// of spill (ptxas, CUDA 12.9).  Any further per-thread state spills more: stage it in shared memory instead.
__global__ void __launch_bounds__(TM_THREADS)
tokenmix_grad_kernel(const float* __restrict__ x_in, const float* __restrict__ x_mid, const float* __restrict__ dy, float* dx, int seqs,
                     const float* __restrict__ ln1_w, const float* __restrict__ ln1_b, const float* __restrict__ w1,
                     const float* __restrict__ b1, const float* __restrict__ w2, const float* __restrict__ ln2_w,
                     float* __restrict__ partial) {
    __shared__ float red[4][8];
    __shared__ float s_w1[32 * 8], s_w2[8 * 32], s_b1[32];
    __shared__ float s_tok[4][32][16];          // per warp: [j][s] = dw2[s,j], [j][8 + s] = dw1[j,s]
    __shared__ float s_db1[4][32], s_db2[4][8];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    for (int i = threadIdx.x; i < 256; i += TM_THREADS) {
        s_w1[i] = w1[i];
        s_w2[i] = w2[i];
        (&s_tok[0][0][0])[i] = 0.0f;
        (&s_tok[0][0][0])[i + 256] = 0.0f;
        (&s_tok[0][0][0])[i + 512] = 0.0f;
        (&s_tok[0][0][0])[i + 768] = 0.0f;
        (&s_tok[0][0][0])[i + 1024] = 0.0f;
        (&s_tok[0][0][0])[i + 1280] = 0.0f;
        (&s_tok[0][0][0])[i + 1536] = 0.0f;
        (&s_tok[0][0][0])[i + 1792] = 0.0f;
    }
    if (threadIdx.x < 32) s_b1[threadIdx.x] = b1[threadIdx.x];
    s_db1[warp][lane] = 0.0f;
    if (lane < 8) s_db2[warp][lane] = 0.0f;
    const float4 g1 = *reinterpret_cast<const float4*>(ln1_w + threadIdx.x * 4);
    const float4 c1 = *reinterpret_cast<const float4*>(ln1_b + threadIdx.x * 4);
    const float4 g2 = *reinterpret_cast<const float4*>(ln2_w + threadIdx.x * 4);
    const float gg1[4] = {g1.x, g1.y, g1.z, g1.w}, cc1[4] = {c1.x, c1.y, c1.z, c1.w};
    float d_ln1w[4] = {}, d_ln1b[4] = {}, d_ln2w[4] = {}, d_ln2b[4] = {};
    __syncthreads();

    const int q0 = blockIdx.x * TG_SEQS, q1 = min(seqs, q0 + TG_SEQS);
    for (int q = q0; q < q1; ++q) {
        const size_t base = static_cast<size_t>(q) * 8 * 512 + threadIdx.x * 4;
        float xv[8][4], dz[8][4], m[8], r[8];
        {
            float gy[8][4];
            load_rows(x_mid, base, xv);
            load_rows(dy, base, gy);
            load_rows(dx, base, dz);
            ln_stats8(xv, m, r, red);
            ln_backward8(xv, m, r, gy, g2, d_ln2w, d_ln2b, dz, red);           // dz = dL/dx_mid
        }
        load_rows(x_in, base, xv);
        ln_stats8(xv, m, r, red);
        float u[8][4], du[8][4];
#pragma unroll
        for (int s = 0; s < 8; ++s)
#pragma unroll
            for (int c = 0; c < 4; ++c) {
                u[s][c] = (xv[s][c] - m[s]) * r[s] * gg1[c] + cc1[c];
                du[s][c] = 0.0f;
            }
#pragma unroll
        for (int s = 0; s < 8; ++s) {
            const float p = warp_sum((dz[s][0] + dz[s][1]) + (dz[s][2] + dz[s][3]));
            if (lane == 0) s_db2[warp][s] += p;
        }
#pragma unroll 1
        for (int j = 0; j < 32; ++j) {
            float w1j[8], w2j[8];
#pragma unroll
            for (int s = 0; s < 8; ++s) { w1j[s] = s_w1[j * 8 + s]; w2j[s] = s_w2[s * 32 + j]; }
            float v[16], vb = 0.0f;
#pragma unroll
            for (int i = 0; i < 16; ++i) v[i] = 0.0f;
#pragma unroll
            for (int c = 0; c < 4; ++c) {
                float h = s_b1[j], da = 0.0f;
#pragma unroll
                for (int s = 0; s < 8; ++s) {
                    h = fmaf(w1j[s], u[s][c], h);
                    da = fmaf(w2j[s], dz[s][c], da);
                }
                const float a = gelu_exact(h);
                const float dh = da * gelu_grad_exact(h);
                vb += dh;
#pragma unroll
                for (int s = 0; s < 8; ++s) {
                    v[s] = fmaf(dz[s][c], a, v[s]);
                    v[8 + s] = fmaf(dh, u[s][c], v[8 + s]);
                    du[s][c] = fmaf(w1j[s], dh, du[s][c]);
                }
            }
            const float t = warp_sum16(v, lane);
            if (!(lane & 1)) s_tok[warp][j][((lane >> 4) & 1) * 8 + ((lane >> 3) & 1) * 4 + ((lane >> 2) & 1) * 2 + ((lane >> 1) & 1)] += t;
            vb = warp_sum(vb);
            if (lane == 0) s_db1[warp][j] += vb;
        }
        ln_backward8(xv, m, r, du, g1, d_ln1w, d_ln1b, dz, red);               // dz = dL/dx_in
#pragma unroll
        for (int s = 0; s < 8; ++s)
            *reinterpret_cast<float4*>(dx + base + s * 512) = make_float4(dz[s][0], dz[s][1], dz[s][2], dz[s][3]);
    }
    __syncthreads();
    float* out = partial + static_cast<size_t>(blockIdx.x) * TG_PARAMS;
#pragma unroll
    for (int c = 0; c < 4; ++c) {
        const int ch = threadIdx.x * 4 + c;
        out[ch] = d_ln1w[c];
        out[512 + ch] = d_ln1b[c];
        out[1576 + ch] = d_ln2w[c];
        out[2088 + ch] = d_ln2b[c];
    }
    for (int i = threadIdx.x; i < 256; i += TM_THREADS) {
        const int j = i >> 3, s = i & 7;
        out[1024 + i] = ((s_tok[0][j][8 + s] + s_tok[1][j][8 + s]) + s_tok[2][j][8 + s]) + s_tok[3][j][8 + s];   // tok_w1[j][s]
        const int s2 = i >> 5, j2 = i & 31;
        out[1312 + i] = ((s_tok[0][j2][s2] + s_tok[1][j2][s2]) + s_tok[2][j2][s2]) + s_tok[3][j2][s2];             // tok_w2[s][j]
    }
    if (threadIdx.x < 32) out[1280 + threadIdx.x] = ((s_db1[0][threadIdx.x] + s_db1[1][threadIdx.x]) + s_db1[2][threadIdx.x]) + s_db1[3][threadIdx.x];
    if (threadIdx.x < 8) out[1568 + threadIdx.x] = ((s_db2[0][threadIdx.x] + s_db2[1][threadIdx.x]) + s_db2[2][threadIdx.x]) + s_db2[3][threadIdx.x];
}

// pips_ln_pool's backward: every one of the 8 rows receives dp / 8, then the LayerNorm backward
__global__ void __launch_bounds__(TM_THREADS)
ln_pool_grad_kernel(const float* __restrict__ x, const float* __restrict__ dp, int seqs, const float* __restrict__ ln_w,
                    float* __restrict__ dx, float* __restrict__ partial) {
    __shared__ float red[4][8];
    const float4 g = *reinterpret_cast<const float4*>(ln_w + threadIdx.x * 4);
    float dw[4] = {}, db[4] = {};
    const int q0 = blockIdx.x * TG_SEQS, q1 = min(seqs, q0 + TG_SEQS);
    for (int q = q0; q < q1; ++q) {
        const size_t base = static_cast<size_t>(q) * 8 * 512 + threadIdx.x * 4;
        float xv[8][4], gy[8][4], out[8][4], m[8], r[8];
        load_rows(x, base, xv);
        const float4 p = *reinterpret_cast<const float4*>(dp + static_cast<size_t>(q) * 512 + threadIdx.x * 4);
#pragma unroll
        for (int s = 0; s < 8; ++s) {
            gy[s][0] = p.x * 0.125f; gy[s][1] = p.y * 0.125f; gy[s][2] = p.z * 0.125f; gy[s][3] = p.w * 0.125f;
            out[s][0] = out[s][1] = out[s][2] = out[s][3] = 0.0f;
        }
        ln_stats8(xv, m, r, red);
        ln_backward8(xv, m, r, gy, g, dw, db, out, red);
#pragma unroll
        for (int s = 0; s < 8; ++s)
            *reinterpret_cast<float4*>(dx + base + s * 512) = make_float4(out[s][0], out[s][1], out[s][2], out[s][3]);
    }
    float* o = partial + static_cast<size_t>(blockIdx.x) * LP_PARAMS;
#pragma unroll
    for (int c = 0; c < 4; ++c) {
        o[threadIdx.x * 4 + c] = dw[c];
        o[512 + threadIdx.x * 4 + c] = db[c];
    }
}

int grad_ctas(int seqs) { return (seqs + TG_SEQS - 1) / TG_SEQS; }

bool misaligned16(const void* p) { return reinterpret_cast<uintptr_t>(p) & 15; }

}  // namespace
}  // namespace pips

using namespace pips;

extern "C" size_t pips_colsum_scratch_floats(int M, int N) {
    return (M > 0 && N > 0) ? colsum_scratch(M, N) : 0;
}

extern "C" int pips_colsum(const float* g, const void* g_hi, const void* g_lo, size_t ld, int M, int N, float* scratch, float* out,
                           void* stream) {
    if ((!g && !g_hi) || !out) return fail("pips_colsum: null pointer");
    if (M <= 0 || N <= 0) return fail("pips_colsum: empty problem");
    if (ld < static_cast<size_t>(N)) return fail("pips_colsum: ld must be >= N");
    if (colsum_scratch(M, N) > 0 && !scratch) return fail("pips_colsum: scratch of pips_colsum_scratch_floats(M, N) floats is required");
    return colsum_launch(g, g_hi, g_lo, ld, M, N, scratch, out, static_cast<cudaStream_t>(stream));
}

extern "C" size_t pips_tokenmix_grad_scratch_floats(int seqs) {
    if (seqs <= 0) return 0;
    const int rows = grad_ctas(seqs);
    return static_cast<size_t>(rows) * TG_PARAMS + colsum_scratch(rows, TG_PARAMS);
}

extern "C" int pips_tokenmix_grad(const float* x_in, const float* x_mid, const float* dy, float* dx, int seqs, const float* ln1_w,
                                  const float* ln1_b, const float* w1, const float* b1, const float* w2, const float* b2,
                                  const float* ln2_w, const float* ln2_b, float* scratch, float* grads, void* stream) {
    if (!x_in || !x_mid || !dy || !dx || !ln1_w || !ln1_b || !w1 || !b1 || !w2 || !b2 || !ln2_w || !ln2_b || !scratch || !grads)
        return fail("pips_tokenmix_grad: null pointer");
    if (seqs <= 0) return fail("pips_tokenmix_grad: no sequences");
    if (misaligned16(x_in) || misaligned16(x_mid) || misaligned16(dy) || misaligned16(dx) || misaligned16(ln1_w)
        || misaligned16(ln1_b) || misaligned16(ln2_w))
        return fail("pips_tokenmix_grad: x_in, x_mid, dy, dx and the LayerNorm parameters must be 16-byte aligned");
    const int ctas = grad_ctas(seqs);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    tokenmix_grad_kernel<<<ctas, TM_THREADS, 0, st>>>(x_in, x_mid, dy, dx, seqs, ln1_w, ln1_b, w1, b1, w2, ln2_w, scratch);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return fail_cuda("pips_tokenmix_grad", e);
    const size_t part = static_cast<size_t>(ctas) * TG_PARAMS;
    return colsum_launch(scratch, nullptr, nullptr, TG_PARAMS, ctas, TG_PARAMS, scratch + part, grads, st);
}

extern "C" size_t pips_ln_pool_grad_scratch_floats(int seqs) {
    if (seqs <= 0) return 0;
    const int rows = grad_ctas(seqs);
    return static_cast<size_t>(rows) * LP_PARAMS + colsum_scratch(rows, LP_PARAMS);
}

extern "C" int pips_ln_pool_grad(const float* x, const float* dp, int seqs, const float* ln_w, const float* ln_b, float* dx,
                                 float* scratch, float* grads, void* stream) {
    if (!x || !dp || !ln_w || !ln_b || !dx || !scratch || !grads) return fail("pips_ln_pool_grad: null pointer");
    if (seqs <= 0) return fail("pips_ln_pool_grad: no sequences");
    if (misaligned16(x) || misaligned16(dp) || misaligned16(dx) || misaligned16(ln_w))
        return fail("pips_ln_pool_grad: x, dp, dx and ln_w must be 16-byte aligned");
    const int ctas = grad_ctas(seqs);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    ln_pool_grad_kernel<<<ctas, TM_THREADS, 0, st>>>(x, dp, seqs, ln_w, dx, scratch);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return fail_cuda("pips_ln_pool_grad", e);
    const size_t part = static_cast<size_t>(ctas) * LP_PARAMS;
    return colsum_launch(scratch, nullptr, nullptr, LP_PARAMS, ctas, LP_PARAMS, scratch + part, grads, st);
}
