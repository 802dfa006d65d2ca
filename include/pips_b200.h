/* pips_b200 -- C ABI of the H100-native PIPs refinement hot path.
 *
 * The reference (aharley/pips) has no FFI / plugin registry: its boundary is the Python class
 * nets.pips.Pips (nets/pips.py:400-611).  This header is what a reference-side binding (ctypes,
 * see INTEGRATION.md) calls instead of the torch ops inside Pips.forward's refinement loop
 * (nets/pips.py:459-559).  Every entry point:
 *   - takes plain device pointers, sizes and a CUDA stream handle (cudaStream_t as void*),
 *   - launches asynchronously on that stream, never allocates device memory, never synchronises,
 *   - returns 0 on success, non-zero on error with the message available from pips_last_error().
 * All tensors are contiguous unless a leading dimension is given.  The feature dimension is 128
 * (nets/pips.py:408).  S (frames per window, the model's constructor argument, nets/pips.py:401) is 8 for the
 * entry points without an S of their own, for the mixer's training kernels and for chained tracking; the inference
 * entry points (pips_refine_iter, pips_corr_gather, pips_init_gather, pips_update, pips_vis_head, pips_heatmap) and the
 * _s / _window siblings, including those of the correlation and score-map gradients, take any 2 <= S <= PIPS_S_MAX.  Sizes that depend on S: the head GEMM's N = PIPS_HEAD_N(S) = 130*S,
 * padded to PIPS_HEAD_PAD(S) rows (a multiple of 256).
 *
 * Layouts
 *   fmaps        (B*S, 128, H8, W8) fp32 NCHW              output of fnet           nets/pips.py:444-445
 *   pyramid      4 levels, (B*S, H_l, W_l, 128) NHWC       avg-pool chain           nets/pips.py:346-352
 *   coords       (B, S, N, 2) fp32, feature-map pixels     loop state               nets/pips.py:453
 *   ffeats       (B*N, S, 128) fp32                        loop state               nets/pips.py:466,:522
 *   mixer rows   r = (b*N + n)*S + s                       the "(B*N, S, C)" order  nets/pips.py:516-522
 */
#ifndef PIPS_B200_H
#define PIPS_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define PIPS_B200_ABI_VERSION 4

enum { PIPS_S = 8, PIPS_C = 128, PIPS_LEVELS = 4, PIPS_RADIUS = 3 };
enum { PIPS_S_MAX = 16 };   /* longest window of the inference entry points (S = 2..16) */
#define PIPS_HEAD_N(S) (130 * (S))
#define PIPS_HEAD_PAD(S) ((130 * (S) + 255) / 256 * 256)
/* row stride of delta: 130*S rounded up to a multiple of 4 floats (the head GEMM's fp32 epilogue stores 16-byte
 * vectors); 130*S for even S */
#define PIPS_DELTA_LD(S) ((130 * (S) + 3) / 4 * 4)
enum { PIPS_KITCHEN = 519, PIPS_KITCHEN_PAD = 576, PIPS_DIM = 512, PIPS_HIDDEN = 2048, PIPS_DEPTH = 12, PIPS_HEAD = 1040 };

/* storage type of the correlation pyramid */
enum { PIPS_FEAT_F32 = 0, PIPS_FEAT_BF16 = 1 };
/* arithmetic of the mixer's dense layers */
enum { PIPS_PREC_F32 = 0,      /* fp32 CUDA-core GEMMs (exact; validation / small problems)            */
       PIPS_PREC_BF16X3 = 1,   /* wgmma,   operands split hi+lo bf16, 3 MMAs per product (~fp32)       */
       PIPS_PREC_BF16 = 2 };   /* wgmma,   plain bf16 operands (fast mode, does not meet 1e-3 px)      */
/* GEMM epilogues */
enum { PIPS_EPI_BIAS = 0,        /* out_f32 = acc + bias                                              */
       PIPS_EPI_BIAS_GELU = 1,   /* out    = gelu_erf(acc + bias)  (bf16 hi[/lo] or fp32)             */
       PIPS_EPI_BIAS_RESID = 2,  /* out_f32 += acc + bias                                             */
       PIPS_EPI_BIAS_GELU_PRE = 3, /* BIAS_GELU into bf16 hi[/lo], and aux = acc + bias (fp32)         */
       PIPS_EPI_GELU_GRAD = 4 }; /* out = (acc + bias) * gelu_erf'(aux), bf16 hi[/lo]                 */

int pips_abi_version(void);
const char* pips_last_error(void);

/* nets/pips.py:346-352 (CorrBlock.__init__): NCHW fp32 fmaps -> 4-level channels-last pyramid.
 * lvl_f32[l] are always written (level 0 is the transposed input); lvl_bf16[l], when the array is
 * non-NULL, receive the same values rounded to bf16. */
int pips_pyramid_build(const float* fmaps_nchw, int frames, int H, int W,
                       float* const* lvl_f32, void* const* lvl_bf16, void* stream);
/* same, for feature maps that are already channels-last (B*S, H, W, 128) -- what the fused encoder path emits */
int pips_pyramid_build_nhwc(const float* fmaps_nhwc, int frames, int H, int W,
                            float* const* lvl_f32, void* const* lvl_bf16, void* stream);

/* utils/samp.py:5-78 via nets/pips.py:463-466: bilinear gather of frame 0 at the query (indices
 * clamped, weights not), broadcast over S.  coords is the full (B,S,N,2) state (frame 0 is read).  With frame_base
 * (chained tracking) "frame 0" is the first frame of track (b,n)'s window, decoded as in pips_corr_gather: frame
 * min(base, T-1) of clip b for base >= 0, min(~base, T-1) for a backward window (base < 0). */
int pips_init_gather(const float* lvl0_f32, int B, int S, int N, int H, int W, const float* coords,
                     const int* frame_base /* NULL or [B*N] */, int frames_per_batch,
                     float* ffeat /* (B*N,128) */, float* ffeats /* (B*N,S,128) */, void* stream);
/* pips_init_gather with a per-track clip table (several videos in one pyramid), decoded as in pips_corr_gather_clips. */
int pips_init_gather_clips(const float* lvl0_f32, int B, int S, int N, int H, int W, const float* coords,
                           const int* frame_base /* [B*N] */, int frames_per_batch, const int* clip /* NULL or [B*N][2] */,
                           float* ffeat /* (B*N,128) */, float* ffeats /* (B*N,S,128) */, void* stream);

/* nets/pips.py:502,:513 (CorrBlock.corr + .sample) fused with the layout glue :517-522 and
 * utils/misc.py:44-69 (get_3d_embedding): writes the 519-wide mixer input row
 *   [ ffeat 128 | corr 4x49 | sin/cos(flow_x) 64 | (flow_y) 64 | (t) 64 | flow_x flow_y t | 0-pad to 576 ]
 * for every (b,n,s) without materialising the all-pairs volume.  Any of x_hi/x_lo/x_f32 may be NULL.
 * Chained long-video tracking (chain_demo.py:40-83): when frame_base is non-NULL the pyramid holds
 * frames_per_batch (T) frames per batch element and track (b,n) with base = frame_base[b*N+n] reads, at step s,
 * frame min(base + s, T-1) when base >= 0 (a forward window), and frame max(t - s, 0) with t = min(~base, T-1) when
 * base < 0 (a backward window from frame t: the chain on the time-reversed clip). */
int pips_corr_gather(const void* const* lvl, int feat_dtype, int B, int S, int N, int H, int W,
                     const float* coords, const float* ffeats, const float* times /* [S] */,
                     const int* frame_base /* NULL or [B*N] */, int frames_per_batch,
                     void* x_hi, void* x_lo, float* x_f32, int ldx, void* stream);
/* pips_corr_gather with a per-track clip table: several clips of different lengths concatenated in one pyramid of
 * B * frames_per_batch frames (frames_per_batch still sizes the tensor maps).  clip[b*N+n] = {first, count} (int32
 * pairs): the first pyramid frame of track (b,n)'s clip and its number of frames, count >= 1 and first + count <=
 * B * frames_per_batch (not checked: the kernels trust the table).  Step s then reads pyramid frame
 *   first + min(base + s, count-1)             for base >= 0 (forward: the clip's last frame is replicated)
 *   first + max(min(~base, count-1) - s, 0)    for base <  0 (backward: clamped at the clip's frame 0)
 * with base = frame_base[b*N+n] counted inside the clip, so a window never reads another clip's frames.  A clip table
 * requires frame_base (an error otherwise); clip == NULL is pips_corr_gather. */
int pips_corr_gather_clips(const void* const* lvl, int feat_dtype, int B, int S, int N, int H, int W,
                           const float* coords, const float* ffeats, const float* times /* [S] */,
                           const int* frame_base /* [B*N] */, int frames_per_batch, const int* clip /* NULL or [B*N][2] */,
                           void* x_hi, void* x_lo, float* x_f32, int ldx, void* stream);

/* Several pyramids of different map sizes in one call (videos of different frame sizes tracked together): group g
 * holds frames[g] frames whose level 0 is H[g] x W[g] (at least 8 x 8); lvl[g][l] is its level l, channels-last
 * (frames[g], H[g] >> l, W[g] >> l, 128), in the storage type the entry point names.  1 <= G <= PIPS_MAX_GROUPS. */
#define PIPS_MAX_GROUPS 32
typedef struct pips_groups {
    int G;
    const void* lvl[PIPS_MAX_GROUPS][PIPS_LEVELS];
    int H[PIPS_MAX_GROUPS], W[PIPS_MAX_GROUPS];   /* level 0 */
    int frames[PIPS_MAX_GROUPS];
} pips_groups;

/* pips_corr_gather_clips over the pyramids of `groups` (levels in feat_dtype): table[b*N+n] = {first, count, group, 0}
 * (int32, 16 bytes per track) names the pyramid group of track (b,n) and its clip {first, count} among that group's
 * frames, decoded as in pips_corr_gather_clips; the window's boxes, clamps and taps use the group's map sizes.
 * 0 <= group < G, count >= 1, first + count <= frames[group] (not checked: the kernels trust the table).  frame_base
 * and the table are required. */
int pips_corr_gather_groups(const pips_groups* groups, int feat_dtype, int B, int S, int N,
                            const float* coords, const float* ffeats, const float* times /* [S] */,
                            const int* frame_base /* [B*N] */, const int* table /* [B*N][4] */,
                            void* x_hi, void* x_lo, float* x_f32, int ldx, void* stream);
/* pips_init_gather_clips over the pyramids of `groups`, decoded as in pips_corr_gather_groups: lvl[g][0] is read as
 * group g's fp32 level 0 (the other levels are not read and may be NULL). */
int pips_init_gather_groups(const pips_groups* groups, int B, int S, int N, const float* coords,
                            const int* frame_base /* [B*N] */, const int* table /* [B*N][4] */,
                            float* ffeat /* (B*N,128) */, float* ffeats /* (B*N,S,128) */, void* stream);

/* Backward of pips_corr_gather's correlation columns (x[:, 128:324]) for training (csrc/corr_grad.cu), with respect to
 * the ffeats and the 4 fp32 levels; the coordinates get no gradient.  S == 8 (the _window siblings below take
 * 2 <= S <= PIPS_S_MAX), fp32, no frame_base.  dcorr is the
 * gradient of those 196 columns, (B*N*S, ld_dcorr) in mixer row order, ld_dcorr >= 196.  Per unit and level the
 * adjoint of the 49-tap blend is an 8x8 weight matrix A over the unit's footprint (the pixels pips_corr_gather read):
 *   A[j][i] = (1/sqrt(128)) sum_{dy,dx in {0,1}} w_{dy,dx} dcorr[l*49 + (i-dx)*7 + (j-dy)]   (0 <= i-dx, j-dy < 7)
 * Every output element is written once, summed in a fixed order (deterministic, no atomics).
 * pips_corr_grad_feats: dffeat_rows (B*N, S, 128) = sum over levels and footprint pixels of A * level pixel.
 * pips_corr_grad_levels: dlvl[l] (B*S, H>>l, W>>l, 128) = sum over the frame's units, in ascending n, of A * ffeat
 *   (ffeat_rows (B*N, S, 128)); pixels no footprint covers are 0. */
int pips_corr_grad_feats(const float* const* lvl, int B, int S, int N, int H, int W, const float* coords,
                         const float* dcorr, int ld_dcorr, float* dffeat_rows, void* stream);
int pips_corr_grad_levels(int B, int S, int N, int H, int W, const float* coords, const float* ffeat_rows,
                          const float* dcorr, int ld_dcorr, float* const* dlvl, void* stream);
/* pips_corr_grad_feats / pips_corr_grad_levels for windows of 2 <= S <= PIPS_S_MAX frames (the entry points above take
 * S == 8 only): the same arguments and checks; at S == 8 the same kernels, so the same bits. */
int pips_corr_grad_feats_window(const float* const* lvl, int B, int S, int N, int H, int W, const float* coords,
                                const float* dcorr, int ld_dcorr, float* dffeat_rows, void* stream);
int pips_corr_grad_levels_window(int B, int S, int N, int H, int W, const float* coords, const float* ffeat_rows,
                                 const float* dcorr, int ld_dcorr, float* const* dlvl, void* stream);

/* nn.Linear on tensor cores: out = epi(A[M,K] . W[N,K]^T + bias).  a_lo/w_lo NULL => plain bf16. */
int pips_gemm_tc(const void* a_hi, const void* a_lo, int lda, int a_rows,
                 const void* w_hi, const void* w_lo, int ldw, int w_rows,
                 int M, int N, int K, const float* bias, int epilogue,
                 float* out_f32, int ldo, void* out_hi, void* out_lo, int ldh, void* stream);

/* pips_gemm_tc with an fp32 side tensor aux (row stride ld_aux) for the two pre-activation epilogues: BIAS_GELU_PRE
 * also writes the pre-activation acc + bias there (what the GELU backward needs); GELU_GRAD reads it and writes
 * (acc + bias) * GELU'(aux) with the exact-erf derivative -- the FC2 input gradient of the mixer's backward.  Both need
 * N % 8 == 0 and an 8-byte aligned aux; the other epilogues ignore aux (may be NULL). */
int pips_gemm_tc_aux(const void* a_hi, const void* a_lo, int lda, int a_rows,
                     const void* w_hi, const void* w_lo, int ldw, int w_rows,
                     int M, int N, int K, const float* bias, int epilogue,
                     float* out_f32, int ldo, void* out_hi, void* out_lo, int ldh,
                     float* aux, int ld_aux, void* stream);

/* ---- backward of the DeltaBlock mixer (csrc/gemm_tc.cu, csrc/mixer_grad.cu).  Every sum runs in a fixed order that
 * depends on the shape only: no atomics, the same bits on any GPU. ----
 * Weight gradient of a dense layer on the tensor cores, bf16x3: dw[n,k] = sum_m G[m,n] X[m,k] for m < M, with
 * G (M, N) row stride ldg and X (M, K) row stride ldx as bf16 (hi, lo) pairs; dw (N, K) fp32, dense.  N, K, ldg, ldx
 * multiples of 8, every pointer 16-byte aligned.  M is split into chunks whose partial sums go to scratch
 * (pips_wgrad_scratch_floats(M, N, K) floats; may be NULL when that is 0). */
size_t pips_wgrad_scratch_floats(int M, int N, int K);
int pips_wgrad(const void* g_hi, const void* g_lo, int ldg, const void* x_hi, const void* x_lo, int ldx, int M, int N, int K,
               float* scratch, float* dw, void* stream);
/* column sums out[n] = sum_{m < M} g[m*ld + n]: of fp32 g, or (g == NULL) of the bf16 pair g_hi + g_lo.  The bias
 * gradients of the dense layers.  scratch: pips_colsum_scratch_floats(M, N) floats (may be NULL when that is 0). */
size_t pips_colsum_scratch_floats(int M, int N);
int pips_colsum(const float* g, const void* g_hi, const void* g_lo, size_t ld, int M, int N, float* scratch, float* out,
                void* stream);
/* Backward of pips_tokenmix for one mixer block (nets/pips.py:117-118), one sequence of 8 rows x 512 per CTA:
 * x_in, the block input; x_mid, the residual stream after token mixing (what pips_tokenmix leaves in x); dy, the
 * gradient of LN2's output.  dx (seqs*8, 512) holds the gradient of the block output on entry and that of the block input
 * on return (the FC branch's residual included).  grads (2600 floats) receives the parameter gradients:
 *   ln1_w[512] ln1_b[512] tok_w1[32*8] tok_b1[32] tok_w2[8*32] tok_b2[8] ln2_w[512] ln2_b[512].
 * scratch: pips_tokenmix_grad_scratch_floats(seqs) floats. */
size_t pips_tokenmix_grad_scratch_floats(int seqs);
int pips_tokenmix_grad(const float* x_in, const float* x_mid, const float* dy, float* dx, int seqs, const float* ln1_w,
                       const float* ln1_b, const float* w1, const float* b1, const float* w2, const float* b2,
                       const float* ln2_w, const float* ln2_b, float* scratch, float* grads, void* stream);
/* Backward of pips_ln_pool: dp (seqs, 512), the gradient of the pooled rows -> dx (seqs*8, 512), and the LayerNorm's
 * parameter gradients grads = ln_w[512] ln_b[512].  scratch: pips_ln_pool_grad_scratch_floats(seqs) floats. */
size_t pips_ln_pool_grad_scratch_floats(int seqs);
int pips_ln_pool_grad(const float* x, const float* dp, int seqs, const float* ln_w, const float* ln_b, float* dx,
                      float* scratch, float* grads, void* stream);

/* the same contract in fp32 on CUDA cores (PIPS_PREC_F32) */
int pips_gemm_f32(const float* a, int lda, const float* w, int ldw, int M, int N, int K,
                  const float* bias, int epilogue, float* out, int ldo, void* stream);

/* nets/pips.py:117 (token-mixing PreNormResidual: LN -> Conv1d(8,32,1) -> GELU -> Conv1d(32,8,1) -> +x)
 * followed by the LayerNorm of the channel-mixing block (:118, :100), in place on x (seqs*8, 512).
 * y_* receive LN2(x_new) as the A operand of FC1. */
int pips_tokenmix(float* x, int seqs, const float* ln1_w, const float* ln1_b,
                  const float* w1 /* (32,8) */, const float* b1, const float* w2 /* (8,32) */, const float* b2,
                  const float* ln2_w, const float* ln2_b, void* y_hi, void* y_lo, float* y_f32, void* stream);
/* pips_tokenmix for windows of 2 <= S <= PIPS_S_MAX frames: x (seqs*S, 512), w1 (4S, S), b1 [4S], w2 (S, 4S), b2 [S]
 * (Conv1d(S,4S,1) -> GELU -> Conv1d(4S,S,1)).  Only the seqs*S rows of x and y are read or written. */
int pips_tokenmix_s(float* x, int seqs, int S, const float* ln1_w, const float* ln1_b, const float* w1, const float* b1,
                    const float* w2, const float* b2, const float* ln2_w, const float* ln2_b, void* y_hi, void* y_lo,
                    float* y_f32, void* stream);

/* the same with the two contractions as wgmma MMAs (channels as the M dimension, bf16x3 folded into K); bf16
 * outputs only.  Selected inside pips_tokenmix by PIPS_B200_TOKENMIX=tc; see csrc/tokenmix_tc.cu for its status. */
int pips_tokenmix_tc(float* x, int seqs, const float* ln1_w, const float* ln1_b, const float* w1, const float* b1,
                     const float* w2, const float* b2, const float* ln2_w, const float* ln2_b, void* y_hi, void* y_lo,
                     void* stream);
int pips_tokenmix_tc_s(float* x, int seqs, int S, const float* ln1_w, const float* ln1_b, const float* w1, const float* b1,
                       const float* w2, const float* b2, const float* ln2_w, const float* ln2_b, void* y_hi, void* y_lo,
                       void* stream);

/* nets/pips.py:120-121: final LayerNorm(512) then mean over the S rows of each sequence. */
int pips_ln_pool(const float* x, int seqs, const float* ln_w, const float* ln_b,
                 void* p_hi, void* p_lo, float* p_f32, void* stream);
/* the same over x (seqs*S, 512), 2 <= S <= PIPS_S_MAX: the mean is the sum of the S normalised rows divided by S */
int pips_ln_pool_s(const float* x, int seqs, int S, const float* ln_w, const float* ln_b,
                   void* p_hi, void* p_lo, float* p_f32, void* stream);

/* ---- results written straight into every rank's memory over NVLink (SURVEY.md section 8e: "fusing the coord
 * all-gather into the update epilogue") ----
 * Particle-sharded runs: rank g owns particles [n_offset, n_offset + N) of n_total.  out[r] is rank r's copy of the
 * FULL (B,S,n_total,2) result of the current iteration, mapped into this process (pips_peer_open; out[own rank] is
 * the local allocation).  The update kernel stores its slice into all of them, so after pips_peer_barrier every
 * rank holds the whole result and no collective library call sits on the data path.  n_peers == 0: off. */
#define PIPS_MAX_PEERS 16
typedef struct pips_peer_out {
    float* out[PIPS_MAX_PEERS];
    int n_peers, n_offset, n_total;
} pips_peer_out;

/* cudaMalloc + cudaIpcGetMemHandle: *ptr is the local allocation, handle (64 bytes) goes to the other ranks. */
int pips_peer_alloc(size_t bytes, void** ptr, unsigned char* handle64);
/* cudaIpcOpenMemHandle (peer access enabled lazily) / cudaIpcCloseMemHandle / cudaFree */
int pips_peer_open(const unsigned char* handle64, void** ptr);
int pips_peer_close(void* ptr);
int pips_peer_free(void* ptr);
/* copy src (rows, cols) fp32, contiguous, into dst[r] (rows, cols_total) at column col_offset, for r < n_peers */
int pips_peer_scatter(const float* src, int rows, int cols, float* const* dst, int n_peers, int cols_total, int col_offset,
                      void* stream);
/* flag barrier across the ranks of one node: store `epoch` into flags[r][rank] of every rank r (system-scope release
 * after a system fence), then wait until flags[rank][r] >= epoch for all r.  flags[r] is rank r's int[PIPS_MAX_PEERS]
 * array as mapped here.  Traps after timeout_ms (a lost rank must not hang the device). */
int pips_peer_barrier(int* const* flags, int rank, int n_peers, int epoch, int timeout_ms, void* stream);

/* nets/pips.py:525-539: split delta, ffeats += GELU(Linear(GroupNorm(1,128)(dfeat))), coords += dcoord,
 * re-lock frame 0, emit coords*stride.  delta is (B*N, S*130) with row stride PIPS_DELTA_LD(S) (S*130 for even S),
 * 2 <= S <= PIPS_S_MAX. */
int pips_update(const float* delta, float* coords, const float* coords0, float* ffeats,
                const float* gn_w, const float* gn_b, const float* wu /* (128,128) */, const float* bu,
                float* out_px /* (B,S,N,2) */, float stride, int B, int S, int N, void* stream);
/* pips_update that also stores coords*stride into every rank's full-size result (peer may be NULL) */
int pips_update_peer(const float* delta, float* coords, const float* coords0, float* ffeats,
                     const float* gn_w, const float* gn_b, const float* wu, const float* bu,
                     float* out_px, float stride, int B, int S, int N, const pips_peer_out* peer, void* stream);

/* nets/pips.py:559: vis_e = Linear(128,1)(ffeats) -> (B,S,N) logits */
int pips_vis_head(const float* ffeats, const float* w, const float* b, float* vis, int B, int S, int N, void* stream);

/* nets/pips.py:504-511 for chosen particles only (SURVEY.md 8f-3): the dense score map
 *   fcp[b,s,j,:,:] = sum_l interpolate(<ffeats[b,s,sel[j]], fmaps_l[b,s]> / sqrt(C), (H8,W8), bilinear, align_corners=True)
 * read from the pyramid levels (channels-last, feat_dtype); ffeats is the loop state ((b*N+n), s, c).
 * sel[n_sel]: particle indices in [0,N); slot[n_sel] (or NULL = identity): position of query j in the output;
 * out element (b*S+s, slot, y, x) lives at out[(b*S+s)*out_frame_stride + (slot*H8 + y)*W8 + x].
 * scratch: pips_heatmap_scratch_floats(B*S, n_sel, H8, W8) floats. */
size_t pips_heatmap_scratch_floats(int frames, int n_sel, int H8, int W8);
int pips_heatmap(const void* const* lvl, int feat_dtype, int B, int S, int N, int H8, int W8, const float* ffeats,
                 const int* sel, const int* slot, int n_sel, float* scratch, float* out, size_t out_frame_stride, void* stream);

/* nets/pips.py:58-90 (score_map_loss) without the dense score maps (csrc/scoremap_loss.cu).  The score map of
 * nets/pips.py:504-511 is fcp[b,s,n,p] = <ffeats[b,s,n], G[b,s,p]> with
 *   G[b,s,p,:] = sum_l interpolate(fmap_l[b,s], (H8,W8), bilinear, align_corners=True)(p,:) / sqrt(C).
 * pips_scoremap_basis: G from the fp32 pyramid levels lvl_f32[4] (channels-last) as a bf16 (hi, lo) pair,
 *   G_hi / G_lo (frames, H8*W8, 128).  Once per forward.
 * pips_scoremap_loss: one iteration.  ffeats is the loop state ((b*N+n), s, c) at the start of the iteration;
 *   target (B,S,N) int32 is y*W8 + x of the row's target pixel, or -1 for a row the loss ignores.  For every row
 *   r = (b*S + s)*N + n it writes pos_part[r] = softplus(-fcp[t]) and neg_part[r, k] = sum of softplus(fcp[p]) over
 *   the pixels p != t of split k (both 0 for target -1).  The score GEMM runs in bf16x3; scores never reach memory.
 * pips_scoremap_splits: n_split, the number of pixel splits (columns of neg_part); a function of H8*W8 only. */
int pips_scoremap_splits(int H8, int W8);
int pips_scoremap_basis(const float* const* lvl_f32, int frames, int H8, int W8, void* G_hi, void* G_lo, void* stream);
int pips_scoremap_loss(const void* G_hi, const void* G_lo, const float* ffeats, int B, int S, int N, int H8, int W8,
                       const int* target, float* neg_part, float* pos_part, void* stream);
/* pips_scoremap_loss for windows of 2 <= S <= PIPS_S_MAX frames (pips_scoremap_loss itself takes S == 8 only). */
int pips_scoremap_loss_window(const void* G_hi, const void* G_lo, const float* ffeats, int B, int S, int N, int H8, int W8,
                              const int* target, float* neg_part, float* pos_part, void* stream);

/* Backward of the score-map loss over `iters` iterations (csrc/scoremap_grad.cu), without the dense score maps.
 * coef (device, 2 floats) holds g/(eps+K) and g/(eps+K(P-1)): g the upstream gradient, K the kept rows times iters,
 * P = H8*W8, eps = 1e-6.  target is that of pips_scoremap_loss; G_hi / G_lo that of pips_scoremap_basis.  Each output
 * element is summed in a fixed order (deterministic, no atomics); the score GEMMs run in bf16x3.  S == 8; the _window
 * siblings take 2 <= S <= PIPS_S_MAX.
 * pips_scoremap_grad_feats: dffeats = dloss/dffeats, both (iters, B*S, N, 128) fp32 frame-major
 *   (ffeats[i, b*S+s, n] is the ffeats of track (b, n) in frame s at the start of iteration i).
 * pips_scoremap_grad_basis: dG = dloss/dG (B*S, H8*W8, 128) fp32, from F_hi / F_lo, the bf16 (hi, lo) split of those
 *   ffeats (iters, B*S, N, 128).
 * pips_scoremap_basis_grad: the adjoint of pips_scoremap_basis: dG -> the fp32 channels-last level gradients
 *   dlvl_f32[l] (B*S, H8>>l, W8>>l, 128). */
int pips_scoremap_grad_feats(const void* G_hi, const void* G_lo, const float* ffeats, int iters, int B, int S, int N,
                             int H8, int W8, const int* target, const float* coef, float* dffeats, void* stream);
int pips_scoremap_grad_basis(const void* G_hi, const void* G_lo, const void* F_hi, const void* F_lo, int iters, int B,
                             int S, int N, int H8, int W8, const int* target, const float* coef, float* dG, void* stream);
/* pips_scoremap_grad_feats / pips_scoremap_grad_basis for windows of 2 <= S <= PIPS_S_MAX frames: the same arguments,
 * checks and kernels (at S == 8 the same bits). */
int pips_scoremap_grad_feats_window(const void* G_hi, const void* G_lo, const float* ffeats, int iters, int B, int S, int N,
                                    int H8, int W8, const int* target, const float* coef, float* dffeats, void* stream);
int pips_scoremap_grad_basis_window(const void* G_hi, const void* G_lo, const void* F_hi, const void* F_lo, int iters,
                                    int B, int S, int N, int H8, int W8, const int* target, const float* coef, float* dG,
                                    void* stream);
int pips_scoremap_basis_grad(const float* dG, int frames, int H8, int W8, float* const* dlvl_f32, void* stream);

/* v -> (hi, lo) bf16 with hi = rn(v), lo = rn(v - hi); lo may be NULL.  Used to pack weights. */
int pips_split_bf16(const float* src, void* hi, void* lo, size_t n, void* stream);

/* ---- channels-last element-wise stages of fnet (BasicEncoder, nets/pips.py:131-281; upstream of the loop) ----
 * InstanceNorm2d statistics of y (N, HW, C) NHWC: stats = [N][2][C] (mean, rstd); partial is [N][chunks][3][C] scratch. */
int pips_inorm_stats(const float* y, int N, int HW, int C, float* partial, int chunks, float* stats, void* stream);
/* out = relu_out?( relu_main?( norm(y) ) + norm?(r) ); written as plain fp32 and/or as the [hi|lo|hi] TF32 split
 * (3*C channels at row stride split_ld) that conv2d_3xtf32 consumes.  stats_y / r / stats_r may be NULL. */
int pips_inorm_apply(const float* y, const float* stats_y, const float* r, const float* stats_r, int relu_main, int relu_out,
                     float* out_plain, float* out_split, int split_ld, int N, int HW, int C, void* stream);
/* F.interpolate(bilinear, align_corners=True) (nets/pips.py:269-272) of src (N,Hs,Ws,C) into channels
 * [c_off, c_off+C) of the split concat dst (N,Ho,Wo,3*Ctot). */
int pips_resize_split3(const float* src, int N, int Hs, int Ws, int C, float* dst, int Ho, int Wo, int Ctot, int c_off,
                       void* stream);

/* bf16 (hi, lo) flavours of the two functions above: the operand layout of pips_conv_tc (row stride pair_ld /
 * Ctot channels).  The K-padding channels are written as zero by these calls themselves: pips_inorm_apply_pair
 * zeroes [C, pair_ld); pips_resize_pair zeroes [c_off+C, Ctot) when fewer than 64 channels remain after its slice
 * (i.e. the slice is the last one before the padding of a row padded to a multiple of 64). */
int pips_inorm_apply_pair(const float* y, const float* stats_y, const float* r, const float* stats_r, int relu_main, int relu_out,
                          float* out_plain, void* out_hi, void* out_lo, int pair_ld, int N, int HW, int C, void* stream);
int pips_resize_pair(const float* src, int N, int Hs, int Ws, int C, void* dst_hi, void* dst_lo, int Ho, int Wo, int Ctot, int c_off,
                     void* stream);
/* nn.Conv2d (3x3 / 1x1, stride 1 / 2; nets/pips.py:135-136,:170,:221-223) as an implicit GEMM on the tensor cores
 * (wgmma, bf16x3).  x_hi/x_lo (N,H,W,Cp) bf16 with Cp % 64 == 0; w_hi/w_lo (BN, R*S*Cp) bf16,
 * k = (r*S + s)*Cp + ci, BN = Cout rounded up to 64/128/256 with zero rows; out (N,Ho,Wo,Cout) fp32; bias may be NULL. */
int pips_conv_tc(const void* x_hi, const void* x_lo, int N, int H, int W, int Cp, const void* w_hi, const void* w_lo,
                 int Cout, int R, int S, int stride, int pad, const float* bias, float* out, void* stream);

/* 3x3 / stride 1 / pad 1 convolution with 64 input and 64 output channels (BasicEncoder layer1, nets/pips.py:135-136):
 * every input row is loaded once into a ring of row buffers and serves all 9 filter taps (csrc/conv_rows.cu).
 * x_hi/x_lo (N,H,W,64) bf16, w_hi/w_lo (64, 9*64) bf16 [k = (r*3+s)*64 + ci], out (N,H,W,64) fp32.  partial (optional):
 * (N, pips_conv_rows_chunks(H,W), 3, 64) per-chunk (mean, M2, count) of `out` per channel -- the InstanceNorm
 * statistics (nets/pips.py:154-157), merged by pips_inorm_finalize. */
int pips_conv_rows_chunks(int H, int W);
int pips_conv_rows(const void* x_hi, const void* x_lo, int N, int H, int W, const void* w_hi, const void* w_lo, float* out,
                   float* partial, void* stream);
/* (mean, 1/sqrt(var + 1e-5)) per (image, channel) from `chunks` partial rows per image.  A partial row is three vectors of
 * C floats: the chunk's mean, M2 (sum of squared deviations from that mean) and pixel count; the counts of an image add up
 * to HW.  (ABI 4; ABI 3 stored (sum, sum of squares), which cancels catastrophically on flat images.) */
int pips_inorm_finalize(const float* partial, int N, int chunks, int HW, int C, float* stats, void* stream);

int pips_conv_tc_aniso(const void* x_hi, const void* x_lo, int N, int H, int W, int Cp, const void* w_hi, const void* w_lo,
                       int Cout, int R, int S, int stride_y, int stride_x, int pad_y, int pad_x, const float* bias, float* out,
                       void* stream);
/* pips_conv_tc_aniso that also accumulates, in its epilogue, the InstanceNorm partial statistics of its output
 * (nets/pips.py:154-157): partial (N, pips_conv_tc_chunks(geometry), 3, Cout) fp32 per-chunk (mean, M2, count) per
 * channel; the chunking depends on the image geometry only.  Merge with pips_inorm_finalize. */
int pips_conv_tc_chunks(int H, int W, int R, int S, int stride_y, int stride_x, int pad_y, int pad_x);
int pips_conv_tc_stats(const void* x_hi, const void* x_lo, int N, int H, int W, int Cp, const void* w_hi, const void* w_lo,
                       int Cout, int R, int S, int stride_y, int stride_x, int pad_y, int pad_x, const float* bias, float* out,
                       float* partial, void* stream);
/* nets/pips.py:436 + the unfolding of the 7x7/2 stem (:206) into a 4x1 stride-1 convolution: rgb (N,3,H,W) fp32
 * (dtype 0) or bf16 (dtype 1), 0..255 -> (N, Ho+3, Wo, 64) bf16 (hi, lo), Ho = (H-1)/2+1, Wo = (W-1)/2+1; pixel (j, ox)
 * holds input rows y = 2j-3 (channels 0..31) and y = 2j-2 (channels 32..63), channel k = s*3 + colour of a row =
 * 2*(rgb/255)-1 at x = 2*ox + s - 3, zero outside the image / for k >= 21.  (ABI 3; ABI 2 unfolded the columns only.) */
int pips_stem_pack(const void* rgb, int dtype, int N, int H, int W, void* out_hi, void* out_lo, void* stream);

/* ---- the whole feature encoder in one call (csrc/encoder.cu; BasicEncoder.forward, nets/pips.py:247-281) ----
 * Filters of one convolution: the bf16 (hi, lo) pack of the weight pack's fnet.<conv>.w_hi / .w_lo entries
 * (pips_conv_tc's layout; the stem's is pips_stem_pack's 4x1 layout, (64, 4*64)) and its bias [Cout] fp32.  Only conv3's
 * bias is read (it may be NULL: no bias): every other convolution feeds an InstanceNorm, which removes a per-channel
 * constant again. */
typedef struct pips_conv_weights {
    const void *w_hi, *w_lo;
    const float* b;
} pips_conv_weights;

/* one field per convolution, named as the pack's fnet.* entries with '.' -> '_', in module order */
typedef struct pips_encoder_weights {
    pips_conv_weights conv1;
    pips_conv_weights layer1_0_conv1, layer1_0_conv2, layer1_1_conv1, layer1_1_conv2;
    pips_conv_weights layer2_0_conv1, layer2_0_conv2, layer2_0_downsample_0, layer2_1_conv1, layer2_1_conv2;
    pips_conv_weights layer3_0_conv1, layer3_0_conv2, layer3_0_downsample_0, layer3_1_conv1, layer3_1_conv2;
    pips_conv_weights layer4_0_conv1, layer4_0_conv2, layer4_0_downsample_0, layer4_1_conv1, layer4_1_conv2;
    pips_conv_weights conv2, conv3;
} pips_encoder_weights;

/* Scratch bytes of one pips_encode call: the stem operand, the convolution outputs, the partial statistics, the (hi, lo)
 * pairs and the concatenation, each region 256-byte aligned.  A pure function of the shapes, covering every kernel
 * choice of PIPS_B200_CONV_ROWS / PIPS_B200_CONV_STATS; 0 for shapes pips_encode refuses. */
size_t pips_encode_workspace_bytes(int N, int H, int W, int stride);
/* Kernels one pips_encode call of these shapes launches under the current PIPS_B200_CONV_ROWS / PIPS_B200_CONV_STATS
 * (0 for refused shapes). */
int pips_encode_launches(int N, int H, int W, int stride);
/* rgb (N,3,H,W) with values 0..255, fp32 (dtype 0) or bf16 (dtype 1) -> fmaps_nhwc (N, H/stride, W/stride, 128) fp32,
 * channels-last: the input of pips_pyramid_build_nhwc.  stride 4 or 8, H, W >= stride, 1 <= N <= 65535.  Enqueues
 * the stem (pips_stem_pack + 4x1 wgmma convolution), the 8 ResBlocks, the 4 resizes into the concatenation and the
 * head on `stream`: no allocation, no synchronisation, capturable into a CUDA graph.  workspace: at least
 * pips_encode_workspace_bytes(N, H, W, stride) bytes, 256-byte aligned; fmaps_nhwc 16-byte aligned.
 * keep: NULL, or 9 pointers (16-byte aligned) that receive the block boundaries, fp32 channels-last: [0] the stem's
 * output (N, (H-1)/2+1, (W-1)/2+1, 64), [1 + 2l + j] the output of ResBlock j of layer l+1 (64, 96, 128, 128 channels,
 * halved in size per layer from layer 2 on).  Arguments are checked before the first launch. */
int pips_encode(const pips_encoder_weights* w, const void* rgb, int dtype, int N, int H, int W, int stride, void* workspace,
                size_t workspace_bytes, float* fmaps_nhwc, float* const* keep, void* stream);

/* ---- backward of the feature encoder (csrc/conv_grad.cu, csrc/encoder_grad.cu).  Every sum runs in a fixed order that
 * depends on the shape only: no atomics, the same bits on any GPU. ----
 * Weight gradient of a convolution on the tensor cores, bf16x3:
 *   dw[co, (r*S + s)*Cp + ci] = sum_{n,oy,ox} dy[n,oy,ox,co] * x[n, oy*stride_y + r - pad_y, ox*stride_x + s - pad_x, ci]
 * x (N, H, W, Cp) bf16 (hi, lo) as pips_conv_tc reads it (zero outside the image); dy bf16 (hi, lo) of channel pitch
 * ldy >= Cout (multiple of 8): (N, Ho, Wo, ldy) with dy_step 1, or, with dy_step 2 (stride-2 convolutions only),
 * zero-dilated on the input's (N, H, W, ldy) grid with output pixel (oy, ox) at (2oy, 2ox).  dw (Cout, R*S*Cp) fp32,
 * dense.  The pixels are split into chunks whose partial sums go to scratch
 * (pips_conv_wgrad_scratch_floats(N, Ho, Wo, Cout, R*S*Cp) floats; may be NULL when that is 0). */
size_t pips_conv_wgrad_scratch_floats(int N, int Ho, int Wo, int Cout, int K);
int pips_conv_wgrad(const void* dy_hi, const void* dy_lo, int ldy, int dy_step, const void* x_hi, const void* x_lo, int N, int H,
                    int W, int Cp, int Cout, int R, int S, int stride_y, int stride_x, int pad_y, int pad_x, float* scratch,
                    float* dw, void* stream);
/* Backward of pips_inorm_apply_pair's main branch (nets/pips.py:154-157 + ReLU): with g = g0 (+ g1) (+ g2) the gradient
 * of the forward's output (N, H, W, C) fp32, masked by the ReLUs the forward applied (recomputed from y, stats, r,
 * stats_r, relu_main, relu_out exactly as the forward computed them), and x_hat = (y - mean) * rstd:
 *   dy = rstd * (g - mean(g) - x_hat * mean(g * x_hat))            (means per image and channel over H*W)
 * written as a bf16 (hi, lo) pair of row stride pair_ld (channels [C, pair_ld) zero), on the (H, W) grid, or with
 * dil_h, dil_w != 0 zero-dilated on that (2H or 2H-1, 2W or 2W-1) grid (pixel (y, x) at (2y, 2x), zeros elsewhere).
 * g_out (optional): g after the output ReLU's mask only -- the gradient of the residual branch.  r requires relu_out.
 * scratch: pips_inorm_grad_scratch_floats(N, H*W, C) floats, 16-byte aligned. */
size_t pips_inorm_grad_scratch_floats(int N, int HW, int C);
int pips_inorm_grad(const float* y, const float* stats, const float* r, const float* stats_r, int relu_main, int relu_out,
                    const float* g0, const float* g1, const float* g2, int N, int H, int W, int C, float* scratch, void* dy_hi,
                    void* dy_lo, int pair_ld, int dil_h, int dil_w, float* g_out, void* stream);
/* Adjoint of pips_resize_pair (bilinear, align_corners=True, (Hs, Ws) -> (Ho, Wo)): out (N, Hs, Ws, C) fp32 from the
 * channels [c_off, c_off + C) of g (N, Ho, Wo, ldg) fp32.  A gather: every source pixel sums the destination pixels
 * whose taps touch it, in a fixed order. */
int pips_resize_grad(const float* g, int ldg, int c_off, int N, int Ho, int Wo, float* out, int Hs, int Ws, int C, void* stream);

/* Whole-iteration operator: everything between `for itr in range(iters)` and the append of
 * coords*stride (nets/pips.py:499-539, minus the dead fcp heat-map :504-511). */
typedef struct pips_layer_weights {
    const float *ln1_w, *ln1_b, *tok_w1, *tok_b1, *tok_w2, *tok_b2, *ln2_w, *ln2_b;
    const float *fc1_b, *fc2_b;
    const void *fc1_w_hi, *fc1_w_lo, *fc2_w_hi, *fc2_w_lo;   /* bf16 (2048,512) / (512,2048)            */
    const float *fc1_w_f32, *fc2_w_f32;                      /* used by PIPS_PREC_F32 only             */
} pips_layer_weights;

typedef struct pips_weights {
    const void *in_w_hi, *in_w_lo;        /* (512, 576) bf16, K zero-padded from 519                   */
    const float* in_w_f32;                /* (512, 576) fp32                                           */
    const float* in_b;
    pips_layer_weights layer[PIPS_DEPTH];
    const float *out_ln_w, *out_ln_b;
    const void *head_w_hi, *head_w_lo;    /* (PIPS_HEAD_PAD(S), 512) bf16, rows zero-padded from 130*S: */
                                          /* (1280, 512) for S = 8                                     */
    const float* head_w_f32;              /* (130*S, 512)                                              */
    const float* head_b;
    const float *gn_w, *gn_b, *upd_w, *upd_b, *vis_w, *vis_b;
} pips_weights;

typedef struct pips_workspace {
    int rows_alloc;                       /* allocated mixer rows (>= B*N*S, multiple of 128)          */
    int seqs_alloc;                       /* allocated pooled rows (>= B*N, multiple of 128)           */
    void *x0_hi, *x0_lo;  float* x0_f32;  /* (rows_alloc, 576)                                         */
    float* x;                             /* (rows_alloc, 512) residual stream                         */
    void *y_hi, *y_lo;    float* y_f32;   /* (rows_alloc, 512)                                         */
    void *h_hi, *h_lo;    float* h_f32;   /* (rows_alloc, 2048)                                        */
    void *p_hi, *p_lo;    float* p_f32;   /* (seqs_alloc, 512)                                         */
    float* delta;                         /* (seqs_alloc, PIPS_DELTA_LD(S)): 130*S used, 1040 at S = 8  */
} pips_workspace;

typedef struct pips_problem {
    int B, S, N, H, W;                    /* H, W of pyramid level 0; 2 <= S <= PIPS_S_MAX (8 with a   */
                                          /* clip table or groups)                                     */
    int feat_dtype, precision;
    const void* lvl[PIPS_LEVELS];
    const float* times;                   /* [S] = linspace(0,S,S)  nets/pips.py:519                   */
    float* coords;                        /* (B,S,N,2) in/out                                          */
    const float* coords0;                 /* (B,S,N,2) initial coords (frame 0 is re-locked)           */
    float* ffeats;                        /* (B*N,S,128) in/out                                        */
    float stride;
    const int* frame_base;                /* NULL, or [B*N] window starts for chained tracking         */
    int frames_per_batch;                 /* frames per batch element in the pyramid when frame_base   */
    pips_peer_out peer;                   /* n_peers > 0: also scatter coords*stride to every rank     */
} pips_problem;

/* DeltaBlock.forward on prepared input rows (nets/pips.py:304-311, mixer :111-123): x0 -> ws->delta */
int pips_mixer_forward(const pips_weights* w, const pips_workspace* ws, int seqs, int precision, void* stream);
/* the same for a model of window length 2 <= S <= PIPS_S_MAX: seqs*S mixer rows, delta (seqs, PIPS_DELTA_LD(S)) */
int pips_mixer_forward_s(const pips_weights* w, const pips_workspace* ws, int seqs, int S, int precision, void* stream);

/* one refinement iteration; out_px receives coords*stride (B,S,N,2) */
int pips_refine_iter(const pips_problem* p, const pips_weights* w, const pips_workspace* ws,
                     float* out_px, void* stream);
/* pips_refine_iter whose correlation reads each track's window inside its own clip: pips_corr_gather_clips with
 * p->frame_base (required when clip is non-NULL) and clip [B*N][2]; the mixer and the update are unchanged. */
int pips_refine_iter_clips(const pips_problem* p, const int* clip /* NULL or [B*N][2] */, const pips_weights* w,
                           const pips_workspace* ws, float* out_px, void* stream);
/* pips_refine_iter whose correlation reads each track's window in its own pyramid group: pips_corr_gather_groups
 * over `groups` (levels in p->feat_dtype) with p->frame_base (required) and table [B*N][4] (required).  p->lvl, p->H,
 * p->W and p->frames_per_batch are ignored; the mixer and the update are unchanged. */
int pips_refine_iter_groups(const pips_problem* p, const pips_groups* groups, const int* table /* [B*N][4] */,
                            const pips_weights* w, const pips_workspace* ws, float* out_px, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* PIPS_B200_H */
