/* libprogen_b200.so — C ABI of the CUDA-native ProGen hot path (NVIDIA H100, sm_90a).
 *
 * Drop-in boundary (SURVEY.md §8(b)): the reference exposes `ProGen(**kwargs) -> .init / .apply`
 * (lucidrains/progen progen_transformer/progen.py:235-243) and everything below that call is executed by XLA.
 * This library replaces that device path.  Each entry point names the reference lines whose arithmetic it owns.
 *
 * Conventions
 *  - every function returns 0 on success or a negative PROGEN_ERR_* code; `progen_last_error()` (thread-local) has
 *    the text.  Nothing allocates: the caller owns every buffer and workspace.  All work is asynchronous on `stream`
 *    (a cudaStream_t passed as void*), no internal synchronisation, no global mutable state except a cache of TMA
 *    descriptors keyed by (pointer, shape).
 *  - tokens are rows: activations are row-major [T = B * seq_len, features]; `ld*` are element strides.
 *  - dtype codes: PROGEN_F32 = 0, PROGEN_BF16 = 1.  The residual stream and all parameter gradients are fp32.
 *  - sm_90a only (`progen_device_check`); there is no CPU or other-architecture fallback.
 */
#ifndef PROGEN_B200_H
#define PROGEN_B200_H
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define PROGEN_F32 0
#define PROGEN_BF16 1

#define PROGEN_BACKEND_SIMT 0     /* fp32-exact CUDA-core GEMM (mixed_precision=False path, progen.py:235) */
#define PROGEN_BACKEND_TC 1       /* TMA + wgmma GEMM, bf16 operands / fp32 accumulate */

/* GEMM epilogues (fused with the matmul the reference line performs) */
#define PROGEN_EPI_STORE 0     /* out = acc (+bias)                      progen.py:219-222 (logits), 185 (SGU proj)   */
#define PROGEN_EPI_ROTARY 1    /* out = rotary(acc)                      progen.py:83-87 (to_qkv, rotary on q,k,v)    */
#define PROGEN_EPI_RESIDUAL 2  /* out(f32) = (aux|out)(f32) + acc + bias   progen.py:103+230, 148+231                    */
#define PROGEN_EPI_GLU 3       /* out = val*gelu(gate), out2 = pre-act   progen.py:137-141; out2 NULL: not stored     */
#define PROGEN_EPI_GELU 4      /* out = gelu(pre), out2 = pre-act        progen.py:137,143;  out2 NULL: not stored     */
#define PROGEN_EPI_GLU_BWD 5   /* out = d(pre-act) from acc = d(GLU out) (backward of 3)                               */
#define PROGEN_EPI_GELU_BWD 6  /* out = acc * gelu'(pre-act)             (backward of 4)                               */
#define PROGEN_EPI_ACCUM 7     /* out(f32) += acc  (weight gradients; optional tril mask for SGU spatial_weights)     */

const char* progen_version(void);
const char* progen_last_error(void);
int progen_device_check(void);
/* number of kernels this library has launched in this process (bench.py reports the per-run delta) */
long long progen_launch_count(void);

/* D[M,N] (+)= A[M,K] * B[N,K]^T.  Operand X(m,k): K-major -> X[m*ld + k]; MN-major -> X[k*ld + m].
 * Replaces every jnp matmul/einsum of the path: hk.Linear (progen.py:70-71,125-126,164,221), the SGU spatial
 * einsum 'n d, m n -> m d' (progen.py:181; causal=1 skips the masked upper-triangular K tiles), and their
 * transposes in the backward pass (jax.value_and_grad, utils.py:72). */
typedef struct progen_gemm_t {
  int32_t M, N, K;
  int32_t a_mn_major, b_mn_major;
  int32_t batch;         /* independent problems (grid z), >= 1 */
  int32_t batch_reduce;  /* 1: all batches accumulate into the same output (needs EPI_ACCUM + atomic) */
  int32_t causal;        /* 0 none, 1 lower (k < m0+128 only), 2 upper (k >= m0 only) */
  int32_t split_k;       /* >= 1; > 1 needs EPI_ACCUM + atomic */
  int32_t in_dtype, out_dtype, epi_kind, backend;
  int32_t seq_len, dim_head;          /* EPI_ROTARY */
  int32_t atomic, tril, tril_rows;    /* EPI_ACCUM */
  int64_t lda, ldb;
  int64_t a_batch_rows, b_batch_rows, d_batch_rows;   /* stored rows to skip per batch (0 = operand shared) */
  int64_t ldo, ldo2, ldaux;
  const void* A;
  const void* B;
  void* out;
  void* out2;
  const float* bias;
  const void* aux;
  const float* rot_sin;   /* [seq_len, dim_head/2], fixed_pos_embedding progen.py:24-28 */
  const float* rot_cos;
  float* colsum;          /* EPI_GLU_BWD / EPI_GELU_BWD, nullable: colsum[c] += sum over rows of the stored out[., c]
                             (the pre-activation Linear's bias gradient; 16-byte aligned on the TC backend) */
  /* Optional tail operand pair (K2 = 0: none): the accumulator is A*B^T + A2*B2^T, with A2(m,k) / B2(n,k) for k < K2
   * addressed like A / B through lda2 / ldb2 and their own major flags, before the unchanged epilogue.  The tail's
   * k-blocks run after the K loop of (A, B), in order, as if [A | A2] and [B | B2] were one operand pair (the TC backend
   * zero-fills the tail's last k-block).  This is a low-rank adapter's x*A*B folded into its projection's GEMM.  TC:
   * K2 % 8 == 0, a2/b2 major flags equal to a/b's, 16-byte aligned A2 / B2 and lda2 / ldb2 % 8 == 0.  Refused with a
   * tail: split_k > 1, causal, batch > 1, batch_reduce and EPI_ACCUM. */
  int64_t lda2, ldb2;
  const void* A2;
  const void* B2;
  int32_t K2, a2_mn_major, b2_mn_major, _pad_tail;
} progen_gemm_t;

int progen_gemm(const progen_gemm_t* desc, void* stream);

/* hk.Embed row gather — progen.py:207,226.  x is the fp32 residual stream [T, d]. */
int progen_embed_fwd(const int* tokens, const float* table, float* x, long long T, int d, int V, void* stream);
/* gradient of the gather: dtable[v,:] += sum_{t: tokens[t]==v} dx[t,:] */
int progen_embed_bwd(const int* tokens, const float* dx, float* dtable, long long T, int d, int V, void* stream);

/* y = shift_tokens(LayerNorm(x) * scale) — progen.py:22,43-46,74-77,132-135 (shift=1) and 170, 220 (shift=0).
 * Saves mean / rstd per row for the backward pass. */
int progen_ln_shift_fwd(const void* x, long long ldx, int x_dtype, const float* scale, void* y, long long ldy, int y_dtype,
                        float* mean, float* rstd, long long T, int d, int seq_len, int shift, void* stream);
/* backward of the above (dscale nullable: a frozen scale); residual=1 accumulates into the fp32 residual gradient `dres` [T,d] and mirrors it to `dout`;
 * `dres_colsum` (nullable, residual only) += column sums of the updated dres = the bias gradient of the Linear that
 * produced this residual branch's input (saves a separate pass over dres). */
int progen_ln_shift_bwd(const void* dy, long long lddy, int act_dtype, const void* x, long long ldx, int x_dtype,
                        const float* scale, const float* mean, const float* rstd, float* dres, void* dout, long long ldo,
                        float* dscale, float* dres_colsum, long long T, int d, int seq_len, int shift, int residual,
                        void* stream);

/* out[c] += sum_t in[t,c] — bias gradients of every hk.Linear */
int progen_colsum(const void* in, long long ld, int dtype, float* out, long long T, int N, void* stream);

/* cross_entropy + masked_mean + batch mean — utils.py:42-59,76 (pad-as-EOS mask, Q8); fused forward + d(logits).
 * *loss must be zeroed by the caller; inv_batch = 1/global_batch (DDP: a sum over ranks yields the global mean). */
int progen_ce_fwd_bwd(const void* logits, int dtype, const int* labels, float* weights, float* loss, void* dlogits,
                      int dlogits_dtype, int B, int n, int V, float inv_batch, void* stream);

/* scoring (inference): logp[t] = mask_t * log_softmax(logits[t])[label_t] with the loss mask of utils.py:54-56 (Q8: non-pad
 * labels plus the first pad; labels clamped to [0, V) like progen_ce_fwd_bwd); seq_ll[b] = sum_t logp[b, t] and
 * seq_count[b] = sum_t mask_t, reduced in a fixed order (bitwise independent of B).  logp: [B*n]; seq_ll, seq_count: [B].
 * -seq_ll / seq_count is the per-sequence cross_entropy of utils.py:45-59. */
int progen_token_logprob(const void* logits, int dtype, const int* labels, float* logp, float* seq_ll, float* seq_count,
                         int B, int n, int V, void* stream);
/* preference (DPO) head over B = 2 * pairs rows: rows 0..pairs-1 are chosen, row i + pairs is the rejected row of pair i;
 * ref_ll [B] holds the frozen reference's sums in the same order.  Runs progen_token_logprob (logp [B*n], seq_ll and
 * seq_count [B] as there: s(row) = seq_ll), then per pair, in double, z = beta * ((s(c) - ref_c) - (s(r) - ref_r)) and
 * loss_i = softplus(-z), and the per-token weights [B*n] w_t = -(d loss / d s(row)) * mask_t = +-beta * sigma(-z) *
 * inv_pairs * mask_t, then the CE kernel of progen_ce_fwd_bwd with those weights: dlogits = w_t * (softmax - onehot).
 * stats [pairs, 4] = (s(c), s(r), z, loss_i); *loss = inv_pairs * sum_i loss_i (written, not accumulated).  ce_scratch is
 * one float the CE kernel accumulates its unused weighted NLL into.  No float atomics reach stats, loss or weights: they
 * are the same bits in every launch.  Refused: null pointers, pairs < 1, beta or inv_pairs not finite and > 0. */
int progen_preference_head(const void* logits, int dtype, const int* labels, const float* ref_ll, float* logp, float* seq_ll,
                           float* seq_count, float* weights, float* stats, float* loss, float* ce_scratch, void* dlogits,
                           int dlogits_dtype, int pairs, int n, int V, float beta, float inv_pairs, void* stream);
/* distillation head (DESIGN.md §3.13): student logits s [B*n, V] in dtype, teacher logits z fp32 with row b, position t at
 * teacher + (b * teacher_row_stride + t) * V (teacher_row_stride >= n: the teacher may run at a longer row length), labels
 * [B*n] with the loss mask m_t of progen_ce_fwd_bwd (Q8) and c_b = sum_t m_t.  Per position, lq = log_softmax(s / tau),
 * lp = log_softmax(z / tau), KL_t = sum_v exp(lp_v) (lp_v - lq_v) (terms whose exp(lp_v) underflows to 0 add 0) and
 * CE_t = -log_softmax(s)[label_t] (label clamped to [0, V)).  stats [B, 2] = (KL_b, CE_b) = sum_t m_t (KL_t, CE_t) / c_b;
 * *loss = inv_batch * sum_b [(1 - alpha) tau^2 KL_b + alpha CE_b] in double, rows in order (written, not accumulated);
 * dlogits [B*n, V] in dlogits_dtype = inv_batch m_t / c_b [(1 - alpha) tau (softmax(s / tau) - softmax(z / tau)) +
 * alpha (softmax(s) - onehot(label_t))], every row written (+0.0 where m_t = 0; those positions do not read the teacher).
 * weights [B*n] and scratch [2*B*n] are fp32 workspaces.  No float atomics reach stats, loss or dlogits: they are the same
 * bits in every launch.  Refused: null pointers, V % 4 != 0, teacher_row_stride < n, tau not finite and > 0, alpha
 * outside [0, 1], inv_batch not finite and > 0, dtypes outside the progen_ce_fwd_bwd combinations. */
int progen_distill_head(const void* logits, int dtype, const float* teacher, long long teacher_row_stride, const int* labels,
                        float* weights, float* scratch, float* stats, float* loss, void* dlogits, int dlogits_dtype, int B,
                        int n, int V, float tau, float alpha, float inv_batch, void* stream);
/* policy-gradient head (DESIGN.md §3.14): policy logits s [B*n, V] in dtype, reference logits z fp32 with row b, position
 * t at ref + (b * ref_row_stride + t) * V (ref_row_stride >= n), labels [B*n], span [B, 2] int32 (lo_b, hi_b) clamped to
 * [0, n] on the device, advantage [B] fp32.  Per position t of S_b = {lo_b <= t < hi_b}, N_b = |S_b|: pi = softmax(s_t),
 * rho = softmax(z_t), logp_t = log pi[label_t] (label clamped to [0, V)), KL_t = sum_v pi_v (log pi_v - log rho_v) (terms
 * whose pi_v underflows to 0 add 0).  L_b = (1 / N_b) sum_{S_b} (-A_b logp_t + beta KL_t); *loss = inv_rows sum_b L_b in
 * double, rows in order (written, not accumulated); stats [B, 3] = (sum_{S_b} logp_t / N_b, sum_{S_b} KL_t / N_b, N_b);
 * dlogits [B*n, V] in dlogits_dtype = inv_rows / N_b [A_b (pi - onehot(label_t)) + beta pi (log pi - log rho - KL_t)]
 * on S_b and +0.0 elsewhere, every row written.  z may be null iff beta == 0; with beta == 0 it is never read, and
 * outside the spans it is never read either.  scratch [2*B*n] is an fp32 workspace.  No float atomics reach stats, loss
 * or dlogits: they are the same bits in every launch, and row b's do not depend on the other rows.  Refused: null
 * pointers, V % 4 != 0, ref_row_stride < n, beta not finite or < 0, beta > 0 with a null z, inv_rows not finite and > 0,
 * dtypes outside the progen_ce_fwd_bwd combinations. */
int progen_policy_head(const void* logits, int dtype, const float* ref, long long ref_row_stride, const int* labels,
                       const int* span, const float* advantage, float* scratch, float* stats, float* loss, void* dlogits,
                       int dlogits_dtype, int B, int n, int V, float beta, float inv_rows, void* stream);
/* out[b, :] = sum_t mask_t x[b, t, :] / sum_t mask_t (fp32, fixed order) over rows of x [B*n, d] (stride ldx), with the
 * same mask as above: for a sequence of L residues, input positions 0..L (BOS and every residue). */
int progen_masked_mean_pool(const void* x, long long ldx, int dtype, const int* labels, float* out, int B, int n, int d,
                            void* stream);
/* backward of progen_masked_mean_pool: dy[b, t, :] = demb[b, :] / count_b at counted positions, 0 at every other position;
 * dy [B*n, d] (stride ldy) in dtype, every row written (no memset needed).  d % 4 == 0, ldy % 4 == 0. */
int progen_masked_mean_pool_bwd(const float* demb, const int* labels, void* dy, long long ldy, int dtype, int B, int n, int d,
                                void* stream);

/* property head on pooled embeddings (all fp32): pred [B, C] = emb [B, d] W [d, C] + bias [C].
 *   regression (C >= 1, targets y [B, C]):        row_loss_b = sum_c (pred_bc - y_bc)^2 / C
 *   classification (C >= 2, classes cls [B]):      row_loss_b = logsumexp(pred_b) - pred_b[cls_b]   (cls clamped to [0, C))
 * *loss = inv_batch * sum_b row_loss_b (inv_batch = 1/global_batch, like progen_ce_fwd_bwd); dpred [B, C] = d loss / d pred;
 * dw [d, C], db [C] and demb [B, d] the gradients of loss.  loss, dw and db are written, not accumulated, and every sum
 * over rows runs in row order without atomics: every output is the same bits in every launch.  With y and cls both null
 * only pred is written (inference) and the other pointers may be null.  C > PROGEN_PROPERTY_MAX_OUTPUTS is refused. */
#define PROGEN_PROPERTY_MAX_OUTPUTS 64
#define PROGEN_TASK_REGRESSION 0
#define PROGEN_TASK_CLASSIFICATION 1
int progen_property_head(const float* emb, const float* w, const float* bias, int B, int d, int C, int task, const float* y,
                         const int* cls, float inv_batch, float* pred, float* row_loss, float* loss, float* dpred, float* dw,
                         float* db, float* demb, void* stream);

/* residue (per-position) head (DESIGN.md §3.11): pred [B*L, C] (fp32) = h [B*L, d] W [d, C] + bias, h the final LayerNorm
 * output in dtype (stride ldh), L any row length of a cut view; a position's prediction does not depend on the other rows.
 * Targets in the same [B*L] layout: y [B*L, C] float (regression; a position is unlabelled when its values are NaN) or
 * cls [B*L] int (classification; -1 = unlabelled).  Training (y or cls non-null, B <= 4096): *count = N, the labelled
 * positions; pos_loss [B*L] (0 where unlabelled); *loss = sum over labelled positions of pos_loss / N, in double, rows in
 * order; dpred [B*L, C] = d loss / d pred (0 where unlabelled); dy [B*L, d] in dtype (stride ldy) = dpred W^T, +0.0 on
 * unlabelled rows, every row written.  Regression pos_loss = sum_c (p - y)^2 / C, classification lse(p) - p[y].  Every
 * sum runs in a fixed order: the outputs are the same bits in every launch.  With y and cls null only pred is written. */
int progen_residue_head(const void* h, long long ldh, int dtype, const float* w, const float* bias, int B, int L, int d, int C,
                        int task, const float* y, const int* cls, float* pred, float* pos_loss, int* count, float* loss,
                        float* dpred, void* dy, long long ldy, void* stream);
/* weight gradient of the residue head: dw [d, C] = sum h^T dpred and db [C] = sum dpred over the labelled positions
 * (unlabelled ones are skipped), written, not accumulated.  Each row's positions are summed in ascending order into
 * workspace [B, (d + 1) C] floats, then the rows in row order: the order does not depend on L, so a cut view and the
 * full-length view of the same rows give the same bits. */
int progen_residue_head_wgrad(const void* h, long long ldh, int dtype, const float* dpred, const float* y, const int* cls,
                              int B, int L, int d, int C, float* workspace, float* dw, float* db, void* stream);

/* backward of apply_rotary_pos_emb (progen.py:36-41) on the [T, ncols] q|k|v gradient, in place */
int progen_rotary_bwd(void* dqkv, long long ld, int dtype, const float* sin_t, const float* cos_t, long long T, int ncols,
                      int seq_len, int dim_head, void* stream);

/* sliding-window attention with one look-back window — progen.py:88-102 (q,k,v already rotated, [T, 3*heads*dim_head]).
 * `_simt`: fp32-exact CUDA-core kernels.  lse / delta: [T, heads] fp32.  The backward needs seq_len % window == 0; the
 * forward takes a partial last window (any seq_len for `_simt`, seq_len % 64 == 0 for `_tc`) and then computes the first
 * seq_len rows of the forward at a longer length, bitwise (causality: no key at or beyond seq_len is read). */
int progen_local_attn_fwd_simt(const void* qkv, void* out, float* lse, int dtype, int B, int seq_len, int window, int heads,
                               int dim_head, void* stream);
int progen_local_attn_bwd_simt(const void* qkv, const void* out, const void* dout, const float* lse, void* dqkv,
                               float* delta, int dtype, int B, int seq_len, int window, int heads, int dim_head,
                               void* stream);
/* the backward over a partial last window (any seq_len > 0), for a training step cut to its rows' counted length: a key
 * streams its own window's queries up to min(window end, seq_len) and the next window's below seq_len.  The rows of a
 * cut call are bitwise the first seq_len rows of the backward at a longer length whose dout is zero from seq_len on.  At
 * whole windows it makes the same launches, with the same bounds, as progen_local_attn_bwd_simt. */
int progen_local_attn_bwd_cut_simt(const void* qkv, const void* out, const void* dout, const float* lse, void* dqkv,
                                   float* delta, int dtype, int B, int seq_len, int window, int heads, int dim_head,
                                   void* stream);

/* tensor-core version (bf16, dim_head 64, window % 64 == 0): flash-style with TMA-fed K/V (or Q/dO) tiles and wgmma,
 * scores stay on chip; same buffers as above.  With rot_sin/rot_cos set, the backward applies the rotary backward to
 * dq|dk|dv in its epilogue. */
int progen_local_attn_fwd_tc(const void* qkv, void* out, float* lse, int B, int seq_len, int window, int heads, int dim_head,
                             void* stream);
int progen_local_attn_bwd_tc(const void* qkv, const void* out, const void* dout, const float* lse, void* dqkv, float* delta,
                             const float* rot_sin, const float* rot_cos, int B, int seq_len, int window, int heads, int dim_head,
                             void* stream);
/* the tensor-core backward over a partial last window (seq_len % 64 == 0, the forward's rule); same contract as
 * progen_local_attn_bwd_cut_simt, same launcher and launches as progen_local_attn_bwd_tc. */
int progen_local_attn_bwd_cut_tc(const void* qkv, const void* out, const void* dout, const float* lse, void* dqkv,
                                 float* delta, const float* rot_sin, const float* rot_cos, int B, int seq_len, int window,
                                 int heads, int dim_head, void* stream);

/* SGU gating — progen.py:182-184: out = xs * (Gp + spatial_biases[m]) and its backward (dxs, dGp, dbias; dbias nullable) */
int progen_sgu_gate_fwd(const void* xs, long long ldx, const void* gp, long long ldg, const float* bias, void* out,
                        long long ldo, int dtype, long long T, int C, int seq_len, void* stream);
int progen_sgu_gate_bwd(const void* ds, long long ldds, const void* xs, long long ldx, const void* gp, long long ldg,
                        const float* bias, void* dxs, long long lddx, void* dgp, long long lddg, float* dbias, int dtype,
                        long long T, int C, int seq_len, void* stream);
/* da *= gelu'(u) (tanh-approximate GELU, jax.nn.gelu default — progen.py:143) */
int progen_gelu_bwd(void* da, const void* u, int dtype, long long numel, void* stream);
int progen_cast_f32(const float* in, void* out, int out_dtype, long long numel, void* stream);
/* out = scale * in, cast to out_dtype (in == out allowed for PROGEN_F32): the scaled compute copy s*B of a low-rank adapter
 * and the scale of its gradient.  numel % 4 == 0, 16-byte aligned buffers. */
int progen_scale_cast_f32(const float* in, void* out, int out_dtype, float scale, long long numel, void* stream);
/* out = tril(spatial_weights) in the act dtype — the mask of progen.py:178-179 applied once per parameter update */
int progen_tril_cast(const float* w, void* out, int out_dtype, int n, void* stream);

/* optimizer: optax.chain(clip_by_global_norm, adamw(mask = ndim > 1), apply_every(k)) — train.py:115-121,189-190 */
int progen_optim_workspace_floats(void);
int progen_grad_sqnorm(const float* g, long long n, float* workspace, float* out_sqnorm, void* stream);
/* one optimizer call.  The step-dependent scalars (Adam count, bias corrections, emit = count % apply_every == 0) live in
 * a 32-byte device `state` ({int64 count; float bc1, bc2; int32 emit; pad}, zeroed before the first call) that a 1-thread
 * kernel advances: every launch argument is step-invariant, so a captured CUDA graph of the whole training step
 * (train.py:186-190) can be replayed.  p_lp (may be null) receives the bf16 mirror of the parameters whenever they change */
int progen_adamw_step(float* p, void* p_lp, const float* g, float* m, float* v, float* acc, long long n, long long n_decay,
                      const float* gnorm_sq, float lr, float b1, float b2, float eps, float wd, float max_norm,
                      int apply_every, void* state, void* stream);

/* ---- KV-cached decode (BASELINE config 5; replaces the full re-forward per token of utils.py:115-117) ----
 * Weights are TRANSPOSED copies ([out, in], fp32 or bf16 per `wdtype`); caches and scratch are fp32 device buffers owned
 * by the caller.  One layer of progen_decode_run_t's `layers`, a DEVICE array of `depth` entries; the cache and state
 * pointers hold all B sequences of the launch, batch-major. */
typedef struct progen_decode_layer_t {
  int32_t kind;                /* 0 GLU, 1 GELU, 2 gMLP/SGU  (progen.py:210-212) */
  int32_t _pad;
  const float* ln1_scale;      /* [d] */
  const void* wqkv_t;          /* [3*inner, d] */
  const void* wo_t;            /* [d, inner] */
  const float* bo;             /* [d] */
  const float* ln2_scale;      /* [d] */
  const void* win_t;           /* [2*hid | hid, d]; GLU: rows [0,hid) value, [hid,2hid) gate */
  const float* bin;
  const void* wout_t;          /* [d, hid | hid/2] */
  const float* bout;           /* [d] */
  const float* sgu_ln_scale;   /* [hid/2] */
  const float* sgu_w;          /* [n, n] fp32 spatial_weights (row p is read up to column p) */
  const float* sgu_b;          /* [n] */
  const void* sgu_proj_t;      /* [hid/2, hid/2] */
  const float* sgu_proj_b;
  float* kcache;               /* [B, heads, n, dim_head] rotated keys (a head's keys are contiguous: the windowed read streams) */
  float* vcache;               /* [B, heads, n, dim_head] rotated values */
  float* shift1;               /* [B, 2, d/2] previous position's LN half (attention block), indexed by position parity */
  float* shift2;               /* [B, 2, d/2] previous position's LN half (feed-forward block) */
  float* gn_hist;              /* [B, n, hid/2] normalised gate history (gMLP layers) */
} progen_decode_layer_t;

/* Whole-generation decode in ONE persistent cooperative kernel (csrc/decode_persist.cu): consumes positions
 * pos0 .. pos0 + nsteps - 1 of B sequences in lock step (reference utils.py:106-135 per sequence; sample.py:66-71).
 * `layers` is a DEVICE array of `depth` progen_decode_layer_t (cache and state layouts above).  Sequence b keeps its
 * prime before start[b]: position p+1 is sampled (seq[b][p+1] += id, quirk Q5) iff p+1 >= start[b].  grid_bar (one uint32) must be zero on entry; att_count ([B * heads] int32) is reserved (the attention
 * merges no longer use a global counter).  Limits: B <= 64, dim_head a power of two in [8, 64], window <= 512, V <= 512,
 * feature widths <= 8192. */
typedef struct progen_decode_run_t {
  int32_t n, d, heads, dim_head, inner, window, hid, V, depth, wdtype, shift_tokens, top_k;
  int32_t B, pos0, nsteps, _pad;
  const float* embed;          /* [V, d] */
  const float* lnf_scale;      /* [d] */
  const void* whead_t;         /* [V, d] */
  const float* bhead;          /* [V] */
  const float* rot_sin;        /* [n, dim_head/2] */
  const float* rot_cos;
  const progen_decode_layer_t* layers;   /* device */
  int32_t* seq;                /* [B, n] token ids; sampled ids are ADDED in place (sampler 0) or written (sampler 1) */
  const int32_t* start;        /* [B] first sampled position of each sequence */
  const float* noise;          /* [B, n, V] gumbel noise, or NULL for the greedy limit */
  float* logits_all;           /* [B, n, V] every step's logits (may be NULL) */
  float* x;                    /* [B, d] residual stream */
  float* q;                    /* [B, inner] */
  float* att;                  /* [B, inner] */
  float* att_part;             /* [B, heads, ceil(2*window/32), dim_head + 4] partial (max, sum, -, -, out) per 32-key slice */
  int32_t* att_count;          /* [B, heads] reserved (non-null) */
  float* u;                    /* [B, hid] */
  float* sg;                   /* [8, B, hid/2] partial spatial gates (up to 8 splits of the history range) */
  float* pj;                   /* [B, hid/2] */
  float* logits;               /* [B, V] */
  uint32_t* grid_bar;          /* grid barrier counter */
  long long* prof;             /* optional [2][160][2] clock64 at entry / exit of every grid barrier of the launch's last
                                  step, for CTA 0 and the last CTA, then [160][8] marks inside CTA 0's phases (NULL: off) */
  /* Sampler selector.  0: the reference sampler above (quirks Q5-Q7, `noise`, seq[b][p+1] += id).  1: the standard sampler:
   * keep the logits >= the top_k-th largest (ties kept; top_k 0 = off), q = softmax(l / temperature) over them, keep the
   * smallest prefix of the q-descending order (ties: lower id first) whose mass reaches top_p, draw the first maximal
   * l / temperature + Gumbel over the kept ids (temperature 0: first maximal raw logit), seq[b][p+1] = id.  The Gumbel noise
   * is Philox4x32-10 generated in the kernel: key (seed lo, seed hi), counter (c >> 2, p + 1, sample_id lo, sample_id hi),
   * word c & 3 = x, u = (2 (x >> 9) + 1) 2^-24, g = -log(-log u).  Drawing id 0 (EOS) sets end[b] = p + 1 and counts the
   * sequence in n_ended; it draws nothing after that (a row with no id to draw, all logits NaN, draws EOS).  When every sequence has ended the launch stops after that position's
   * sampler phase. */
  int32_t sampler;
  float temperature;           /* sampler 1: >= 0, finite; 0 = greedy */
  float top_p;                 /* sampler 1: (0, 1]; 1 = off */
  int32_t _pad1;
  uint64_t seed;               /* sampler 1: Philox key */
  const int64_t* sample_id;    /* [B] sampler 1: each sequence's Philox stream */
  float* token_logp;           /* [B, n] or NULL: log_softmax(logits[p])[seq[p+1]] at [b, p+1] for every drawn p+1 */
  int32_t* end;                /* [B] sampler 1: position of the sampled EOS, n if none (initialised to n by the caller) */
  int32_t* n_ended;            /* sampler 1: sequences that have sampled EOS (zeroed by the caller) */
  int32_t* steps_run;          /* sampler 1: positions this launch consumed */
  /* Sampler-1 constraints, per-draw transforms of the logits l at p before the filter above (sampler 0: neutral only).
   * token_logp stays l[id] - logsumexp(l) of the raw logits.  In fp32: a[c] = l[c] > 0 ? l[c] / repetition_penalty :
   * l[c] * repetition_penalty for every id c present in seq[b] at positions max(1, p + 1 - W) .. p (W = repetition_window,
   * 0 = the whole row; BOS excluded; each id counts once), else a[c] = l[c]; then a += logit_bias (-inf bans an id); then
   * a[0] = -inf while p + 1 < start[b] + min_new_tokens.  The candidates are the ids whose a is neither -inf nor NaN; the
   * filter and the draw above run on a over them (the softmax maximum is the candidates' maximum of a), and a row with
   * none draws EOS.  Off (the unconstrained code) when logit_bias and position_bias (below) are NULL, repetition_penalty
   * is 1 and min_new_tokens is 0; a zero-initialised struct must set repetition_penalty to 1. */
  const float* logit_bias;     /* [V] or NULL */
  float repetition_penalty;    /* finite, > 0; 1 = off */
  int32_t repetition_window;   /* >= 0; 0 = every position since BOS */
  int32_t min_new_tokens;      /* >= 0: the first min_new_tokens draws of a row are never EOS */
  int32_t _pad2;
  /* Row queue (sampler 1, B >= 2; the four pointers NULL and num_rows 0 = no queue): the B sequences of the launch become slots that decode the
   * Q = num_rows rows of a queue.  seq, start, end, token_logp and sample_id are then indexed by the queue row ([Q] /
   * [Q, n]); caches and scratch stay per slot.  Slot b decodes row slot_row[b] (-1: idle) at position slot_pos[b], which
   * it advances by one per step.  A row retires when it draws EOS or position max_length - 1; its slot counts it in
   * `done` and claims q = next_row++: for q < Q the slot restarts at position 0 of row q (slot_pos = 0, token-shift
   * slot 0 of every layer zeroed, x = embedding of seq[q][0]), otherwise it goes idle and writes nothing outside its own
   * caches and scratch.  The launch ends after the sampler phase in which `done` reaches Q, or after nsteps steps
   * (pos0 is not used: positions come from slot_pos).  A row's bits do not depend on its slot or on the other rows, so a
   * queue gives the same rows as launches of B rows each (the attention and SGU plans are those of the batch tile's
   * class).  The caller initialises slot_row[b] = b and slot_pos[b] in [0, max_length - 1) for every slot (Q >= B),
   * next_row = B, done = 0, end[q] = n.  logits_all needs Q == B. */
  int32_t* slot_row;           /* [B] device */
  int32_t* slot_pos;           /* [B] device */
  int32_t* next_row;           /* device: the next unclaimed queue row */
  int32_t* done;               /* device: rows retired */
  int32_t num_rows;            /* Q */
  int32_t max_length;          /* in [2, n]: a row's last drawn position is max_length - 1 (0: n; needed by a queue
                                  and by motif constraints) */
  /* Position-specific bias (sampler 1; both pointers NULL = off): tables of per-offset logit biases.  For the draw of
   * position p + 1 of row r (the queue row when there is a queue), j = p + 1 - start[r] is the 0-based generated offset;
   * if t = position_bias_table[r] >= 0 and j < position_bias_len, a[c] += position_bias[(t * position_bias_len + j) * V
   * + c] in fp32 (its own rounding, no FMA), after the logit bias and before the min_new_tokens EOS ban above.  -inf bans
   * an id at that offset; an offset whose only candidate is one id forces it.  token_logp is unchanged. */
  const float* position_bias;        /* [tables, position_bias_len, V] or NULL */
  const int32_t* position_bias_table;/* [rows]: the table of each row, -1 = none */
  int32_t position_bias_len;         /* in [1, n] when position_bias is set */
  int32_t _pad3;
  /* Motif constraints (sampler 1; NULL = off): a DEVICE progen_motif_t (below).  Needs max_length (above) in [2, n] in
   * static launches too: a row's last drawn position is max_length - 1 with or without a queue. */
  const struct progen_motif_t* motif;
} progen_decode_run_t;

/* Motif constraints of sampler 1 (DESIGN.md §3.3, progen_b200/motif.py): P PROSITE patterns, each of m <= 64 positions
 * (a class of ids, mandatory or optional), matched against a row's generated tokens t_1..t_L.  A row's state is one
 * bitset D per pattern (bit i: positions 0..i match a suffix of the tokens so far, optional positions skipped) and a flags
 * word (bit 0: the required pattern is met).  Reading id c >= 1, with z = !(anchors & 1) || (c is t_1):
 *   D' = closure((((D | (z ? lead : 0)) << 1) | z) & mask[k][c]),  closure(X): X |= (X << 1) & optional until stable.
 * A pattern matches at c when D' has bit `last`.  The required pattern (pattern 0 when required = 1) is met once it
 * matched (anchors & 2, '>': only when it matched at the latest token); its lookahead after c is 0 when met, else
 * need[msb(D')] (D' != 0), need[64] (D' == 0 and the start state stays active), or never.  Per draw at position p + 1 of
 * row r, after every other adjustment above, an id becomes -inf when: c >= 1 and the required pattern's lookahead exceeds
 * the positions left after it, max_length - p - 2; c >= 1 and it completes an avoided pattern (a '>'-anchored one only
 * at p + 1 = max_length - 1); c = 0 while the required pattern is not met, or while the D of a '>'-anchored avoided
 * pattern has bit `last`.  After the draw of a residue, the row's state becomes its D' and flags. */
typedef struct progen_motif_pattern_t {
  uint64_t optional;           /* bit i: position i is optional */
  uint64_t lead;               /* the positions before the first mandatory one (states reached without a residue) */
  uint64_t last;               /* the bit of the pattern's last position */
  uint64_t anchors;            /* bit 0 '<' (at t_1), bit 1 '>' (at t_L) */
} progen_motif_pattern_t;
typedef struct progen_motif_t {
  int32_t num_patterns;        /* P in [1, 9] */
  int32_t required;            /* 1: pattern 0 is required and the others avoided; 0: every pattern is avoided */
  int32_t need[65];            /* required pattern: fewest residues completing it from the state of bit i; [64]: from
                                  the start.  Computed with logit_bias's bans; non-increasing in i; >= 2^30: never */
  int32_t _pad;
  progen_motif_pattern_t pattern[9];
  const uint64_t* mask;        /* [P, V] device: bit i of mask[k * V + c] = id c matches position i of pattern k */
  uint64_t* state;             /* [rows, P + 1] device, zeroed by the caller: row r's D of every pattern, then its flags
                                  (indexed by the queue row when there is a queue) */
} progen_motif_t;

int progen_decode_run(const progen_decode_run_t* run, void* stream);

/* decoder weight refresh (DESIGN.md §3.14): one leaf of a BatchDecoder written in place from device fp32 state.  w is
 * the engine's leaf [in, out] (a vector leaf: in = 1), a [in, rank] and b [rank, out] its adapter (rank 0: none; a and b
 * may then be null).  With c(o) = o, or with interleave = 1 the engine's GLU column order (value_j at 2j, gate_j at
 * 2j + 1, j < out / 2) mapped to haiku's (value | gate): dst [out, in] in dst_dtype (fp32, or bf16 round-to-nearest) =
 * cast(w[i, c(o)] + scale * sum_r a[i, r] b[r, c(o)]), r in increasing order with every product and sum rounded on its
 * own (no FMA): a float32 host replay gives the same bits.  in = 1 is a plain (de-interleaving) copy dst[o] = w[c(o)].
 * Refused: null w or dst, in or out < 1, rank outside [0, 64], rank > 0 with a null a or b, in = 1 or a non-finite
 * scale, interleave with an odd out, dst_dtype not fp32 or bf16. */
int progen_decode_load_weight(const float* w, const float* a, const float* b, int rank, float scale, int in, int out,
                              int interleave, void* dst, int dst_dtype, void* stream);
/* Prefill of the decoder's caches from an inference forward (generation with `prefill='forward'`): a strided row gather
 * with conversion to fp32,
 *   dst[b * dst_b_stride + g * dst_g_stride + r * dst_row_stride + c]
 *     = fp32(src[(row_map[b] * src_seq_rows + row0 + r) * ld + col0 + g * cols + c])
 * for b < B, g < groups, r < rows, c < cols.  src is a forward activation [src_seqs * src_seq_rows, ld] in src_dtype;
 * row_map ([B] int32, device) names the forward sequence of each decoder row (entries are clamped to [0, src_seqs)), so one
 * forward of a prompt fills every row that uses it.  With the caches of progen_decode_run_t: k / v rows 0..P-1 of the
 * rotated q|k|v (col0 = inner or 2 inner, groups = heads, cols = dim_head) into kcache / vcache [B, heads, n, dim_head];
 * LN-output row P, channels [0, d/2), which after the token shift holds position P-1's half, into slot P & 1 of
 * shift1 / shift2 [B, 2, d/2]; normalised-gate rows 0..P-1 into gn_hist [B, n, hid/2].  16-byte source vectors: cols, col0
 * and ld multiples of 4 (fp32) or 8 (bf16), src and dst 16-byte aligned, dst strides multiples of 4.  rows = 0 is a no-op. */
int progen_gather_rows_f32(const void* src, long long ld, int src_dtype, int src_seqs, long long src_seq_rows,
                           const int32_t* row_map, int B, int row0, int rows, int col0, int groups, int cols, float* dst,
                           long long dst_b_stride, long long dst_g_stride, long long dst_row_stride, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* PROGEN_B200_H */
