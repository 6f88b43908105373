/* rp_b200.h - C ABI of librp_b200.so: the H100 (sm_90a) kernels behind RePlay's sequential-recommender hot path.
 *
 * The reference (sb-ai-lab/RePlay @ b4e051e8) has NO FFI on this path: its extension points are Python protocols and
 * Lightning hooks (SURVEY.md §8b).  Each entry point below therefore cites the reference *Python* call it replaces;
 * INTEGRATION.md shows the ctypes stub a RePlay maintainer would add at that call site.
 *
 * Conventions (all functions):
 *   - caller owns all memory; pointers are device pointers unless the name says host; no allocation inside;
 *   - asynchronous with respect to the host, ordered on `stream` (a cudaStream_t / CUstream passed as void*);
 *   - scratch memory is passed in by the caller, sized by the matching *_workspace() function;
 *   - return value: 0 = ok, < 0 = argument / shape / alignment error (RP_E*), > 0 = a cudaError_t;
 *   - never throws, keeps no global mutable state besides cached driver entry points / device attributes;
 *   - bf16 tensors are row-major with 16-byte aligned base and row pitch.
 */
#ifndef RP_B200_H
#define RP_B200_H
#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define RP_OK 0
#define RP_EINVAL (-1)     /* null pointer / unsupported flag */
#define RP_ESHAPE (-2)     /* unsupported size */
#define RP_EALIGN (-3)     /* pointer or pitch not 16-byte aligned */
#define RP_EDRIVER (-4)    /* CUDA driver entry point unavailable / tensor-map encode failed */
#define RP_EWORKSPACE (-5) /* workspace too small */

/* library / build info: returns a static string such as "rp_b200 0.1 sm_90a" */
const char* rp_version(void);

/* ---------------------------------------------------------------------------------------------------------------
 * Predict head:  logits = hq . table^T  ->  seen-item mask  ->  top-K        (one fused pass, logits never stored)
 *   replaces  EmbeddingTyingHead.forward          replay/nn/head.py:29-34
 *                                                  replay/models/nn/sequential/sasrec/model.py:286-307 (legacy)
 *             SeenItemsFilter._compute_scores     replay/nn/lightning/postprocessor/seen_items.py:56-83
 *             RemoveSeenItems._compute_scores     replay/models/nn/sequential/postprocessors/postprocessors.py:55-95
 *             torch.topk(logits, k, dim=1)        replay/nn/lightning/callback/predictions_callback.py:90
 *                                                  replay/models/nn/sequential/callbacks/prediction_callbacks.py:93
 * ------------------------------------------------------------------------------------------------------------- */

/* seen_ids int64 [n_users, S] (any order, duplicates allowed, ids outside [0,item_count) are padding)
 *   -> out_sorted int32 [n_users, S], ascending, padding = INT32_MAX.
 * inv_map (optional, int32 [item_count]): position of each item in candidates_to_score, -1 if absent; when given the
 * output holds candidate positions instead of item ids (seen_items.py:68-71,80-81).
 * 1 <= S <= 4096 (one block sorts a user's list in shared memory), else RP_ESHAPE.  rp_score_topk takes any S: the
 * Python wrapper (ops.seen_prepare) prepares longer lists with a device-side sort to the same contract. */
int rp_seen_prepare(const int64_t* seen_ids, int n_users, int S, int item_count, const int32_t* inv_map,
                    int32_t* out_sorted, void* stream);

/* Workspace of rp_score_topk.  K <= 32: per (user, item split, 32-column part) sorted partial lists of K (score, column)
 * pairs.  32 < K <= 1024: per (user, item split) a buffer of C = max(2K, K + 64) rounded up to a power of two keys
 * (8 bytes each) and its count; the item splits are capped so that one user's buffers hold at most 65 536 keys, and the
 * size never decreases as n_users or K grows.  Both: one shared admission threshold per user. */
size_t rp_score_topk_workspace(int n_users, int n_items, int d, int K);

/* hq bf16 [n_users, d]; table bf16 [n_items, d] (the rows that are scored: all items, or the gathered candidates);
 * bias fp32 [round_up(n_items,128)] or NULL (BERT4Rec head); seen_sorted from rp_seen_prepare or NULL (no filter); candidates int64 [n_items] or NULL
 * (maps a scored column back to an item id, predictions_callback.py:91-92).
 * out_ids int64 [n_users, K], out_scores fp32 [n_users, K], sorted by (score desc, column asc), exact and bit-identical
 * from run to run.  When fewer than K columns are unmasked, the remaining slots hold the user's masked columns in
 * ascending order (then -1) with score -inf.
 * d in {64,128,256,512}; 1 <= K <= min(1024, n_items), else RP_ESHAPE.  K <= 32 keeps a sorted list per thread in
 * registers; larger K admits candidates into workspace buffers that are compacted to K entries by a radix select. */
int rp_score_topk(const void* hq, const void* table, const float* bias, const int32_t* seen_sorted, int S, int n_users,
                  int n_items, int d, int K, const int64_t* candidates, int64_t* out_ids, float* out_scores,
                  void* workspace, size_t workspace_bytes, void* stream);

/* ---------------------------------------------------------------------------------------------------------------
 * Training head: full-catalog cross entropy fused with the logits GEMM, forward and backward
 *   replaces  logits = hidden . E^T                 replay/nn/head.py:29-34 ; replay/nn/sequential/sasrec/model.py:258-265
 *             torch.nn.CrossEntropyLoss (mean)       replay/nn/loss/ce.py:49-81
 *                                                    replay/models/nn/sequential/sasrec/lightning.py:335-355
 *                                                    replay/models/nn/sequential/bert4rec/lightning.py:332-351
 *             and autograd's backward of both.
 * hc bf16 [capacity, d]: hidden rows of the VALID targets, compacted (rows >= *n_valid are ignored but must be finite);
 * table bf16 [n_items, d] (tied item table or the untied Linear weight); bias fp32 [round_up(n_items,128)] or NULL
 * (bert4rec/model.py:363-382: logits = F.linear(h, W, b)); d_bias fp32 [n_items] is overwritten when bias is given;
 * labels int32 [capacity]; n_valid int32 [1] IN DEVICE MEMORY (keeps the step graph-capturable).
 * ------------------------------------------------------------------------------------------------------------- */
size_t rp_ce_head_workspace(int capacity_tokens, int n_items, int d);

/* loss_out fp32 [2] = { mean CE over the valid targets, 1 / n_valid }; lse fp32 [capacity];
 * cvec fp32 [round_up(capacity,128)], 16-byte aligned (per-token exponent offsets for the backward; entries >= capacity
 * must be -inf).
 * d_hc (optional, bf16 [capacity, d], d <= 256): enables the FUSED training path - a single pass accumulates the row sums of
 * exp(s) against a fixed reference maximum together with the un-normalised gradient sum_i exp(s_i) E_i, so the separate
 * log-sum-exp pass disappears and d_hc is final after this call.  A device-side Cauchy-Schwarz bound on |s| guards the
 * trick; when it fails the two-pass kernels run instead (both variants are enqueued, the losing one exits immediately), so
 * the call stays CUDA-graph capturable.  n_valid_hint: host estimate of *n_valid (0 = unknown), load-balance only. */
int rp_ce_head_fwd(const void* hc, const void* table, const float* bias, const int32_t* labels, const int32_t* n_valid,
                   int capacity, int n_items, int d, float* loss_out, float* lse, float* cvec, void* d_hc, int n_valid_hint,
                   void* workspace, size_t workspace_bytes, void* stream);

/* gradients of the mean CE for d(loss) = 1:  d_hc bf16 [capacity, d] (rows < *n_valid; already produced by the forward when
 * `fused` != 0 and the bound held, otherwise computed here); d_table fp32 [n_items, d] is OVERWRITTEN (softmax part) and
 * then atomically corrected by the one-hot part; d_bias fp32 [n_items] likewise iff bias.  `fused` must equal
 * (d_hc != NULL) of the matching forward call and then needs the same workspace.  d in {64,128,256}: fused wgmma passes
 * (logits never leave the registers).  d = 512: a [128 x 512] fp32 accumulator does not fit them, so the softmax numerators
 * of a token chunk are materialised in bf16 inside the workspace (chunk sized by RP_CE_WIDE_G_BYTES, default 8 GiB) and
 * three GEMMs per chunk produce dH and dE; with a bias, a fixed-order column sum of each chunk gives d_bias (bitwise
 * reproducible).  The workspace is then always required.
 * n_valid_hint: host estimate of *n_valid (0 = unknown), load-balance only. */
/* Per-row variants of the full-catalog head, single positive label per position:
 *   row_weight  fp32 [capacity], >= 0, in the compacted order of the valid targets (NULL = 1): loss = mean_t w_t ce_t
 *               replaces  replay/nn/loss/logout_ce.py:148-228 LogOutCEWeighted (and :10-145 LogOutCE = the plain head) ;
 *                         replay/nn/loss/ce.py:84-143 CEWeighted
 *   loss_kind 1 LogInCE   replay/nn/loss/login_ce.py:102-239: loss_t = -clamp(log(p_t + log_eps), -clamp, clamp) with p_t the
 *               softmax probability of the positive over the catalog; gradient = CE gradient of the row x p / (p + eps)
 * Same buffers and fused behaviour as rp_ce_head_fwd; rp_ce_head_bwd with the same workspace completes it. */
int rp_ce_head_fwd_w(const void* hc, const void* table, const float* bias, const int32_t* labels, const int32_t* n_valid,
                     int capacity, int n_items, int d, float* loss_out, float* lse, float* cvec, void* d_hc, int n_valid_hint,
                     const float* row_weight, int loss_kind, float log_eps, float clamp, void* workspace,
                     size_t workspace_bytes, void* stream);
int rp_ce_head_bwd(const void* hc, const void* table, const float* bias, const int32_t* labels, const int32_t* n_valid,
                   int capacity, int n_items, int d, const float* loss_out, const float* cvec, void* d_hc, float* d_table,
                   float* d_bias, int fused, int n_valid_hint, void* workspace, size_t workspace_bytes, void* stream);

/* Full-catalog BCE head, single positive label per position, over the same buffers (workspace: rp_ce_head_workspace):
 *   replaces  BCEWithLogitsLoss(reduction="sum")(logits, onehot(y)) / T_v     replay/nn/loss/bce.py:10-95
 *                                                   replay/models/nn/sequential/bert4rec/lightning.py:273-305
 *   loss_out fp32 [2] = { sum_t [sum_i softplus(x_ti) - x_t,y_t] / T_v, 1 / T_v },  x = hc . table^T (+ bias).
 * The sigmoid is bounded: no log-sum-exp, no bound guard, no second pass.  d_hc (optional, d <= 256) enables the fused
 * forward + dH pass; loss and d_hc are bitwise reproducible.  The backward overwrites d_table (and d_bias iff bias) with
 * (sigmoid - onehot)^T . hc / T_v and its column sums; `fused` must equal (d_hc != NULL && d <= 256) of the forward.
 * d in {64,128,256,512} with or without bias (512: materialised sigmoid chunks, rp_gemm act 4).  The BCE head reads
 * bias entries < n_items only, so a bias of exactly n_items entries is enough here. */
int rp_bce_head_fwd(const void* hc, const void* table, const float* bias, const int32_t* labels, const int32_t* n_valid,
                    int capacity, int n_items, int d, float* loss_out, void* d_hc, int n_valid_hint, void* workspace,
                    size_t workspace_bytes, void* stream);
int rp_bce_head_bwd(const void* hc, const void* table, const float* bias, const int32_t* labels, const int32_t* n_valid,
                    int capacity, int n_items, int d, const float* loss_out, void* d_hc, float* d_table, float* d_bias,
                    int fused, int n_valid_hint, void* workspace, size_t workspace_bytes, void* stream);
/* Positive SETS for the full-catalog BCE head (replay/nn/loss/bce.py:51-95 with num_positives > 1, no bias): the target of
 * row t is 1 at every distinct id in [0, n_items) among labels_p [capacity, num_positives] (rp_prepare_batch_multi; the
 * slot mask is not read), labels[t] being one of them.  rp_bce_head_fwd / _bwd on labels score labels[t]; then
 *   rp_bce_head_multi_fwd  loss_out[0] -= loss_out[1] x sum of the other ids' logits (row_sum fp32 [capacity] scratch;
 *                          rows summed in a fixed order)
 *   rp_bce_head_multi_bwd  d_hc[t] -= loss_out[1] x sum of their table rows (bf16, read-modify-write),
 *                          d_table[y] -= loss_out[1] x hc[t] (fp32 atomics)
 * Ids outside [0, n_items) are skipped (the reference's scatter_ fails on them). */
int rp_bce_head_multi_fwd(const void* hc, const void* table, const int32_t* labels, const int32_t* labels_p,
                          const int32_t* n_valid, int capacity, int num_positives, int n_items, int d, float* loss_out,
                          float* row_sum, void* stream);
int rp_bce_head_multi_bwd(const void* hc, const void* table, const int32_t* labels, const int32_t* labels_p,
                          const int32_t* n_valid, int capacity, int num_positives, int n_items, int d, const float* loss_out,
                          void* d_hc, float* d_table, void* stream);

/* ---------------------------------------------------------------------------------------------------------------
 * Transformer body.  All activations are token-major bf16 [T = B*L, d]; weights are the bf16 shadow of the fp32 masters.
 * ------------------------------------------------------------------------------------------------------------- */

/* Generic batched GEMM  C[m,n] = epilogue(alpha * sum_k A(m,k) B(n,k))  on wgmma.
 *   replaces  torch.nn.MultiheadAttention in/out projections   replay/nn/sequential/sasrec/transformer.py:36-46,99-106
 *             Conv1d(d,d,1) / Linear FFN layers                  replay/nn/ffn.py:43-57 ; models/nn/sequential/sasrec/model.py:490-506
 *                                                                models/nn/sequential/bert4rec/model.py:516-527
 *             and autograd's backward of all of them (dX = dY.W, dW = dY^T.X read in place through MN-major descriptors).
 * Operand X is a 2-D bf16 array [x_rows, x_cols] with pitch ldx; x_mn = 0: stored [M or N rows, K cols] (K-major),
 * x_mn = 1: stored [K rows, M or N cols].  Batch element bz = outer*inner + in addresses rows r0 + outer*ro + in*ri and
 * columns c0 + outer*co + in*ci.  C: element offset c_off0 + outer*c_oo + in*c_oi, row pitch ldc.
 * The contraction runs over whole 64-element chunks of the STORED array: with K % 64 != 0 the tail reads the elements
 * that follow the batch element's K range inside [x_rows, x_cols] (e.g. the next batch element's rows or columns); only
 * elements past the stored array read as 0.  Callers that contract over a padded length (the
 * attention backwards over L with b_off = (0, L, ...)) keep the pad columns of the other operand zero.
 * out_mode 0: bf16 store, 1: fp32 atomic add (split_k >= 1), 2: fp32 store, 3: fp32 store of the split-K partial at
 * C + ksplit * c_split_stride (deterministic two-stage split-K; reduce with rp_reduce_splits), 4: fp32 C += x as a plain
 * read-modify-write (split_k == 1, every element has one owner).  K split s covers chunks [kc*s/S, kc*(s+1)/S) of the
 * kc = ceil(K_eff / 64) chunks; a split with no chunk stores (out_mode 3) or adds (out_mode 1) zeros.  Every split runs
 * the epilogue on its partial sum, so split_k > 1 takes only alpha and rowmask: bias, act, residual, gate, C2, drop_p or
 * post_drop_p with split_k > 1 is RP_EINVAL.
 * Epilogue order: alpha, bias[N], act (0 none, 1 ReLU, 2 GELU-erf, 3 exp2 with a per-row offset, 4 sigmoid times 2^(per-row
 * offset): x = sigmoid(x) * exp2(row_exp2_offset[m]), exactly 0 where the offset is -inf; act 4 takes K-major operands
 * only), Philox dropout (drop_p; seed + *seed_ptr, drop_offset, element (row bz*M + m, column n) of the stream of
 * csrc/rp_philox.cuh: drop_row_key / drop_col_key / drop_mix), gate (x *= gate != 0 ? gate_scale : 0, same geometry as C),
 * residual (bf16, same geometry as C), post-residual dropout (post_drop_p, post_drop_offset, same row and column keys),
 * rowmask[rowmask_off0 + outer*rowmask_oo + m] (indexed by outer, not by in).
 * row_exp2_offset is indexed by m alone, whatever the batch element.
 * C2 (optional, bf16, geometry of C) receives the value after the bias and before the activation; gate_mode 1 multiplies
 * by gelu'(gate) instead of the (gate != 0) test.
 * Left untouched: rows >= M, columns >= N, the pitch padding of every row, and all of a 128-row tile that m_limit skips
 * (in every split's partial too).
 * Alignment (RP_EALIGN): A, B 16-byte aligned with lda, ldb and the column offsets c0, co, ci multiples of 8; out_mode 0: C 16-byte aligned and ldc, c_off0,
 * c_oo, c_oi multiples of 8; a residual: 16-byte aligned with ldc and the C offsets multiples of 8; C2: 4-byte aligned with
 * ldc and the C offsets even. */
typedef struct rp_gemm_desc {
  const void* A; long long a_rows, a_cols, lda; int a_mn;
  const void* B; long long b_rows, b_cols, ldb; int b_mn;
  int M, N, K, batch, inner;
  int a_r0, a_ro, a_ri, a_c0, a_co, a_ci;
  int b_r0, b_ro, b_ri, b_c0, b_co, b_ci;
  void* C; long long ldc, c_off0, c_oo, c_oi; int out_mode;
  float alpha; const float* bias; int act;
  const void* residual; const uint8_t* rowmask; long long rowmask_off0, rowmask_oo;
  float drop_p; unsigned long long seed, drop_offset; const unsigned long long* seed_ptr;
  int split_k;
  const void* gate; float gate_scale;
  void* C2; int gate_mode; float post_drop_p; unsigned long long post_drop_offset;
  long long c_split_stride;
  const float* row_exp2_offset;                    /* act 3: x = exp2(x * log2(e) + row_exp2_offset[m]); act 4: see above */
  const int32_t* m_limit_dev; int m_limit_base;    /* device scalar: 128-row tiles with m0 + base >= *limit are skipped */
  const int32_t* k_limit_dev; int k_limit_base;    /* device scalar: the contraction stops at *limit - base, rounded up to
                                                      a whole 64-element chunk (operands beyond the limit must be finite) */
} rp_gemm_desc;
int rp_gemm(const rp_gemm_desc* g, void* stream);
/* dst[i] (+)= sum_s src[s * stride + i], i < n (n, stride multiples of 4) */
int rp_reduce_splits(const float* src, int n_splits, long long stride, long long n, float* dst, int accumulate, void* stream);

/* Fused multi-head attention forward for L <= 512, head_dim in {64,128}: S = Q.K^T, causal / key-padding mask derived
 * from pad_mask (no [B*H,L,L] mask tensor), softmax, dropout, O = P.V.  Q, K and V of a 128-query tile stay in shared
 * memory, except at head_dim 128 with L > 256, where V streams through a ring of 64-key stages (same outputs and saves).
 *   replaces  torch.nn.MultiheadAttention's SDPA core + replay/nn/mask.py:18-51 (new path: causal & pad keys masked)
 *             models/nn/sequential/sasrec/model.py:229-231,435 (legacy: causal only) ; bert4rec/model.py:494 (pad keys only)
 * q/k/v: 2-D bf16 arrays whose rows are tokens; head h reads columns x_c0 + h*head_dim.  out: bf16 [B*L, ldo].
 * p_save (optional) bf16 [B*H, Lp, Lp] receives exp(s - rowmax) (Lp = round_up(L,64), must be zero-initialised once),
 * inv_sum fp32 [B*H, Lp] the reciprocal row sums - the inputs of rp_attn_softmax_bwd. */
typedef struct rp_attn_desc {
  const void* q; long long q_rows, q_cols, ldq; int q_c0;
  const void* k; long long k_rows, k_cols, ldk; int k_c0;
  const void* v; long long v_rows, v_cols, ldv; int v_c0;
  int B, H, L, head_dim;
  int causal, mask_pad_keys;
  const uint8_t* pad_mask;
  void* out; int ldo;
  void* p_save; float* inv_sum;
  float drop_p; unsigned long long seed, drop_off; const unsigned long long* seed_ptr;
  float* m_save;  /* optional fp32 [B*H, Lp]: row max in exp2 units, input of rp_attn_bwd */
  float scale;    /* softmax scale; 0 -> 1/sqrt(head_dim).  Padded head slots (true head_dim 32 / 48 / 50 inside a 64-wide
                     slot) pass 1/sqrt(true head_dim) */
  /* Packed rows (causal, head_dim 64, L <= 256; both or neither, NULL = padded rows b*L + position): sequence b holds its
   * positions seq_first[b] .. L-1 in rows seq_off[b] ... of q / k / v / out (rp_row_plan).  Masks and dropout stay keyed
   * by position; inv_sum / m_save row i is position (seq_first[b] & ~63) + i. */
  const int32_t* seq_first; const int32_t* seq_off;
} rp_attn_desc;
int rp_attn_fwd(const rp_attn_desc* a, void* stream);

/* Fused attention backward (L <= 256, head_dim 64), one CTA per (sequence, head): recomputes S^T = K.Q^T and
 * dP^T = V.dO^T on wgmma, forms P / dS in registers from the forward's row statistics (m_save, inv_sum) and accumulates
 * dV = Pd^T.dO, dK = dS^T.Q, dQ = dS.K with the bf16 operands as register A operands (deterministic) - the [B*H, L, L]
 * matrices of the un-fused path are never written.  Replaces autograd's backward of the SDPA core of
 * torch.nn.MultiheadAttention (replay/nn/sequential/sasrec/transformer.py:99-106 ; bert4rec/model.py:494).
 * q/k/v/d_out/out: token-major 2-D bf16 arrays; dq/dk/dv: outputs (rows b*L + i, columns x_c0 + h*64). */
typedef struct rp_attn_bwd_desc {
  const void* q; long long q_rows, q_cols, ldq; int q_c0;
  const void* k; long long k_rows, k_cols, ldk; int k_c0;
  const void* v; long long v_rows, v_cols, ldv; int v_c0;
  const void* d_out; long long do_rows, do_cols, ld_do;
  const void* out; int ldo;
  int B, H, L, head_dim;
  int causal, mask_pad_keys;
  const uint8_t* pad_mask;
  const float* m_save; const float* inv_sum;
  void* dq; int ld_dq, dq_c0;
  void* dk; int ld_dk, dk_c0;
  void* dv; int ld_dv, dv_c0;
  float drop_p; unsigned long long seed, drop_off; const unsigned long long* seed_ptr;
  float scale;    /* as in rp_attn_desc */
  const int32_t* seq_first; const int32_t* seq_off;   /* packed rows as in rp_attn_desc; dq / dk / dv rows likewise */
} rp_attn_bwd_desc;
int rp_attn_bwd(const rp_attn_bwd_desc* a, void* stream);

/* Softmax backward between the batched attention-backward GEMMs (un-fused path, any supported head_dim): in place, dpd := dS = P*(dP - sum P*dP)*scale and
 * p_save := P*dropmask/keep (the A operand of dV). */
int rp_attn_softmax_bwd(void* p_save, void* dpd, const float* inv_sum, int BH, int L, float scale, float drop_p,
                        unsigned long long seed, unsigned long long drop_off, const unsigned long long* seed_ptr,
                        void* stream);

/* predict(): attention of ONE query row per (sequence, head) - the last position - against that sequence's keys
 * (SasRec.forward_inference keeps only hidden[:, -1, :], nn/sequential/sasrec/model.py:301; legacy model.py:157).
 * q, out: compact bf16 [B, H*head_dim]; k, v: token-major 2-D arrays (rows b*L + j, head h at columns x_c0 + h*head_dim). */
int rp_attn_last(const void* q, const void* k, const void* v, long long ldk, long long ldv, int k_c0, int v_c0,
                 const uint8_t* pad_mask, int B, int H, int L, int head_dim, int mask_pad_keys, void* out, float scale /* 0: 1/sqrt(head_dim) */,
                 void* stream);

/* int64 ids / bool masks of one [B, L] batch -> int32 ids (pads -> pad_id) and the compacted valid-target list
 * (replaces the masked_fill / boolean-index preparation in nn/loss/ce.py:70-80 and models/.../sasrec/model.py:236-239).
 * labels/target_mask may be NULL (predict). */
int rp_prepare_batch(const int64_t* ids, const uint8_t* pad_mask, const int64_t* labels, const uint8_t* target_mask, int T,
                     int pad_id, int n_items, int32_t* ids32, int32_t* valid_idx, int32_t* labels_c, int32_t* n_valid,
                     int32_t* scratch /* >= ceil(T/1024) ints, needed with targets */, void* stream);

/* Multi-positive targets (replay/nn/loss/base.py:49-154): labels int64 / target_mask bool [T, num_positives], 1 <=
 * num_positives <= RP_MAX_POSITIVES.  A position is live when one of its slots has the mask set and an id in [0, n_items);
 * live_mask [T] and live_label [T] (its first such id) are written and then compacted by rp_prepare_batch into valid_idx /
 * labels_c / n_valid (pass live_label / live_mask to rp_row_plan).  For compacted row t < *n_valid, labels_p[t*P + k] is
 * slot k's raw id saturated to int32 and slot_mask[t*P + k] = mask set and id in [0, n_items); *n_pairs = number of set
 * slot_mask entries.  All on the device. */
#define RP_MAX_POSITIVES 32
int rp_prepare_batch_multi(const int64_t* ids, const uint8_t* pad_mask, const int64_t* labels, const uint8_t* target_mask,
                           int T, int num_positives, int pad_id, int n_items, int32_t* ids32, int64_t* live_label,
                           uint8_t* live_mask, int32_t* valid_idx, int32_t* labels_c, int32_t* labels_p, uint8_t* slot_mask,
                           int32_t* n_valid, int32_t* n_pairs, int32_t* scratch, void* stream);

/* Row plan of a causal training batch (packed body): seq_first[b] = first position of sequence b whose pad_mask is set or
 * that holds a valid target (L if none); the positions seq_first[b] .. L-1 of all sequences are packed back to back:
 * seq_off[b] = first packed row, *n_rows = packed row count, row_tok[r] = token b*L + position of packed row r,
 * valid_rows[k] = packed row of valid_idx[k] (k < *n_valid; valid_idx may be NULL).  All on the device. */
int rp_row_plan(const uint8_t* pad_mask, const int64_t* labels, const uint8_t* target_mask, int B, int L, int n_items,
                const int32_t* valid_idx, const int32_t* n_valid, int32_t* seq_first, int32_t* seq_off, int32_t* n_rows,
                int32_t* row_tok, int32_t* valid_rows, void* stream);

/* x[t] = table[ids[t]] * scale + pos[pos0 + t % L] -> dropout -> (zero pad rows)      nn/sequential/sasrec/agg.py:37-53,
 * models/nn/sequential/sasrec/model.py:346-357 ; and its backward (fp32 atomics into d_table, pad row frozen).
 * pos / d_pos NULL: no positional term (TiSASRec's item input, model.py:597-604), and no positional gradient. */
int rp_embed_fwd(const void* table, const float* pos, const int32_t* ids, const uint8_t* pad_mask, int T, int L, int d,
                 int pos0, float scale, int zero_pad_rows, float drop_p, unsigned long long seed, unsigned long long drop_off,
                 const unsigned long long* seed_ptr, void* out, void* stream);
int rp_embed_bwd(const void* dx, const int32_t* ids, const uint8_t* pad_mask, int B, int L, int d, int pad_id, int pos0,
                 float scale, int zero_pad_rows, float drop_p, unsigned long long seed, unsigned long long drop_off,
                 const unsigned long long* seed_ptr, float* d_table, float* d_pos, void* stream);
/* The same on packed rows (rp_row_plan): row r < *n_rows_dev is token row_tok[r]; dropout keyed by the token.  T = capacity. */
int rp_embed_fwd_rows(const void* table, const float* pos, const int32_t* ids, const uint8_t* pad_mask, const int32_t* row_tok,
                      const int32_t* n_rows_dev, int T, int L, int d, int pos0, float scale, int zero_pad_rows, float drop_p,
                      unsigned long long seed, unsigned long long drop_off, const unsigned long long* seed_ptr, void* out,
                      void* stream);
int rp_embed_bwd_rows(const void* dx, const int32_t* ids, const uint8_t* pad_mask, const int32_t* row_tok,
                      const int32_t* n_rows_dev, const int32_t* seq_first, const int32_t* seq_off, int B, int L, int d,
                      int pad_id, int pos0, float scale, int zero_pad_rows, float drop_p, unsigned long long seed,
                      unsigned long long drop_off, const unsigned long long* seed_ptr, float* d_table, float* d_pos,
                      void* stream);

/* SASRec input with side features (nn/embedding.py SequenceEmbedding + nn/agg.py SumAggregator, csrc/rp_features.cu):
 *   x[r] = dropout((table[ids[t]] + sum_f term_f(t)) * scale + pos[pos0 + t % L]),  t = r or row_tok[r] (packed rows)
 * with the dropout stream of rp_embed_fwd (row key = token t).  Feature kinds and their term:
 *   RP_FEAT_CAT       values int32 [T]:    table[v] (bf16 [n_rows, d]); v == padding_value or outside [0, n_rows): zero
 *   RP_FEAT_BAG_SUM   values int32 [T, K]: sum of table[v_j] over the non-padding entries (torch.nn.EmbeddingBag "sum")
 *   RP_FEAT_BAG_MEAN  the same divided by their count; an all-padding bag gives zero ("mean")
 *   RP_FEAT_NUM       values fp32 [T, K]:  v . W^T + b, table = W fp32 [d, K] (padded rows zero), bias fp32 [d]
 *   RP_FEAT_IDENT     values fp32 [T, K]:  v itself, K = the true hidden size (scattered into the head slots by hd_valid)
 * Numerical features take consecutive val_col ranges (0, K0, K0 + K1, ...), at most RP_FEAT_MAX_NUM_COLS columns in all.
 * Backward (the item table and the positions stay with rp_embed_bwd / _rows): dS = scale * dropout'(dx) is added into each
 * categorical d_table row (fp32 atomics, padding rows untouched, mean bags scaled by 1 / count).  With numerical features
 * it also writes d_s bf16 [rows, d] = dS and v_rows bf16 [rows, v_ld] (numerical values at their val_col, other columns
 * zero), the operands of rp_wgrad_group for dW = dS^T . V and db = column sums of dS.  v_ld a multiple of 8.
 * RP_EINVAL: null pointer, unknown kind, drop_p outside [0, 1); RP_ESHAPE: d, hd_valid, n_feats, widths, val_col, v_ld. */
#define RP_FEAT_MAX 16
#define RP_FEAT_MAX_NUM_COLS 64
#define RP_FEAT_CAT 0
#define RP_FEAT_BAG_SUM 1
#define RP_FEAT_BAG_MEAN 2
#define RP_FEAT_NUM 3
#define RP_FEAT_IDENT 4
typedef struct rp_feature {
  int kind, width, n_rows, padding_value, val_col;
  const void* values;
  const void* table;
  const float* bias;
  float* d_table;
} rp_feature;
int rp_feature_embed_fwd(const void* item_table, const float* pos, const int32_t* ids, const rp_feature* feats, int n_feats,
                         int T, int L, int d, int hd_valid, int pos0, float scale, float drop_p, unsigned long long seed,
                         unsigned long long drop_off, const unsigned long long* seed_ptr, void* out, void* stream);
int rp_feature_embed_fwd_rows(const void* item_table, const float* pos, const int32_t* ids, const rp_feature* feats,
                              int n_feats, const int32_t* row_tok, const int32_t* n_rows_dev, int T, int L, int d, int hd_valid,
                              int pos0, float scale, float drop_p, unsigned long long seed, unsigned long long drop_off,
                              const unsigned long long* seed_ptr, void* out, void* stream);
int rp_feature_embed_bwd(const void* dx, const rp_feature* feats, int n_feats, int T, int d, int hd_valid, float scale,
                         float drop_p, unsigned long long seed, unsigned long long drop_off, const unsigned long long* seed_ptr,
                         void* d_s, void* v_rows, int v_ld, void* stream);
int rp_feature_embed_bwd_rows(const void* dx, const rp_feature* feats, int n_feats, const int32_t* row_tok,
                              const int32_t* n_rows_dev, int T, int d, int hd_valid, float scale, float drop_p,
                              unsigned long long seed, unsigned long long drop_off, const unsigned long long* seed_ptr,
                              void* d_s, void* v_rows, int v_ld, void* stream);
/* The BERT form (legacy BERT4Rec's BertEmbedding with side features, bert4rec/model.py:173-296):
 *   x[t] = dropout(where(tok_mask[t], table[ids[t]] + sum_f term_f(t), mask_emb) + pos[t % L])
 * with no scale, pos == NULL for no positional term, and the dropout stream of rp_bert_embed_fwd (row key = token t), so
 * all-zero side tables and values give exactly rp_bert_embed_fwd's output.  Kinds RP_FEAT_CAT and RP_FEAT_IDENT only; any
 * other kind is RP_EINVAL.  A BERT categorical table has no padding row: pass padding_value = -1, so every id in
 * [0, n_rows) is a row.  An id outside [0, n_rows) adds zero (the reference raises IndexError there).  T a multiple of L.
 * Backward (the item table, mask_emb and pos stay with rp_bert_embed_bwd): dS = dropout'(dx) is added into each categorical
 * d_table row with fp32 atomics, at tokens with pad_mask && tok_mask only; identity features take no gradient. */
int rp_bert_feature_embed_fwd(const void* item_table, const void* mask_emb, const float* pos, const int32_t* ids,
                              const uint8_t* tok_mask, const rp_feature* feats, int n_feats, int T, int L, int d, int hd_valid,
                              float drop_p, unsigned long long seed, unsigned long long drop_off,
                              const unsigned long long* seed_ptr, void* out, void* stream);
int rp_bert_feature_embed_bwd(const void* dx, const uint8_t* pad_mask, const uint8_t* tok_mask, const rp_feature* feats,
                              int n_feats, int T, int d, int hd_valid, float drop_p, unsigned long long seed,
                              unsigned long long drop_off, const unsigned long long* seed_ptr, void* stream);
/* SASRec input through ConcatAggregator (nn/agg.py:56-109 ; nn/sequential/sasrec/agg.py:37-53), every feature at its own
 * width w_f:
 *   X[r] = [segments | 0],  Y = X . W^T + b (rp_gemm, fp32 [rows, d], W bf16 [d, kp]),  x[r] = dropout(Y[r] * scale + pos[pos0 + t % L])
 * rp_concat_gather(_rows) writes X bf16 [rows, kp]: the item's true hidden features (padded columns skipped by hd_valid) at
 * columns item_col.., feature k's w_f = seg_dim[k] values at seg_col[k]..; columns past the segments are zero.  Segment
 * terms, each summed in fp32 and rounded to bf16 once:
 *   RP_FEAT_CAT / _BAG_SUM / _BAG_MEAN   as in rp_feature_embed_fwd, over table bf16 [n_rows, w_f]
 *   RP_FEAT_NUM                          v . W_f^T + b_f, table = W_f fp32 [w_f, K], bias fp32 [w_f] (val_col consecutive)
 *   RP_FEAT_IDENT                        v itself, K == w_f
 * The segments must tile [0, width) exactly and kp be a multiple of 64 with width <= kp <= RP_CONCAT_MAX_COLS.
 * rp_concat_embed_fwd is the elementwise pass after the projection; its dropout is rp_embed_fwd's stream (row key = token t),
 * so a concat model drops the elements its item-only model drops.  rp_gemm's epilogue cannot take it: its bias comes after
 * alpha, it has no per-position row and its dropout is keyed by the output row, which is not the token on packed rows.
 * Backward: dY = scale * dropout'(dx) (rp_feature_embed_bwd with no features writes it as d_s), dX = dY . W (rp_gemm),
 * rp_concat_scatter adds dX's item segment into d_item fp32 [., d] (pad_id frozen) and each categorical segment into its
 * d_table fp32 [n_rows, w_f] (fp32 atomics, padding rows frozen, mean bags by 1 / count) and stages the numerical values
 * in v_rows as rp_feature_embed_bwd does; rp_wgrad_group gives dW / db of the projection (dY^T . X) and of the numerical
 * features (dX^T . v_rows, their block at (seg_col, val_col)); rp_embed_pos_bwd gives the positions.
 * row_tok / n_rows_dev: both (packed rows, *n_rows_dev of the T rows) or neither.  RP_EINVAL: null pointer, unknown kind,
 * drop_p outside [0, 1); RP_ESHAPE: d, hd_valid, n_feats, segments, kp, widths, val_col, v_ld. */
#define RP_CONCAT_MAX_COLS 1024
int rp_concat_gather(const void* item_table, const int32_t* ids, const rp_feature* feats, const int* seg_col, const int* seg_dim,
                     int n_feats, int item_col, int T, int d, int hd_valid, int kp, void* x, void* stream);
int rp_concat_gather_rows(const void* item_table, const int32_t* ids, const rp_feature* feats, const int* seg_col,
                          const int* seg_dim, int n_feats, int item_col, const int32_t* row_tok, const int32_t* n_rows_dev, int T,
                          int d, int hd_valid, int kp, void* x, void* stream);
int rp_concat_embed_fwd(const float* y, const float* pos, const int32_t* row_tok, const int32_t* n_rows_dev, int T, int L, int d,
                        int pos0, float scale, float drop_p, unsigned long long seed, unsigned long long drop_off,
                        const unsigned long long* seed_ptr, void* out, void* stream);
int rp_concat_scatter(const void* dx, const int32_t* ids, float* d_item, int pad_id, const rp_feature* feats, const int* seg_col,
                      const int* seg_dim, int n_feats, int item_col, const int32_t* row_tok, const int32_t* n_rows_dev, int T,
                      int d, int hd_valid, int kp, void* v_rows, int v_ld, void* stream);
/* The positional half of rp_embed_bwd(_rows) alone: d_pos[pos0 + l] += sum over the sequences of dropout'(dx) at position l
 * (new path: no pad-row mask).  seq_first / seq_off (rp_row_plan): both for packed rows, or neither. */
int rp_embed_pos_bwd(const void* dx, const int32_t* seq_first, const int32_t* seq_off, int B, int L, int d, int pos0,
                     float drop_p, unsigned long long seed, unsigned long long drop_off, const unsigned long long* seed_ptr,
                     float* d_pos, void* stream);

/* torch.nn.LayerNorm forward / backward (transformer.py:47-49,60-62 eps 1e-8; model.py:248 eps 1e-5).  With `gather`
 * output row r reads input row gather[r] and only *n_rows_dev rows exist (valid-target compaction); the backward then
 * scatters dx to those rows.  add_to (optional, bf16 [*, d]) is added to dx (residual-branch gradient). */
/* PADDED FEATURE SLOTS (`hd_valid`, 0 = none): the reference's default shapes are not multiples of the 64-wide tensor-core
 * feature tiles (SasRec.from_params: embedding_dim 192 / 4 heads = head_dim 48, nn/sequential/sasrec/model.py:199-253; legacy
 * hidden_size 50, sasrec/lightning.py:30-47; examples: d = 64 / 2 heads = 32).  Such a model is stored with every head in its
 * own slot of 64 columns (128 for head_dim in (64, 128]) whose first hd_valid columns are the real features and whose padded
 * columns are ZERO in every activation, weight, bias and gradient (zero weights keep them zero through every GEMM, the
 * optimizer never moves a parameter whose gradient is zero).  The only operator that is not blind to the padding is LayerNorm:
 * its statistics run over the d_true = (d / slot) * hd_valid real features and its backward sends no gradient into padded
 * inputs - every entry point that contains a LayerNorm takes `hd_valid`; the attention takes the true softmax scale. */
int rp_layernorm_fwd(const void* x, const float* w, const float* b, float eps, int n_rows, int d, const int32_t* n_rows_dev,
                     const int32_t* gather, void* y, float* mean, float* rstd, int hd_valid, void* stream);
/* rp_layernorm_fwd compacting rows for a loss head (gather and n_rows_dev required): the output rows after *n_rows_dev up to
 * the next multiple of 128 (at most n_rows) are also zeroed.  The heads read their input in whole 128-row tiles, and a stale
 * non-finite row there would reach every item's gradient through a zero weight in an MMA. */
int rp_layernorm_fwd_compact(const void* x, const float* w, const float* b, float eps, int n_rows, int d,
                             const int32_t* n_rows_dev, const int32_t* gather, void* y, float* mean, float* rstd, int hd_valid,
                             void* stream);
int rp_layernorm_bwd(const void* dy, const void* x, const float* w, const float* mean, const float* rstd, int n_rows, int d,
                     const int32_t* n_rows_dev, const int32_t* gather, const void* add_to, void* dx, float* dw, float* db,
                     int hd_valid, void* stream);

/* out = in * regenerated dropout mask / keep (and optional row mask); db[c] += column sums of a bf16 [rows, cols] array. */
int rp_dropout_bwd(const void* in, void* out, long long rows, int cols, const uint8_t* rowmask, float drop_p,
                   unsigned long long seed, unsigned long long drop_off, const unsigned long long* seed_ptr, void* stream);
int rp_colsum(const void* dy, int rows, int cols, long long ld, float* db, void* stream);
/* the same for n <= 6 tensors sharing the row count, one launch (the bias gradients of one block's backward) */
int rp_colsum_multi(int n, const void* const* dy, const int* cols, const long long* ld, float* const* db, int rows, void* stream);

/* BERT4Rec embedding: where(token_mask, table[ids], mask_emb) + pos[t % L] (bert4rec/model.py:239-296) and its backward;
 * row gather / scatter with a device-side row count (dst[r] = src[idx[r]] or dst[idx[r]] = src[r]).
 * pos == NULL (forward) / d_pos == NULL (backward): the model has no positional embedding (enable_positional_embedding
 * = False); the forward adds no positional term and the backward skips the positional column sums. */
int rp_bert_embed_fwd(const void* table, const void* mask_emb, const float* pos, const int32_t* ids, const uint8_t* tok_mask,
                      int T, int L, int d, float drop_p, unsigned long long seed, unsigned long long drop_off,
                      const unsigned long long* seed_ptr, void* out, void* stream);
int rp_bert_embed_bwd(const void* dx, const int32_t* ids, const uint8_t* pad_mask, const uint8_t* tok_mask, int B, int L, int d,
                      float drop_p, unsigned long long seed, unsigned long long drop_off, const unsigned long long* seed_ptr,
                      float* d_table, float* d_mask_emb, float* d_pos, void* stream);
int rp_gather_rows(const void* src, const int32_t* idx, int n_max, const int32_t* n_dev, int d, void* dst, int scatter,
                   void* stream);

/* Inference: out-projection + residual + LayerNorm + FFN of one SASRec block in one pass  (h = o Wo^T + bo + q_in ;
 * y = LN(h) ; out = relu(y W1^T + b1) W2^T + b2 + y); h and y never reach HBM.
 * o, q_in, out bf16 [T, d] (out may not alias o / q_in); wo / w1 / w2 bf16 [d, d]; bo, ln_w, ln_b, b1, b2 fp32 [d]; rowmask
 * optional uint8 [T] (0 -> zero row); d in {64,128}.
 *   replaces (eval)  replay/nn/sequential/sasrec/transformer.py:99-110 ; replay/models/nn/sequential/sasrec/model.py:435-441 */
int rp_post_attn_fused(const void* o, const void* q_in, const void* wo, const float* bo, const float* ln_w, const float* ln_b,
                       float eps, const void* w1, const float* b1, const void* w2, const float* b2, const uint8_t* rowmask, int T,
                       int d, void* out, int hd_valid, void* stream);

/* Training forward of everything after the attention of one SASRec block in one pass over the tokens:
 *   h = o Wo^T + bo + q_in ; y = LN(h) ; u = dropout1(relu(y W1^T + b1)) ; out = (y + dropout2(u W2^T + b2)) [* rowmask]
 * writing the activations the backward needs on the way (h, y, u bf16 [T, d]; LayerNorm mean / rstd fp32 [T]): 2 tensors read
 * and 4 written instead of the 14 [T, d] passes of out-projection GEMM + LayerNorm + two FFN GEMMs.  Element (row, column) of a
 * dropout site is kept iff drop_mix(drop_row_key(seed + *seed_ptr, drop_off, row), drop_col_key(column)) >= p * 2^32
 * (csrc/rp_philox.cuh) - the stream of rp_gemm's epilogue and rp_dropout_bwd, so the un-fused backward applies unchanged.  d in {64,128}; out may not alias o / q_in.
 *   replaces (train)  replay/nn/sequential/sasrec/transformer.py:99-110 ; replay/nn/ffn.py:43-57 ;
 *                     replay/models/nn/sequential/sasrec/model.py:435-441,496-506 */
int rp_post_attn_train(const void* o, const void* q_in, const void* wo, const float* bo, const float* ln_w, const float* ln_b,
                       float eps, const void* w1, const float* b1, const void* w2, const float* b2, const uint8_t* rowmask, int T,
                       int d, float drop_p, unsigned long long seed, unsigned long long drop_off1, unsigned long long drop_off2,
                       const unsigned long long* seed_ptr, void* h_save, void* y_save, void* u_save, float* mean_out,
                       float* rstd_out, void* out, int hd_valid, void* stream);
/* Packed rows: only the first *n_rows_dev of the T rows (T, the capacity, sizes the grid and the tensor maps); row r draws its
 * dropout with the key of token row_tok[r] (rp_row_plan).  No row mask. */
int rp_post_attn_train_rows(const void* o, const void* q_in, const void* wo, const float* bo, const float* ln_w, const float* ln_b,
                            float eps, const void* w1, const float* b1, const void* w2, const float* b2, int T, int d, float drop_p,
                            unsigned long long seed, unsigned long long drop_off1, unsigned long long drop_off2,
                            const unsigned long long* seed_ptr, void* h_save, void* y_save, void* u_save, float* mean_out,
                            float* rstd_out, void* out, int hd_valid, const int32_t* n_rows_dev, const int32_t* row_tok,
                            void* stream);

/* Backward of rp_post_attn_train in one pass over the tokens.  Given dz = d loss / d out:
 *   dzm = dz [* rowmask] ;  d_t = dropout2'(dzm) ;  du = (d_t W2) * [u != 0] / keep ;  dy = du W1 + dzm ;
 *   dh = LayerNorm-backward(dy ; h, mean, rstd, ln_w) ;  d_o = dh Wo ;  dln_w / dln_b += column sums (fp32 atomics, one per column and CTA)
 * d_t, du, dh (bf16 [T, d]) are the dY operands of rp_wgrad_group for W2 / W1 / Wo (X = u, y, o); dh is also the residual gradient
 * into the pre-attention part; d_o feeds rp_attn_bwd.  d_t may be NULL when drop_p == 0 and rowmask == NULL (then d_t == dz).
 *   replaces autograd's backward of  replay/nn/sequential/sasrec/transformer.py:107-110 ; replay/nn/ffn.py:43-57 ;
 *                                    replay/models/nn/sequential/sasrec/model.py:436-441,496-506 */
int rp_post_attn_bwd(const void* dz, const void* u, const void* h, const float* mean, const float* rstd, const float* ln_w,
                     const void* w2, const void* w1, const void* wo, const uint8_t* rowmask, int T, int d, float drop_p,
                     unsigned long long seed, unsigned long long drop_off2, const unsigned long long* seed_ptr, void* d_t, void* du,
                     void* dh, void* d_o, float* dln_w, float* dln_b, int hd_valid, void* stream);
int rp_post_attn_bwd_rows(const void* dz, const void* u, const void* h, const float* mean, const float* rstd, const float* ln_w,
                          const void* w2, const void* w1, const void* wo, int T, int d, float drop_p, unsigned long long seed,
                          unsigned long long drop_off2, const unsigned long long* seed_ptr, void* d_t, void* du, void* dh,
                          void* d_o, float* dln_w, float* dln_b, int hd_valid, const int32_t* n_rows_dev,
                          const int32_t* row_tok, void* stream);

/* Everything BEFORE the attention of one SASRec block in one pass over the tokens (training and inference):
 *   q_in = LayerNorm(x) ;  Q = q_in Wq^T + bq ;  [K | V] = x [Wk | Wv]^T + [bk | bv]      (K, V from the un-normalised x)
 * x is read once; q_in (the block's residual), Q, KV and the LayerNorm statistics are written once (LayerNorm + two GEMM
 * launches read x / q_in three times).  w_in bf16 [3d, d] = packed in_proj_weight, b_in fp32 [3d]; d in {64,128}.
 * q_in == NULL and Q == NULL: only [K | V] is computed (ln_w / ln_b unused) - predict()'s final block, whose LayerNorm and
 * Q projection run on the last position of every sequence only.
 *   replaces  replay/nn/sequential/sasrec/transformer.py:99-106 ; replay/models/nn/sequential/sasrec/model.py:434-435 */
int rp_ln_qkv_fused(const void* x, const float* ln_w, const float* ln_b, float eps, const void* w_in, const float* b_in, int T,
                    int d, void* q_in, void* Q, void* KV, float* mean_out, float* rstd_out, int hd_valid, void* stream);
int rp_ln_qkv_fused_rows(const void* x, const float* ln_w, const float* ln_b, float eps, const void* w_in, const float* b_in,
                         int T, int d, void* q_in, void* Q, void* KV, float* mean_out, float* rstd_out, int hd_valid,
                         const int32_t* n_rows_dev, void* stream);
/* Its backward in one pass:  dq_in = dQ Wq + dh ;  t = LayerNorm-backward(dq_in; x, mean, rstd, ln_w) ;  dx = [dK | dV] Wkv + t.
 * dln_w / dln_b fp32 [d] are ACCUMULATED (one fp32 atomic per column and CTA).  dx may not alias an input; d in {64,128}. */
int rp_pre_attn_bwd(const void* dQ, const void* dKV, const void* dh, const void* x, const float* mean, const float* rstd,
                    const float* ln_w, const void* w_in, int T, int d, void* dx, float* dln_w, float* dln_b, int hd_valid,
                    void* stream);
int rp_pre_attn_bwd_rows(const void* dQ, const void* dKV, const void* dh, const void* x, const float* mean, const float* rstd,
                         const float* ln_w, const void* w_in, int T, int d, void* dx, float* dln_w, float* dln_b, int hd_valid,
                         const int32_t* n_rows_dev, void* stream);

/* ALL weight and bias gradients of one transformer block in one launch (+ one deterministic reduction launch):
 *   dW_i[n_out_i, n_in_i] (+)= dY_i[T, n_out_i]^T . X_i[T, n_in_i] ;  db_i[n_out_i] (+)= column sums of dY_i      i < n_pairs <= 8
 * dY_i / X_i are read in place (MN-major wgmma operands, contraction over the tokens); the bias gradient is one extra N = 16
 * MMA per k-step against a tile of ones.  n_out, n_in multiples of 64; at most 48 output tiles of 128 x 128 in one call.
 *   replaces  autograd's weight / bias gradients of  replay/nn/sequential/sasrec/transformer.py:36-46,99-110 ;
 *             replay/nn/ffn.py:43-57 ; replay/models/nn/sequential/sasrec/model.py:407-414,490-506 ; bert4rec/model.py:471-527 */
typedef struct rp_wgrad_pair {
  const void* dY; long long dy_ld; int n_out;   /* bf16 [T, n_out], row pitch dy_ld elements */
  const void* X; long long x_ld; int n_in;      /* bf16 [T, n_in],  row pitch x_ld */
  float* dW; long long dw_ld;                   /* fp32 [n_out, n_in], row pitch dw_ld (multiple of 4) */
  float* db;                                    /* fp32 [n_out] or NULL */
} rp_wgrad_pair;
size_t rp_wgrad_group_workspace(const rp_wgrad_pair* pairs, int n_pairs);
int rp_wgrad_group(const rp_wgrad_pair* pairs, int n_pairs, int T, int accumulate, void* workspace, size_t workspace_bytes,
                   void* stream);
/* Packed rows: the contraction covers the first *n_rows_dev of the T rows (rows past it are never read as nonzero). */
int rp_wgrad_group_rows(const rp_wgrad_pair* pairs, int n_pairs, int T, int accumulate, const int32_t* n_rows_dev,
                        void* workspace, size_t workspace_bytes, void* stream);

/* The optimizer step of models/nn/optimizer_utils/optimizer_factory.py:71-87 / nn/lightning/optimizer.py:44-60 on flat
 * fp32 buffers of n elements (n % 4 == 0, 16-byte aligned); refreshes the bf16 shadow (if not NULL), optionally zeroes the
 * gradient.  lr and the step counter live in device memory (graph-replayable); every call first adds 1 to *step_dev.
 * The gradient is g * grad_scale (1/world after a sum all-reduce), and weight_decay != 0 adds weight_decay * p to it.
 *   RP_OPT_ADAM  torch.optim.Adam(lr, betas, eps, weight_decay): state0 = exp_avg, state1 = exp_avg_sq, bias corrections
 *                from the incremented step.
 *   RP_OPT_SGD   torch.optim.SGD(lr, momentum, weight_decay), dampening 0, no Nesterov; the step counter is not read.
 *                momentum 0: no state (state0 and state1 unused).  momentum != 0: state0 = momentum_buffer, state1 unused.
 *                A buffer that was never written must be zero: its first step then gives momentum * 0 + d = d, which is
 *                torch's clone of d.  A restored buffer is simply used.
 * frozen: per-element mask (or NULL) of parameters the step leaves unchanged; their state still advances.
 * rp_adam_step is rp_optimizer_step(RP_OPT_ADAM, ..., weight_decay 0, momentum 0, ...). */
#define RP_OPT_ADAM 0
#define RP_OPT_SGD 1
int rp_optimizer_step(int kind, float* p, float* g, float* state0, float* state1, void* shadow_bf16, long long n,
                      const float* lr_dev, int32_t* step_dev, float beta1, float beta2, float eps, float weight_decay,
                      float momentum, float grad_scale, const uint8_t* frozen, int zero_grad, void* stream);
int rp_adam_step(float* p, float* g, float* m, float* v, void* shadow_bf16, long long n, const float* lr_dev,
                 int32_t* step_dev, float beta1, float beta2, float eps, float grad_scale, const uint8_t* frozen,
                 int zero_grad, void* stream);
/* Gradient exchange of data-parallel training over NVLink peer memory - ONE kernel inside the captured step graph.
 *   replaces  the bucketed all-reduce of Lightning DDP under loss.backward()  replay/nn/lightning/module.py:62-75 with
 *             Trainer(strategy="ddp"); replay/models/nn/sequential/sasrec/lightning.py:196-209 (SURVEY.md 2.1 / 8e)
 * bufs[w] / states[w] (host arrays of `world` device pointers): rank w's fp32 gradient buffer (n elements, 16-byte aligned)
 * and its state block (rp_peer_allreduce_state_bytes() bytes, zeroed once) as mapped into THIS process - every rank passes
 * pointers into the same symmetric allocation (replay_b200/peer.py).  world in 2..8, one node.  Result: every buffer holds
 * the element-wise sum, bit-identical on all ranks (each element is summed by one rank in rank order and broadcast).
 * Every rank must enqueue it exactly once per step; CUDA-graph capturable; the grid never exceeds the SM count. */
size_t rp_peer_allreduce_state_bytes(void);
int rp_peer_allreduce(void* const* bufs, void* const* states, int rank, int world, long long n, void* stream);
int rp_cast_bf16(const float* src, void* dst, long long n, void* stream);
int rp_counter_add(unsigned long long* counter, unsigned long long inc, void* stream);

/* ---------------------------------------------------------------------------------------------------------------
 * Sampled training heads (SURVEY.md §8 a9 / f.2): logits only for the positive item and n_neg sampled negatives per target.
 *   replaces  SampledLossBase.get_sampled_logits + mask_negative_logits   replay/nn/loss/base.py:40-154,157-196
 *             CESampled.forward / BCESampled.forward                      replay/nn/loss/ce.py:199-249 ; bce.py:154-218
 *             legacy _compute_loss_ce_sampled / _compute_loss_bce_sampled  replay/models/nn/sequential/sasrec/lightning.py:310-376
 *             LogInCESampled.forward / CESampledWeighted.forward           replay/nn/loss/login_ce.py:240-375 ; ce.py:252-330
 * hc / labels / n_valid as for rp_ce_head_fwd (compacted valid targets).  negatives int64: neg_mode 0 = [n_neg] shared by the
 * batch (tensor-core path), 1 = [B*seq_len, n_neg] per position, 2 = [B, n_neg] per sequence (1, 2: rows addressed through
 * valid_idx[t] = flat b*seq_len + l of compacted row t; gather-dot kernels).  kind: RP_LOSS_CE_SAMPLED (negatives equal to the
 * positive or to ignore_index get logit -1e9), RP_LOSS_BCE_SAMPLED (same masking, log_eps / clamp as the reference),
 * RP_LOSS_LEGACY_CE_SAMPLED (log(vocab_size-1) - 1e6*reject - log(min(n_neg, vocab_size) - #reject) correction),
 * RP_LOSS_LEGACY_BCE_SAMPLED (no masking), RP_LOSS_LOGIN_CE_SAMPLED (CE_SAMPLED's masking and softmax over [positive |
 * negatives]; -clamp(log(p + log_eps), -clamp, clamp) of the positive's share p, gradient 0 where the clamp is active),
 * RP_LOSS_CE_SAMPLED_WEIGHTED (CE_SAMPLED's row loss times row_weight[t]; mean over the valid targets, not divided by the
 * weights' sum).  row_weight: fp32 [capacity] in the compacted row order, required (RP_EINVAL) by RP_LOSS_CE_SAMPLED_WEIGHTED
 * and ignored by every other kind.  num_positives (0 or 1: one positive per position) up to RP_MAX_POSITIVES, with kinds
 * CE_SAMPLED, BCE_SAMPLED and CE_SAMPLED_WEIGHTED only: labels, row_weight and slot_mask are [capacity, num_positives]
 * (rp_prepare_batch_multi), every set slot is a pair - its own positive against the row's negatives, which are masked
 * against all num_positives labels of the row - and the mean runs over the *n_pairs pairs (loss_out[1] = 1 / *n_pairs).
 * fwd: loss_out[0] = mean loss, loss_out[1] = 1/T_v,
 * d(loss)/d(logits) stays in the workspace (which need not be zeroed); bwd: d_hc bf16 [capacity, d] rows < *n_valid, d_table
 * fp32 ACCUMULATED (+=: zero it first; rows that no positive and no unmasked negative points at are left as they were).
 * d_hc rows >= *n_valid: untouched with per-row negatives; with shared negatives rows [*n_valid, min(round_up(*n_valid, 128),
 * capacity)) are written with 0 and the rest are untouched.  *n_valid == 0: loss_out = {0, 0}, d_table unchanged.
 * ------------------------------------------------------------------------------------------------------------- */
#define RP_LOSS_CE_SAMPLED 0
#define RP_LOSS_BCE_SAMPLED 1
#define RP_LOSS_LEGACY_CE_SAMPLED 2
#define RP_LOSS_LEGACY_BCE_SAMPLED 3
#define RP_LOSS_LOGIN_CE_SAMPLED 4
#define RP_LOSS_CE_SAMPLED_WEIGHTED 5
typedef struct rp_sampled_desc {
  const void* hc; const void* table; const int32_t* labels; const int32_t* valid_idx; const int64_t* negatives;
  const int32_t* n_valid;
  int capacity, n_items, d, n_neg, neg_mode, seq_len, kind, ignore_index, vocab_size;
  float log_eps, clamp;
  float* loss_out;
  void* workspace; size_t workspace_bytes;
  const float* row_weight;
  int num_positives; const uint8_t* slot_mask; const int32_t* n_pairs;
} rp_sampled_desc;
size_t rp_sampled_head_workspace(int capacity, int d, int n_neg, int neg_mode);
size_t rp_sampled_head_workspace_multi(int capacity, int d, int n_neg, int neg_mode, int num_positives);
int rp_sampled_head_fwd(const rp_sampled_desc* s, void* stream);
int rp_sampled_head_bwd(const rp_sampled_desc* s, void* d_hc, float* d_table, void* stream);

/* ---------------------------------------------------------------------------------------------------------------
 * Scalable cross-entropy head of the legacy SASRec (loss_type="SCE", arXiv 2409.18721):
 *   replaces  ScalableCrossEntropyLoss.__call__          replay/models/nn/loss/sce.py:43-124
 *             SasRec._compute_loss_scalable_ce           replay/models/nn/sequential/sasrec/lightning.py:383-392
 * hc bf16 [capacity, d]: final hidden state of EVERY position (row b * seq_len + l, pad rows included); table bf16
 * [n_items, d]; labels int64 [capacity]; pad_mask [capacity] (1 = real input position); n_rows int32 [1] in device memory =
 * B * seq_len of the batch (<= capacity).  d in {64,128,256,512} is the padded width, d_true the model's hidden size,
 * hd_valid the feature-slot layout (0 = unpadded; else <= 128 with d a multiple of its slot, and d_true must equal the
 * real features of that layout: d / slot * hd_valid, or d when unpadded).  1 <= bucket_size_x <= min(1024, capacity),
 * 1 <= bucket_size_y <= min(1024, n_items) (the fused top-K), else RP_ESHAPE.  The S = X_b . Y_b^T scores and dX run in
 * chunks of buckets whose fp32 share of the workspace stays within RP_SCE_CHUNK_BYTES (environment, read at every call,
 * default 256 MiB; at least one bucket per chunk).
 * Caller-owned outputs: draw fp32 = the standard normals, [n_buckets, d_true] (or [capacity, n_buckets] with mix_x; rows
 * < *n_rows used), drawn from Philox keyed by seed + *rng_counter unless draw_given (then read as given); top_x int64 and
 * score_x fp32 [n_buckets, bucket_size_x] (slots with score -inf hold no row); top_y int64 [n_buckets, bucket_size_y].
 * A row carries loss when it is a real position < *n_rows with a label in [0, n_items); every other row (pad, t >=
 * *n_rows, label outside the catalog) is also left out of the row selection: it scores -inf in top_x.
 * fwd: loss_out fp32 [2] = { mean over the rows with a non-zero per-row max of the bucket CEs (NaN when there is none),
 * 1 / that count rounded once (0 when none) }.
 * stages: RP_SCE_DRAW | RP_SCE_SELECT_X | RP_SCE_SELECT_Y | RP_SCE_BUCKET_CE run in this order (RP_SCE_ALL = one forward;
 * the parts exist for timing).  bwd: d_hc bf16 [capacity, d] OVERWRITTEN for every row (zero where no gradient); no table
 * gradient (the reference scores a detached copy of the table).  Deterministic and CUDA-graph capturable. */
#define RP_SCE_DRAW 1
#define RP_SCE_SELECT_X 2
#define RP_SCE_SELECT_Y 4
#define RP_SCE_BUCKET_CE 8
#define RP_SCE_ALL 15
typedef struct rp_sce_desc {
  const void* hc; const void* table; const int64_t* labels; const uint8_t* pad_mask; const int32_t* n_rows;
  int capacity, n_items, d, d_true, hd_valid;
  int n_buckets, bucket_size_x, bucket_size_y, mix_x;
  unsigned long long seed; const unsigned long long* rng_counter; int draw_given;
  float* draw; int64_t* top_x; float* score_x; int64_t* top_y;
  float* loss_out;
  void* workspace; size_t workspace_bytes;
} rp_sce_desc;
size_t rp_sce_head_workspace(int capacity, int n_items, int d, int n_buckets, int bucket_size_x, int bucket_size_y, int mix_x);
int rp_sce_head_fwd(const rp_sce_desc* s, int stages, void* stream);
int rp_sce_head_bwd(const rp_sce_desc* s, void* d_hc, void* stream);

/* ---------------------------------------------------------------------------------------------------------------
 * Device-side batch construction (SURVEY.md §8 f.1).  All histories are resident in HBM as CSR: offsets [n_seq+1] int64,
 * items [offsets[n_seq]] int32.  One call builds B rows of a [B, L] batch: row b is the window of history seq_index[b]
 * starting at seq_offset[b] (NULL: the LAST L(+1) items), left-padded with pad_value.  Replaces the per-sample host path
 *   TorchSequentialDataset.__getitem__/_pad_sequence/_generate_padding_mask  replay/data/nn/torch_sequential_dataset.py:69-136
 *   SasRecTrainingDataset.__getitem__ (window L+1, inputs [:-1], labels [1:])  replay/models/nn/sequential/sasrec/dataset.py:104-126
 *   Bert4RecUniformMasker.mask + Bert4RecTrainingDataset.__getitem__          .../bert4rec/dataset.py:71-92,163-177
 *   _shift_features (predict: roll left, last = pad, token/pad masks)         .../bert4rec/dataset.py:322-351
 *   Array1DColumn.__getitem__ + NextTokenTransform (new path, torch ops)     replay/data/nn/parquet/impl/array_1d_column.py:70-84,
 *                                                                            impl/indexing.py:42-78, replay/nn/transform/next_token.py:65-96
 * and the default collate.  mode: RP_BATCH_SASREC_TRAIN -> ids, pad_mask, labels, aux_mask = target_padding_mask;
 * RP_BATCH_PREDICT -> ids, pad_mask; RP_BATCH_BERT_TRAIN -> ids (= inputs), pad_mask, labels (= positive_labels),
 * aux_mask = token_mask (0 = masked) drawn as (u * pad) >= mask_prob with the reference's two corner-case fix-ups, u from
 * `uniforms` [B, L] when given (bit-exact against the reference masker fed the same numbers) else Philox4x32-10 keyed by
 * (seed, draw0 + b); RP_BATCH_BERT_PREDICT -> shifted ids, pad_mask, aux_mask = token_mask.
 * query_out [B] (optional) = query_ids[seq_index[b]] (or the index itself when query_ids is NULL).
 * ------------------------------------------------------------------------------------------------------------- */
#define RP_BATCH_SASREC_TRAIN 0
#define RP_BATCH_PREDICT 1
#define RP_BATCH_BERT_TRAIN 2
#define RP_BATCH_BERT_PREDICT 3
int rp_build_batch(const int64_t* offsets, const int32_t* items, long long n_seq, const int32_t* seq_index,
                   const int32_t* seq_offset, int B, int L, int mode, int pad_value, float mask_prob, const float* uniforms,
                   unsigned long long seed, unsigned long long draw0, const int64_t* query_ids, int64_t* ids,
                   uint8_t* pad_mask, int64_t* labels, uint8_t* aux_mask, int64_t* query_out, void* stream);

/* Feature columns of the same store, cut in the same launch (rp_build_batch_features).  A column holds one entry per
 * event of every history, aligned with `items` (event e of history s is offsets[s] + k):
 *   RP_BATCH_COL_INT   one integer per event, values int32 or int64 (in_bytes 4 / 8)           -> out int64 [B, L]
 *   RP_BATCH_COL_FLOAT `width` floats per event ([n_events, width]), float32 or float64        -> out [B, L, width]
 *                      (width 1: a scalar, out [B, L]); out_bytes 4 = float32 (rounded to nearest), 8 = float64
 *   RP_BATCH_COL_LIST  a list of any length per event: list_offsets [n_events + 1] into values (int32 / int64);
 *                      out int64 [B, L, width]: each event's LAST `width` entries left-padded to width with the padding
 *                      value (Array2DColumn.__getitem__, replay/data/nn/parquet/impl/array_2d_column.py:72-92)
 * Every column uses the ids' window, offset and shift: a position that is padding in the ids (and the last position of
 * RP_BATCH_BERT_PREDICT) is pad_int / pad_float in every element.  Integer outputs take pad_int, float outputs pad_float
 * converted to the output type.
 * Query lists hold one integer list per stored history instead of one entry per event (a user's ground-truth or train
 * items): list_offsets [n_seq + 1] into values (int32 / int64), out int64 [B, width] from the list of seq_index[b],
 * independent of the window and of every mode's shift:
 *   RP_BATCH_COL_QUERY_LIST       the list's FIRST `width` entries, right-padded with pad_int
 *                                 (TorchSequentialValidationDataset._get_ground_truth / _get_train,
 *                                 replay/data/nn/torch_sequential_dataset.py:263-285)
 *   RP_BATCH_COL_QUERY_LIST_LAST  the list's LAST `width` entries, left-padded with pad_int (Array1DColumn.__getitem__,
 *                                 replay/data/nn/parquet/impl/array_1d_column.py:70-84, indexing.py:42-78)
 * At most RP_BATCH_MAX_COLUMNS columns of all kinds together.  Other arguments as rp_build_batch, which this call runs in
 * the same kernel; n_cols == 0 is rp_build_batch.  RP_EINVAL: null pointer, unknown kind, byte widths other than 4 / 8
 * (integer out_bytes must be 8), width < 1, n_cols outside [0, RP_BATCH_MAX_COLUMNS].  No host synchronisation: the
 * descriptors are passed by value to the kernel. */
#define RP_BATCH_MAX_COLUMNS 16
#define RP_BATCH_COL_INT 0
#define RP_BATCH_COL_FLOAT 1
#define RP_BATCH_COL_LIST 2
#define RP_BATCH_COL_QUERY_LIST 3
#define RP_BATCH_COL_QUERY_LIST_LAST 4
typedef struct rp_batch_column {
  int kind, in_bytes, out_bytes, width;
  const void* values;
  const int64_t* list_offsets;
  void* out;
  long long pad_int;
  double pad_float;
} rp_batch_column;
int rp_build_batch_features(const int64_t* offsets, const int32_t* items, long long n_seq, const int32_t* seq_index,
                            const int32_t* seq_offset, int B, int L, int mode, int pad_value, float mask_prob,
                            const float* uniforms, unsigned long long seed, unsigned long long draw0,
                            const int64_t* query_ids, int64_t* ids, uint8_t* pad_mask, int64_t* labels, uint8_t* aux_mask,
                            int64_t* query_out, const rp_batch_column* cols, int n_cols, void* stream);

/* ---------------------------------------------------------------------------------------------------------------
 * Bring-up self test of the wgmma operand encodings (used by tests/, not by the product path).
 * A, B: bf16 [128,128]; D: fp32 [128,128].  mode bit0: B given as Bt[K,N]; bit1: A read into registers;
 * bit2: A given as At[K,M].  D = A . B^T in every mode.
 * ------------------------------------------------------------------------------------------------------------- */
int rp_selftest_mma(int mode, const void* A, const void* B, float* D, void* stream);
/* exp2 helpers of the CE head's exponential loops: y_poly[i] = ex2_poly(x[i]) (polynomial on the FMA pipe), y_mufu[i] =
 * ex2.approx.ftz(x[i]) (special-function unit), for i < n.  fp32 device arrays. */
int rp_selftest_exp2(const float* x, float* y_poly, float* y_mufu, long long n, void* stream);
/* TMA feed-rate probe (tools/probe_tma.py): every CTA streams `tiles` [box_rows x d] row tiles of a K-major bf16 table through
 * an 8-stage ring with no consumer. */
/* wgmma issue-rate probe (tools/probe_mma.py): mode bit0 B MN-major, bit1 A from registers, bit2 A MN-major, bits 3-4 N = 128 /
 * 256 / 64; one warpgroup per CTA issues iters x 8 MMAs (64xNx16 bf16) and writes its elapsed SM cycles to cycles_out[blockIdx.x]. */
int rp_selftest_mma_probe(int mode, int iters, int grid, long long* cycles_out, void* stream);
int rp_selftest_tma_probe(const void* table, long long rows, int d, int box_rows, int tiles, int same_tile, int grid,
                          void* stream);

/* ---------------------------------------------------------------------------------------------------------------
 * DiffTransformer encoder (replay/nn/sequential/sasrec/diff_transformer.py, replay/nn/attention.py:67-157,
 * replay/nn/ffn.py:60-99; arXiv 2410.05258).  Per head h of true width head_dim <= 64:
 *   lambda_h = exp(sum_j lq1[h,j] lk1[h,j]) - exp(sum_j lq2[h,j] lk2[h,j]) + lambda_init   (fp32, read on the device)
 *   A = softmax(Q1 K1^T s + M) - lambda_h softmax(Q2 K2^T s + M),  O = A V,  out = O / sqrt(mean(O^2) + eps) * rms_scale
 *       * (1 - lambda_init)
 * with M: key j visible to query i iff j <= i and (pad_mask[j] or j == i) - pad rows attend to themselves
 * (replay/nn/mask.py:29-51; the encoder ignores padding_mask).  Column layout of one token row: the q / k array holds per
 * head [q1 (64-wide slot) | q2 (64-wide slot)] at x_c0 + h*128; v / out / o_pre hold per head a v_slot-wide slot (64 for
 * head_dim <= 32, 128 for head_dim <= 64) whose first 2*head_dim columns are real.  L <= 256.
 * ------------------------------------------------------------------------------------------------------------- */
typedef struct rp_diff_lambda {
  const float* q1; const float* k1; const float* q2; const float* k2;   /* fp32 [H, head_dim] each */
  int head_dim; float lambda_init;
} rp_diff_lambda;
typedef struct rp_diff_attn_desc {
  const void* qk; long long ld_qk; int q_c0, k_c0;   /* Q and K columns may live in one array (packed projection) */
  const void* v; long long ldv; int v_c0;
  const uint8_t* pad_mask;                          /* [B*L], 1 = real item */
  int B, H, L, head_dim, v_slot;
  float scale;                                      /* 1/sqrt(head_dim) */
  float eps;                                        /* per-head RMSNorm eps (1e-5) */
  rp_diff_lambda lam;
  const float* rms_scale;                           /* fp32 [v_slot], zero beyond 2*head_dim */
  void* out; long long ldo;                         /* bf16 normalised output */
  /* training saves (all NULL in eval; a NULL e1_save switches every save off): o_pre = O before the per-head RMSNorm
   * (geometry of out); e1 / e2 bf16 [B*H, Lp, Lp] = exp(s - rowmax) of either map (zero where masked; Lp = round_up(L, 64); rows >= L are not written,
   * so the buffers are zero-initialised once); inv1 / inv2 fp32 [B*H, Lp] the reciprocal row sums */
  void* o_pre; void* e1_save; void* e2_save; float* inv1; float* inv2;
  float* o32_save; float* o2_save;                  /* fp32, geometry of out: O_pre and A2 . V (inputs of the lambda gradient) */
} rp_diff_attn_desc;
int rp_diff_attn_fwd(const rp_diff_attn_desc* a, void* stream);
/* Row-wise backward between the batched rp_gemm calls, from the forward's saves and dA = dO_pre . V^T (bf16 [B*H, Lp, Lp]):
 * dS1 = A1 (dA - sum A1 dA) s, dS2 = -lambda A2 (dA - r2) s, A = A1 - lambda A2 (the A operand of dV = A^T dO_pre; A may
 * alias dA), dlam_part fp32 [B*H, Lp] = -r2 per row, with r2 = sum_j A2 dA = dO_pre . (A2 V), dO_pre recomputed in fp32
 * from d_on (bf16, gradient of the normalised output), the forward's o32_save / o2_save and rms_scale (eps of the per-head
 * norm); all of pitch ld_o with v_slot columns per head.  Columns >= L are not written. */
int rp_diff_attn_softmax_bwd(const void* e1, const void* e2, const float* inv1, const float* inv2, const void* dA, void* dS1,
                             void* dS2, void* A, float* dlam_part, int BH, int H, int L, float scale, const rp_diff_lambda* lam,
                             const void* d_on, const float* o32, const float* o2, const float* rms_scale, float eps,
                             long long ld_o, int v_slot, void* stream);
/* dlambda_h = sum over sequences and rows of dlam_part (fixed order) chained into the lambda_* gradients (+=). */
int rp_diff_lambda_bwd(const float* dlam_part, int B, int H, int L, const rp_diff_lambda* lam, float* gq1, float* gk1, float* gq2,
                       float* gk2, void* stream);
/* RMSNorm over groups of `group` columns (64 / 128 / 256 / 512; d a multiple of it, d <= 512): y = x * rstd * w[c % group] * alpha,
 * rstd = 1/sqrt(sum_group x^2 / n_true + eps) - torch.nn.RMSNorm (group = d, the SwiGLU item tower's norms) and the per-head norm of the differential
 * attention (group = v_slot, n_true = 2*head_dim, alpha = 1 - lambda_init).  Padded columns must be zero in x and w.
 * With `gather` output row r reads input row gather[r] and only min(n_rows, *n_rows_dev) rows exist; the backward then
 * writes dx to those input rows.  dw (fp32 [group]) += the weight gradient, reduced in a fixed order through the workspace
 * (rp_rmsnorm_bwd_workspace bytes). */
int rp_rmsnorm_fwd(const void* x, const float* w, float eps, float alpha, int n_rows, int d, int group, int n_true,
                   const int32_t* n_rows_dev, const int32_t* gather, void* y, void* stream);
size_t rp_rmsnorm_bwd_workspace(int group);
int rp_rmsnorm_bwd(const void* dy, const void* x, const float* w, float eps, float alpha, int n_rows, int d, int group, int n_true,
                   const int32_t* n_rows_dev, const int32_t* gather, void* dx, float* dw, void* workspace, size_t workspace_bytes,
                   void* stream);
/* SwiGLU gate: gl bf16 [n_rows, 2F] = [g | l] (pre-activations, biases applied) -> u = silu(g) * l bf16 [n_rows, F];
 * backward dgl = [du * l * silu'(g) | du * silu(g)]. */
int rp_swiglu_fwd(const void* gl, long long n_rows, int F, void* u, void* stream);
int rp_swiglu_bwd(const void* du, const void* gl, long long n_rows, int F, void* dgl, void* stream);

/* ---------------------------------------------------------------------------------------------------------------
 * Candidate compaction of the TwoTower model's sampled losses (replay/nn/sequential/twotower/model.py get_logits(h,
 * candidates) -> item_tower(candidates)): the SwiGLU item tower runs on the distinct items one step references only.
 * Inputs as for rp_sampled_head_fwd: compacted labels [capacity] with *n_valid valid, negatives int64 in neg_mode 0 (shared
 * [n_neg]), 1 (per position [B*seq_len, n_neg], rows valid_idx[t]) or 2 (per sequence [n_neg_rows = B, n_neg], all rows).
 * Outputs: *n_slots; item_of_slot int32 [cap] in ascending item id (-1 from *n_slots on); labels_out int32 [capacity] and
 * negatives_out int64 (the negatives' layout; per-position rows of invalid targets untouched) as slot ids - negatives equal to
 * ignore_index (>= 0) become `cap` (give the head ignore_index = cap), ids outside [0, n_items) become cap + 1 (the head
 * reads row 0, item 0, as it does for such ids over the whole catalog, and never matches a positive); rows_out bf16 [cap, d]
 * = table[item_of_slot[s]], zero rows from *n_slots on; rows_out = null skips the rows (rp_item_feature_embed_fwd builds
 * them with item features).  cap = min(n_items, capacity + negative entries) bounds the slots.
 * No host synchronisation (graph-capturable).  Workspace: rp_tower_compact_workspace(n_items) bytes, need not be zeroed.
 * rp_tower_scatter_rows: d_table fp32 [*, d] row item_of_slot[s] += dx bf16 [n_rows, d] row s, s < min(*n_slots, n_rows);
 * item_of_slot = null: identity over n_rows rows.  Each item has at most one slot: plain stores, deterministic. */
size_t rp_tower_compact_workspace(int n_items);
int rp_tower_compact(const int32_t* labels, const int32_t* n_valid, int capacity, const int64_t* negatives, int n_neg,
                     int neg_mode, int n_neg_rows, const int32_t* valid_idx, int seq_len, int ignore_index, int n_items,
                     const void* table, int d, int cap, int32_t* n_slots, int32_t* item_of_slot, int32_t* labels_out,
                     int64_t* negatives_out, void* rows_out, void* workspace, size_t workspace_bytes, void* stream);
int rp_tower_scatter_rows(const void* dx, const int32_t* item_of_slot, const int32_t* n_slots, int n_rows, int d,
                          float* d_table, void* stream);

/* The item tower's input with side features (ItemTower.forward -> embedder -> SumAggregator, csrc/rp_features.cu):
 *   out[r] = table[i] + sum_f term_f(i)   (bf16 [n_rows, d], summed in fp32, rounded once; no scale, position or dropout)
 * i = item_of_slot[r] for r < *n_slots (zero rows from there on), or i = item0 + r when item_of_slot is null.  The features
 * are rp_feature_embed_fwd's kinds with `values` indexed by item id (the item features reader's columns on the device).
 * rp_item_feature_embed_bwd, from dx = d(out) bf16 [n_rows, d] (the item table's own gradient is rp_tower_scatter_rows'):
 *   item_of_slot set: each slot's row is added into its categorical d_table rows with fp32 atomics (padding rows frozen,
 *     mean bags by 1 / count); plan unused.
 *   item_of_slot null (row r = item r, the whole catalog): the categorical rows are reduced in the fixed order of `plan`,
 *     bitwise reproducible.  The plan lists, per (feature, table row) group with at least one live entry, the entries
 *     (item, weight 1 or 1 / count) in chunks; partial fp32 [n_chunks, d] is its workspace.
 * With numerical features v_rows bf16 [n_rows, v_ld] gets their values at val_col (other columns zero; rows from *n_slots
 * on untouched), so that rp_wgrad_group over (dx, v_rows) gives dW and column sums of dx give db.  Over the catalog the
 * values never change, so v_rows may be null there (staged once by the caller); with item_of_slot it is required.  No host
 * synchronisation.  RP_EINVAL: null pointer, unknown kind; RP_ESHAPE: d, hd_valid, n_feats, widths, val_col, v_ld. */
typedef struct rp_item_feature_plan {
  const int32_t* ent_item;   /* [n_ent] item of each entry, grouped by (feature, table row), chunks contiguous */
  const float* ent_w;        /* [n_ent] 1, or 1 / (live entries of the item's bag) for RP_FEAT_BAG_MEAN */
  const int32_t* chunk_off;  /* [n_chunks + 1] entry range of each chunk; a chunk lies inside one group */
  const int32_t* grp_chunk;  /* [n_groups + 1] chunk range of each group */
  const int32_t* grp_feat;   /* [n_groups] index into feats (a categorical kind) */
  const int32_t* grp_row;    /* [n_groups] table row, distinct per feature */
  float* partial;            /* [n_chunks, d] fp32 workspace */
  int n_chunks, n_groups;
} rp_item_feature_plan;
int rp_item_feature_embed_fwd(const void* item_table, const rp_feature* feats, int n_feats, const int32_t* item_of_slot,
                              const int32_t* n_slots, int n_rows, int item0, int d, int hd_valid, void* out, void* stream);
int rp_item_feature_embed_bwd(const void* dx, const rp_feature* feats, int n_feats, const int32_t* item_of_slot,
                              const int32_t* n_slots, int n_rows, int d, int hd_valid, const rp_item_feature_plan* plan,
                              void* v_rows, int v_ld, void* stream);

/* ---------------------------------------------------------------------------------------------------------------
 * TiSASRec's time-interval attention (replay/models/nn/sequential/sasrec/model.py:532-800, csrc/rp_tisasrec.cu) without
 * the reference's [B, L, L] interval matrix or its [B, L, L, d] embeddings.  Per head h (64-wide slot, true width
 * head_dim), sequence b, query i, key j, with r_ij = min(floor(|t_i - t_j|), time_span) computed in the kernels from the
 * timestamps in their own dtype (0 int64, 1 float32, 2 float64; int64 skips the floor):
 *   S_ij = (q_i . k'_j + q_i . TKm_ij) * scale, causal keys j <= i, softmax -> A, Ad = dropout(A) (site att_off, row key
 *   (b*H + h) * Lp + i, column j: the stream of rp_attn_softmax_bwd), o_i = sum_j Ad_ij (v'_j + TVm_ij)
 * with k' = k + dropout(pos_k), v' = v + dropout(pos_v) (rp_ti_pos_add) and TKm_ij / TVm_ij = dropout(time_k / time_v
 * [r_ij]), element (token b*L + i, key j, padded column c) of sites tk_off / tv_off kept iff
 * drop_mix(drop_row_key(seed + *seed_ptr, off, (b*L + i) * L + j), drop_col_key(c)) >= p * 2^32 - one mask per step,
 * shared by every block.  A query row with pad_mask 0 attends to nothing (A = Ad = 0, hpre = q_in): the reference gives it
 * a uniform row and then zeroes the block's output there, so nothing downstream depends on it.
 * Lp = round_up(L, 64).  q, q_in, hpre, d_o, dq_t: bf16 [B*L, ldq]; time_k / time_v: bf16 [time_span + 1, ld_t] (padded
 * columns zero); d_time_k / d_time_v: fp32 of the same pitch.  L <= 256, H * 64 <= RP_TI_MAX_COLS, 1 <= time_span <=
 * RP_TI_MAX_SPAN (the backward keeps both tables' fp32 gradients of one head in shared memory).
 * rp_ti_attn_fwd: s = q . k'^T fp32 [B*H, Lp, Lp] (rp_gemm) -> a_save, ad bf16 [B*H, Lp, Lp] (ad may alias a_save iff
 *   drop_p == 0; columns up to Lp written) and hpre = q_in + sum_j Ad_ij TVm_ij, the residual of o = Ad . v' (rp_gemm).
 * rp_ti_attn_bwd: dpd = dO . v'^T bf16 [B*H, Lp, Lp] (rp_gemm) is overwritten with dS (scale included), ad with Ad (unless
 *   it aliases a_save), dq_t = sum_j dS_ij TKm_ij (the residual of dQ = dS . k'); d_time_k / d_time_v += the gradients of
 *   the two tables (true columns only).  Each CTA sums its pairs' table gradients in shared memory with fp32 atomics, then
 *   the CTAs' partials (workspace rp_ti_attn_bwd_workspace bytes) are added in a fixed order: the time-table gradients are
 *   NOT bitwise deterministic (the shared-memory sums' order varies); every other output is.
 * rp_ti_pos_add: kv bf16 [T, ld_kv] columns [0, d) += dropout(pos_k[t % L]), [d, 2d) += dropout(pos_v[t % L]) (sites off_k /
 *   off_v, row key t, column c of its table); rp_ti_pos_bwd: d_pos_k / d_pos_v fp32 [L, d] += sum over b in order of the
 *   dropout' of dkv's two halves (deterministic), true columns (c % 64 < head_dim) only. */
#define RP_TI_MAX_SPAN 320
#define RP_TI_MAX_COLS 256
typedef struct rp_ti_attn_desc {
  const void* q; long long ldq;
  const uint8_t* pad_mask;
  const void* times; int times_dtype;
  const void* time_k; const void* time_v; long long ld_t;
  int B, H, L, head_dim, time_span;
  float scale;
  float drop_p; unsigned long long seed; const unsigned long long* seed_ptr;
  unsigned long long att_off, tk_off, tv_off;
} rp_ti_attn_desc;
int rp_ti_attn_fwd(const rp_ti_attn_desc* p, const float* s, const void* q_in, void* a_save, void* ad, void* hpre,
                   void* stream);
size_t rp_ti_attn_bwd_workspace(int B, int H, int time_span);
int rp_ti_attn_bwd(const rp_ti_attn_desc* p, const void* a_save, void* dpd, void* ad, const void* d_o, void* dq_t, void* ws,
                   size_t ws_bytes, float* d_time_k, float* d_time_v, void* stream);
int rp_ti_pos_add(void* kv, long long ld_kv, const float* pos_k, const float* pos_v, int T, int L, int d, float drop_p,
                  unsigned long long seed, const unsigned long long* seed_ptr, unsigned long long off_k,
                  unsigned long long off_v, void* stream);
int rp_ti_pos_bwd(const void* dkv, long long ld_kv, int B, int L, int d, int head_dim, float drop_p, unsigned long long seed,
                  const unsigned long long* seed_ptr, unsigned long long off_k, unsigned long long off_v, float* d_pos_k,
                  float* d_pos_v, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* RP_B200_H */
