// rp_ce_head.cu - fused full-catalog cross-entropy head (training), forward and backward, without ever materialising the
// [tokens, items] logits.
//
// Replaces   logits = hidden . E^T               replay/nn/head.py:29-34, replay/nn/sequential/sasrec/model.py:258-265
//            torch.nn.CrossEntropyLoss(mean)     replay/nn/loss/ce.py:49-81 ; models/nn/sequential/sasrec/lightning.py:335-355
// and their autograd backward (dHidden, dE).
//
// Inputs are the COMPACTED valid-target rows Hc[T_v, d] (bf16, capacity T rows; T_v lives in device memory so the whole
// step stays CUDA-graph capturable), the item table E[I, d] (bf16) and labels[T_v].
//
//   ce_fwd_kernel      CTA = 128 tokens x an item split.  S = Hc.E^T tile by tile (wgmma, registers); an online
//                      (max, sum-exp) per row.                                                  -> partial (m, s)
//   ce_finalize_kernel lse, loss = mean(lse - z_y), per-token exponent offset c_t = -lse*log2e + log2(1/T_v)
//   ce_bwd_kernel<ROW> CTA = 128 tokens, loops over item tiles:   G = exp2(S*log2e + c_row) (bf16, kept in registers as
//                      the A operand), dH += G . E_tile  (B = the same smem tile, MN-major)
//                      final: dH[t] -= E[y_t] / T_v                                             -> dHc bf16 [T_v, d]
//   ce_bwd_kernel<COL> CTA = 128 items, loops over token tiles:   S^T = E_tile . Hc^T, G = exp2(S^T*log2e + c_col),
//                      dE += G . Hc_tile                                                          -> dE fp32 [I, d] (=)
//   ce_label_scatter   dE[y_t] -= Hc[t] / T_v   (the one-hot part of softmax - onehot, sparse)
//
// The full-catalog BCE head (rp_bce_head_*) runs on the same tile loops:
//   loss = (1/T_v) sum_t [ sum_i softplus(x_ti) - x_t,y_t ],  x = s + b,  dx = (sigmoid(x) - onehot) / T_v
// replacing  BCEWithLogitsLoss(sum) / T_v            replay/nn/loss/bce.py:10-95 ; bert4rec/lightning.py:273-305
//   ce_bwd_kernel<3>   rows = tokens: G = sigmoid(S + b) (bf16 A operand), dH += G . E_tile, row sums of softplus
//   ce_bwd_kernel<4>   rows = items: G = sigmoid(S^T + b_row) over the valid tokens, dE = G . Hc / T_v, d_bias = rowsum / T_v
//   ce_fwd_kernel<BCE> row sums of softplus only (the un-fused forward, and the loss at d = 512)
// The sigmoid is bounded, so there is no log-sum-exp, no bound guard and no second pass; rows past T_v and columns past the
// split end are masked explicitly (sigmoid(0) = 1/2 would leak where CE's exp(-inf) = 0 does not).
#include <type_traits>

#include "rp_host.h"
#include "rp_gemm_desc.h"
#include "rp_sm90.cuh"

namespace rp {

static constexpr int kT = 128;                  // tile edge (rows per CTA, columns per MMA tile)
static constexpr int kChunk = 128 * 128;        // bytes of one [128 rows x 64 bf16] swizzled chunk
static constexpr float kLog2e = 1.4426950408889634f;
static constexpr float kLn2 = 0.6931471805599453f;
// CTA layout of the head kernels: warpgroups 0 / 1 own rows [0, 64) / [64, 128) of the row tile; the same threads also feed
// the TMA ring (a separate producer warp would cap the registers of the accumulating threads)
static constexpr int kThreads = 256;
static constexpr int kTN = 64;                  // grid of the column splits of the fused pass (ce_bwd_kernel tiles: TN)

// BCE per logit x, with e = exp(-|x|):  sigmoid = (x >= 0 ? 1 : e) / (1 + e),  softplus = max(x, 0) + log1p(e).
// The log1p terms are summed as lg2 of the product of a column tile's (1 + e) factors (at most 32 per thread and row, each in
// (1, 2], so the product stays below 2^32): a logit costs two special-function operations (ex2, rcp) instead of three.
__device__ __forceinline__ float bce_sigmoid(float x, float& one_plus_e) {
  const float e = ex2f(-fabsf(x) * kLog2e);
  one_plus_e = 1.f + e;
  return __fdividef(x >= 0.f ? 1.f : e, one_plus_e);
}
// ----------------------------------------------------------------------------------------------------------------
// forward
// ----------------------------------------------------------------------------------------------------------------
// BCE = true: per (row, split) sum of softplus(s + b) over the split's columns instead of the (max, sum-exp) pair; `part` then
// holds floats, element (t, split) at [t * n_splits + split].
template <int KCH, int NSTAGE, bool BCE = false>
__global__ void __launch_bounds__(kThreads, 1)
ce_fwd_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
              const int32_t* __restrict__ n_valid_ptr, int n_items, int n_splits, const float* __restrict__ bias,
              float2* __restrict__ part /* [T, n_splits] (m in log2 units, s) */,
              const int32_t* __restrict__ skip_if_safe) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sA = smem;
  uint8_t* sB = smem + KCH * kChunk;
  __shared__ uint64_t bar_a, bar_full[NSTAGE], bar_empty[NSTAGE];

  const int lane = threadIdx.x & 31;
  const int tok_tile = blockIdx.x / n_splits, split = blockIdx.x % n_splits;
  if (skip_if_safe && *skip_if_safe != 0) return;  // the fused pass covers this step
  const int n_valid = *n_valid_ptr;
  const int t0 = tok_tile * kT;
  if (t0 >= n_valid) return;  // uniform for the CTA
  const int n_tiles_total = (n_items + kT - 1) / kT;
  const int j_begin = (int)(((long long)n_tiles_total * split) / n_splits);
  const int j_end = (int)(((long long)n_tiles_total * (split + 1)) / n_splits);

  if (threadIdx.x == 0) {
    mbar_init(&bar_a, 1);
    for (int i = 0; i < NSTAGE; ++i) {
      mbar_init(&bar_full[i], 1);
      mbar_init(&bar_empty[i], 8);
    }
    fence_barrier_init();
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
  }
  __syncthreads();
  const int n_chunks = (j_end - j_begin) * KCH;
  auto issue = [&](int i) {   // thread 0: chunk i of the item tiles -> stage i % NSTAGE
    const uint32_t s = i % NSTAGE;
    mbar_wait(&bar_empty[s], ((i / NSTAGE) & 1) ^ 1);
    mbar_arrive_expect_tx(&bar_full[s], kChunk);
    tma_load_2d(sB + s * kChunk, &tmB, &bar_full[s], (i % KCH) * 64, (j_begin + i / KCH) * kT);
  };
  if (threadIdx.x == 0) {
    mbar_arrive_expect_tx(&bar_a, KCH * kChunk);
    for (int kc = 0; kc < KCH; ++kc) tma_load_2d(sA + kc * kChunk, &tmA, &bar_a, kc * 64, t0);
    for (int i = 0; i < NSTAGE && i < n_chunks; ++i) issue(i);
  }
  const int t = threadIdx.x & 127, wg = threadIdx.x >> 7;
  const int fc = frag_col(t);
  const int ta = t0 + 64 * wg + frag_row(t), tb = ta + 8;   // the two token rows of this thread
  float ma = -1e30f, sa = 0.f, mb = -1e30f, sb = 0.f;      // m in log2 units
  mbar_wait(&bar_a, 0);
  uint32_t it = 0;
  for (int j = j_begin; j < j_end; ++j) {
    float acc[kT / 2];
    for (int kc = 0; kc < KCH; ++kc, ++it) {
      const uint32_t s = it % NSTAGE, ph = (it / NSTAGE) & 1;
      mbar_wait(&bar_full[s], ph);
      const uint32_t a0 = smem_u32(sA + kc * kChunk) + wg * 8192, b0 = smem_u32(sB + s * kChunk);
      wg_fence();
#pragma unroll
      for (int ks = 0; ks < 4; ++ks) WgmmaSS<kT>::template run<0, 0>(acc, desc_k(a0 + ks * 32), desc_k(b0 + ks * 32), (kc | ks) != 0);
      wg_commit();
      wg_wait<0>();
      wg_fence_acc(acc);
      __syncwarp();
      if (lane == 0) mbar_arrive(&bar_empty[s]);
      if (threadIdx.x == 0 && (int)it + NSTAGE < n_chunks) issue((int)it + NSTAGE);
    }
    const int col0 = j * kT + fc;
#pragma unroll
    for (int q = 0; q < kT / 8; ++q)
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int col = col0 + 8 * q + e;
        const float b = (bias && col < n_items) ? __ldg(bias + col) : 0.f;   // untied / biased head (BERT4Rec)
        const bool in = col < n_items;                                        // ragged last tile
        acc[4 * q + e] = in ? acc[4 * q + e] + b : -INFINITY;
        acc[4 * q + 2 + e] = in ? acc[4 * q + 2 + e] + b : -INFINITY;
      }
    if constexpr (BCE) {   // softplus(-inf) = max(-inf, 0) + lg2(1 + 0) = 0: the masked columns add nothing
      float pa = 1.f, pb = 1.f, xa = 0.f, xb = 0.f;
#pragma unroll
      for (int q = 0; q < kT / 8; ++q)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const float va = acc[4 * q + e], vb = acc[4 * q + 2 + e];
          xa += fmaxf(va, 0.f);
          xb += fmaxf(vb, 0.f);
          pa *= 1.f + ex2f(-fabsf(va) * kLog2e);
          pb *= 1.f + ex2f(-fabsf(vb) * kLog2e);
        }
      sa += xa + __log2f(pa) * kLn2;
      sb += xb + __log2f(pb) * kLn2;
      continue;
    }
    float cma = -INFINITY, cmb = -INFINITY;
#pragma unroll
    for (int q = 0; q < kT / 8; ++q) {
      cma = fmaxf(cma, fmaxf(acc[4 * q], acc[4 * q + 1]));
      cmb = fmaxf(cmb, fmaxf(acc[4 * q + 2], acc[4 * q + 3]));
    }
    const float mna = fmaxf(ma, cma * kLog2e), mnb = fmaxf(mb, cmb * kLog2e);
    sa *= ex2f(ma - mna);
    sb *= ex2f(mb - mnb);
    ma = mna;
    mb = mnb;
    float xa = 0.f, xb = 0.f;
#pragma unroll
    for (int q = 0; q < kT / 8; ++q) {
      xa += ex2f(fmaf(acc[4 * q], kLog2e, -mna)) + ex2f(fmaf(acc[4 * q + 1], kLog2e, -mna));
      xb += ex2f(fmaf(acc[4 * q + 2], kLog2e, -mnb)) + ex2f(fmaf(acc[4 * q + 3], kLog2e, -mnb));
    }
    sa += xa;
    sb += xb;
  }
  if constexpr (BCE) {
    sa = quad_sum(sa);
    sb = quad_sum(sb);
    float* zrow = reinterpret_cast<float*>(part);
    if (fc == 0) {
      if (ta < n_valid) zrow[(size_t)ta * n_splits + split] = sa;
      if (tb < n_valid) zrow[(size_t)tb * n_splits + split] = sb;
    }
  } else {
    // the four threads of a quad hold the same rows: merge their (max, sum) pairs
#pragma unroll
    for (int o = 1; o <= 2; o <<= 1) {
      const float oma = __shfl_xor_sync(0xffffffffu, ma, o), osa = __shfl_xor_sync(0xffffffffu, sa, o);
      const float omb = __shfl_xor_sync(0xffffffffu, mb, o), osb = __shfl_xor_sync(0xffffffffu, sb, o);
      const float na = fmaxf(ma, oma), nb = fmaxf(mb, omb);
      sa = sa * ex2f(ma - na) + osa * ex2f(oma - na);
      sb = sb * ex2f(mb - nb) + osb * ex2f(omb - nb);
      ma = na;
      mb = nb;
    }
    if (fc == 0) {
      if (ta < n_valid) part[(size_t)ta * n_splits + split] = make_float2(ma, sa);
      if (tb < n_valid) part[(size_t)tb * n_splits + split] = make_float2(mb, sb);
    }
  }
}

// Per-row variants of the full-catalog head (all single positive label per position):
//   w_ext   sample weights of the valid targets (compacted order): loss = mean_t w_t ce_t
//           replay/nn/loss/logout_ce.py:148-228 LogOutCEWeighted ; replay/nn/loss/ce.py:84-143 CEWeighted
//   kind 1  LogInCE (replay/nn/loss/login_ce.py:170-239): loss_t = -clamp(log(p_t + eps), -c, c), p_t = softmax prob of
//           the positive; its gradient is the CE gradient of the row times p / (p + eps) (0 where the clamp is active)
// Both act as a per-row factor w_t on (softmax - onehot) / T_v: the forward's finalisation writes it to roww[t], folds it into
// the exponent offset cvec[t] = -lse2 + log2(w_t / T_v) the gradient passes exponentiate with, and the one-hot terms read it.
struct CeRowOpts {
  const float* w_ext;    // [capacity] or null
  float* roww;           // [capacity] gradient weight per row (workspace); null only for the plain head without workspace
  int kind;              // 0 CE, 1 LogInCE
  float log_eps, clamp;
};
// row loss and gradient weight from the log-sum-exp (natural log) and the target logit
__device__ __forceinline__ void ce_row_terms(const CeRowOpts& o, int t, float lse, float zy, float& row_loss, float& wg) {
  const float wx = o.w_ext ? o.w_ext[t] : 1.f;
  float lt = lse - zy;
  wg = wx;
  if (o.kind == 1) {
    const float pr = __expf(zy - lse);
    const float lg = __logf(pr + o.log_eps);
    lt = -fminf(fmaxf(lg, -o.clamp), o.clamp);
    wg *= (lg > -o.clamp && lg < o.clamp) ? pr / (pr + o.log_eps) : 0.f;
  }
  row_loss = wx * lt;
}

// lse / loss / per-token exponent offsets.  One warp per token: merges the (max, sum) partials, computes the target logit
// z_y = hc[t] . E[y_t] as a gather-dot (keeps the per-element target pick out of the MMA epilogue), accumulates the loss.
// Deterministic: per-block partial sums, the last block adds them in index order.
__global__ void ce_finalize_kernel(const float2* __restrict__ part, const __nv_bfloat16* __restrict__ hc,
                                   const __nv_bfloat16* __restrict__ table, const int32_t* __restrict__ labels,
                                   const float* __restrict__ bias, const int32_t* __restrict__ n_valid_ptr, int n_part,
                                   int capacity, int d,
                                   float* __restrict__ lse_out, float* __restrict__ cvec, float* __restrict__ block_sums,
                                   unsigned int* __restrict__ ticket, float* __restrict__ loss_out,
                                   const int32_t* __restrict__ skip_if_safe, const CeRowOpts row) {
  if (skip_if_safe && *skip_if_safe != 0) return;
  const int n_valid = *n_valid_ptr;
  const float inv_n = n_valid > 0 ? 1.f / (float)n_valid : 0.f;
  const int lane = threadIdx.x & 31, wpb = blockDim.x >> 5;
  float local = 0.f;
  for (int t = blockIdx.x * wpb + (threadIdx.x >> 5); t < capacity; t += gridDim.x * wpb) {
    if (t < n_valid) {
      const float2* p = part + (size_t)t * n_part;
      float M = -1e30f;
      for (int i = lane; i < n_part; i += 32) M = fmaxf(M, p[i].x);
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) M = fmaxf(M, __shfl_xor_sync(0xffffffffu, M, o));
      float S = 0.f;
      for (int i = lane; i < n_part; i += 32) S += p[i].y * exp2f(p[i].x - M);
      const __nv_bfloat16* hr = hc + (size_t)t * d;
      const __nv_bfloat16* er = table + (size_t)labels[t] * d;
      float z = 0.f;
      for (int c = lane * 2; c < d; c += 64) {
        const float2 a = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(hr + c));
        const float2 b = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(er + c));
        z = fmaf(a.x, b.x, z);
        z = fmaf(a.y, b.y, z);
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        S += __shfl_xor_sync(0xffffffffu, S, o);
        z += __shfl_xor_sync(0xffffffffu, z, o);
      }
      if (bias) z += bias[labels[t]];
      const float lse2 = M + log2f(S);  // log2 units
      const float lse = lse2 * kLn2;
      if (lane == 0) {
        float rl, wg;
        ce_row_terms(row, t, lse, z, rl, wg);
        lse_out[t] = lse;
        cvec[t] = -lse2 + log2f(wg * inv_n);
        if (row.roww) row.roww[t] = wg;
        local += rl;
      }
    } else if (lane == 0) {
      cvec[t] = -INFINITY;  // rows beyond T_v contribute nothing to the backward
    }
  }
  __shared__ float red[32];
  __shared__ bool last;
  if (lane == 0) red[threadIdx.x >> 5] = local;
  __syncthreads();
  if (threadIdx.x == 0) {
    float s = 0.f;
    for (int i = 0; i < wpb; ++i) s += red[i];
    block_sums[blockIdx.x] = s;
    __threadfence();
    last = (atomicAdd(ticket, 1u) == gridDim.x - 1);
  }
  __syncthreads();
  if (last && threadIdx.x == 0) {
    __threadfence();
    float s = 0.f;
    for (int i = 0; i < (int)gridDim.x; ++i) s += reinterpret_cast<volatile float*>(block_sums)[i];
    loss_out[0] = s * inv_n;  // mean over valid targets
    loss_out[1] = inv_n;
  }
}

// Direct completion of the fused pass when the catalog is NOT split over CTAs (n_splits == 1: the CTA has seen every item of
// its 128 tokens): lse, exponent offsets, per-row loss terms and the final bf16 dH are written from the accumulator itself, so
// the partial-gradient round trip through HBM (2 x T_v x d fp32) and ce_fused_finalize_kernel disappear.
struct CeDirect {
  __nv_bfloat16* d_hc;   // null: column-split mode (partials + ce_fused_finalize_kernel)
  float* lse;
  float* cvec;
  float* row_loss;       // [capacity] weighted row losses; summed in a fixed order by ce_loss_reduce_kernel
  CeRowOpts row;         // (row.roww is also what MODE 0 scales its one-hot term with)
  int use_lse_off;       // fused pass as the FALLBACK's gradient pass: exponent offset of row t = -lse[t] (from the two-pass
                         // forward) instead of the fixed reference 0, so G is the softmax itself (z ~ 1) whatever |logit| is
};

// exponent offset of row r in the fused pass (log2 units): 0, or -lse[r] behind the two-pass forward; -inf beyond T_v
__device__ __forceinline__ float crow_of(const CeDirect& d, int r, int n_valid) {
  return r < n_valid ? (d.use_lse_off ? -d.lse[r] * kLog2e : 0.f) : -INFINITY;
}

// loss = mean over the valid targets of row_loss, deterministic (fixed partition + tree); also publishes 1 / T_v
__global__ void __launch_bounds__(1024) ce_loss_reduce_kernel(const float* __restrict__ row_loss, const int32_t* __restrict__ n_valid_ptr,
                                                              const int32_t* __restrict__ safe_flag, float* __restrict__ loss_out,
                                                              int run_if_safe) {
  if (safe_flag && (*safe_flag != 0) != (run_if_safe != 0)) return;
  __shared__ float red[1024];
  const int n_valid = *n_valid_ptr;
  float a = 0.f;
  for (int i = threadIdx.x; i < n_valid; i += 1024) a += row_loss[i];
  red[threadIdx.x] = a;
  __syncthreads();
  for (int o = 512; o > 0; o >>= 1) {
    if ((int)threadIdx.x < o) red[threadIdx.x] += red[threadIdx.x + o];
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    const float inv_n = n_valid > 0 ? 1.f / (float)n_valid : 0.f;
    loss_out[0] = red[0] * inv_n;
    loss_out[1] = inv_n;
  }
}

// ----------------------------------------------------------------------------------------------------------------
// backward (both directions share one kernel)
//   COLCONST = false : rows = tokens (A = Hc tile), columns = items  -> acc = dHc tile [128, d]
//   COLCONST = true  : rows = items  (A = E tile),  columns = tokens -> acc = dE tile  [128, d]
// ----------------------------------------------------------------------------------------------------------------
// MODE 0: rows = tokens, G = softmax/T_v from the stored lse (two-pass fallback)      -> out = dHc bf16
// MODE 1: rows = items (COLCONST), columns = tokens                                    -> out = dE fp32
// MODE 2: rows = tokens, FUSED forward+backward: G~ = exp(s + b) with reference max 0 (valid while |s| is bounded, see
//         ce_bound_kernel), per-row sum of G~ and un-normalised dH~ = sum_i G~ E_i over this CTA's column split
//                                                                                      -> out = partial dH~ fp32, zpart
// CTA = one 128-row tile against the columns [c_begin, c_end) in n_ct tiles of TN columns.  Per column tile: S = A_tile .
// B_tile^T (wgmma, registers), G = exp2(S log2e + offset) in registers, acc += G . B_tile with G as the register A operand
// and the same shared-memory B tile read MN-major.  At the end the [128 x D] accumulator goes through shared memory to the
// row-wise epilogue (thread = row, warpgroup = half of the D columns).
// TN = 128 halves how often the A tile is read from shared memory per column (the S wgmma at N = 64 needs as many bytes per
// cycle as shared memory delivers); d = 256 keeps TN = 64 because a 128-column S does not fit next to its accumulator.
// BCE (rp_bce_head_*), G = sigmoid(x) masked to the live columns, no exponent offsets:
// MODE 3: rows = tokens, the fused pass's split grid: row sums of softplus, dH~ = sum_i G E_i; without column splits
//         d_hc = (dH~ - E[y]) / T_v and the row losses are final (direct.d_hc / direct.row_loss); else partials, zpart
// MODE 4: rows = items (COLCONST), columns = the valid tokens: dE = G . Hc / T_v, d_bias = row sums of G / T_v, the bias of
//         the item row inside the sigmoid
// Eighths of the CE passes' exponentials (MODE 1 and MODE 2) that ex2_poly computes on the FMA pipe instead of MUFU.EX2:
// the fragment columns 8 q + {0, 1} with q % 8 < k, the same columns in every tile.  Per logit the S and dH / dE MMAs cost
// 4 d FLOP and the exponential one MUFU op, so the special-function unit's share grows as d shrinks; the polynomial costs
// ten FMA / integer instructions instead.  Measured on an H100 SXM 80GB at 700 W for k = 1..4 at d = 64, 128 and 256, with and
// without bias (README, "Headroom left"): every k > 0 slowed both passes at d = 128 (config 2, k = 1: fused pass +13 %, dE
// pass +5 %); at d = 64 and 256 only the biased dE pass gained (about 3 % at k = 1) while the unbiased one lost.  So every
// instantiation keeps MUFU.EX2, and k = 0 compiles to the same code as the loop without the split.
__host__ __device__ constexpr int ce_poly_eighths(int /*kch*/, int /*tn*/, int /*mode*/) { return 0; }
template <int KCH, int NSTAGE, int TN, int MODE, bool HAS_BIAS>
__global__ void __launch_bounds__(kThreads, 1)
ce_bwd_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
              const __nv_bfloat16* __restrict__ a_rows /* the row-side matrix (tmA) as a plain pointer */,
              const float* __restrict__ cvec /* [T] exponent offsets per token */, const int32_t* __restrict__ labels,
              const __nv_bfloat16* __restrict__ table, const float* __restrict__ loss_inv /* [1] = 1/T_v */,
              const int32_t* __restrict__ n_valid_ptr, int n_items, const float* __restrict__ bias,
              float* __restrict__ d_bias, void* __restrict__ out, const int32_t* __restrict__ safe_flag, int run_if_safe,
              int n_splits, int capacity, float* __restrict__ zpart, const CeDirect direct) {
  constexpr bool BCE = (MODE >= 3);
  constexpr bool COLCONST = (MODE == 1 || MODE == 4);
  constexpr bool FUSED = (MODE == 2 || MODE == 3);
  constexpr int D = KCH * 64;
  constexpr int kChunkB = TN * 128;       // bytes of one [TN rows x 64 bf16] swizzled chunk of a column tile
  constexpr int kStage = KCH * kChunkB;   // one column tile in shared memory
  constexpr int PITCH = D + 4;            // fp32 accumulator stage (over the ring once the column tiles are done)
  constexpr int kSlots = 2, DW = D / kSlots;
  // MODE 1: the column tile's TN exponent offsets ride the ring in a slot of their own (launch_ce_bwd sizes them), behind the ring and the
  // accumulator stage that reuses it; they are in shared memory once the tile is, so the exponentials never wait on a load
  constexpr bool OFF_RING = COLCONST && !BCE;
  constexpr int kOffBytes = TN * 4;
  constexpr int kPolyEighths = ce_poly_eighths(KCH, TN, MODE);
  if (safe_flag && (*safe_flag != 0) != (run_if_safe != 0)) return;  // fused path vs two-pass fallback (uniform)
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sA = smem;
  uint8_t* sB = smem + KCH * kChunk;
  float* sOff = reinterpret_cast<float*>(sB + (NSTAGE * kStage > kT * PITCH * 4 ? NSTAGE * kStage : kT * PITCH * 4));
  __shared__ float s_row[kT];             // per-row sum of G (FUSED) / of G before the item factor (COLCONST with bias)
  __shared__ float s_dot[kSlots][kT];
  __shared__ uint64_t bar_a, bar_full[NSTAGE];
  __shared__ uint32_t s_released[NSTAGE];   // warps that have released the stage, over all its tiles

  const int lane = threadIdx.x & 31;
  const int n_valid = *n_valid_ptr;
  const int split = FUSED ? blockIdx.x % n_splits : 0;
  const int n_rows = COLCONST ? n_items : n_valid;
  const int n_cols = COLCONST ? n_valid : n_items;
  // column split of the fused pass on a grid of kTN columns whatever TN is, so the splits (and the order in which their
  // partial sums are added) do not depend on the tile size; a split's last tile is masked at c_end
  const int n_grid = (n_cols + kTN - 1) / kTN;
  const int row_tile = FUSED ? blockIdx.x / n_splits : blockIdx.x;
  const int c_begin = FUSED ? (int)(((long long)n_grid * split) / n_splits) * kTN : 0;
  const int c_end = FUSED ? min(n_cols, (int)(((long long)n_grid * (split + 1)) / n_splits) * kTN) : n_cols;
  const int n_ct = c_end > c_begin ? (c_end - c_begin + TN - 1) / TN : 0;
  const int r0 = row_tile * kT;
  if (r0 >= n_rows) return;

  if (threadIdx.x == 0) {
    mbar_init(&bar_a, 1);
    for (int i = 0; i < NSTAGE; ++i) {
      mbar_init(&bar_full[i], 1);
      s_released[i] = 0;
    }
    fence_barrier_init();
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
  }
  __syncthreads();
  // column tile jl -> stage jl % NSTAGE.  Thread 0 fills the ring; after that, the last of the 8 warps to release a stage
  // refills it, so no warp ever waits for the other warpgroup and the two can run out of phase.
  auto issue = [&](int jl) {
    const uint32_t s = jl % NSTAGE;
    mbar_arrive_expect_tx(&bar_full[s], kStage + (OFF_RING ? kOffBytes : 0));
    for (int kc = 0; kc < KCH; ++kc) tma_load_2d(sB + s * kStage + kc * kChunkB, &tmB, &bar_full[s], kc * 64, c_begin + jl * TN);
    // cvec holds round_up(capacity, 128) entries, -inf past the valid tokens: the last tile's slot is read in full
    if (OFF_RING) bulk_load_1d(sOff + s * TN, cvec + c_begin + jl * TN, kOffBytes, &bar_full[s]);
  };
  if (threadIdx.x == 0) {
    mbar_arrive_expect_tx(&bar_a, KCH * kChunk);
    for (int kc = 0; kc < KCH; ++kc) tma_load_2d(sA + kc * kChunk, &tmA, &bar_a, kc * 64, r0);
    for (int jl = 0; jl < NSTAGE && jl < n_ct; ++jl) issue(jl);
  }
  const int t = threadIdx.x & 127, wg = threadIdx.x >> 7;
  const int fc = frag_col(t);
  const int rla = 64 * wg + frag_row(t), rlb = rla + 8;   // this thread's rows inside the tile
  float crow_a = 0.f, crow_b = 0.f;
  if (MODE == 0) {
    crow_a = (r0 + rla < n_valid) ? cvec[r0 + rla] : -INFINITY;
    crow_b = (r0 + rlb < n_valid) ? cvec[r0 + rlb] : -INFINITY;
  }
  if (FUSED && !BCE) {
    crow_a = (r0 + rla < n_valid) ? (direct.use_lse_off ? -direct.lse[r0 + rla] * kLog2e : 0.f) : -INFINITY;
    crow_b = (r0 + rlb < n_valid) ? (direct.use_lse_off ? -direct.lse[r0 + rlb] * kLog2e : 0.f) : -INFINITY;
  }
  float brow_a = 0.f, brow_b = 0.f;   // MODE 4: bias of this thread's item rows
  if (BCE && COLCONST && HAS_BIAS) {
    brow_a = r0 + rla < n_items ? __ldg(bias + r0 + rla) : 0.f;
    brow_b = r0 + rlb < n_items ? __ldg(bias + r0 + rlb) : 0.f;
  }
  float za = 0.f, zb = 0.f;   // FUSED: row sums of G~ (BCE: of softplus); COLCONST with bias: row sums of G (bias gradient)
  float acc[D / 2];
  acc_zero(acc);
  float sacc[TN / 2];
  mbar_wait(&bar_a, 0);
  const uint32_t a_base = smem_u32(sA) + wg * 8192;
  auto issue_s = [&](int jl) {   // S = A_tile . B_tile^T of column tile jl into sacc, one commit group
    mbar_wait(&bar_full[jl % NSTAGE], (jl / NSTAGE) & 1);
    const uint32_t b0 = smem_u32(sB + (jl % NSTAGE) * kStage);
    wg_fence();
#pragma unroll
    for (int kc = 0; kc < KCH; ++kc)
#pragma unroll
      for (int ks = 0; ks < 4; ++ks)
        WgmmaSS<TN>::template run<0, 0>(sacc, desc_k(a_base + kc * kChunk + ks * 32), desc_k(b0 + kc * kChunkB + ks * 32),
                                        (kc | ks) != 0);
    wg_commit();
  };
  // S of the next tile goes out behind dH (below), which keeps all of sacc live beside pk and acc; the BCE token pass, which
  // also carries softplus's terms, would spill at d = 64 and d = 256, so it issues S after dH retires.
  constexpr bool kSAhead = MODE != 3;
  if (n_ct > 0) {
    issue_s(0);
    wg_wait<0>();
    wg_fence_acc(sacc);
  }
  // With S ahead, the warpgroups take turns issuing {dH(j), S(j+1)} (named barriers 2 / 3, warpgroup 0 first), so that one
  // warpgroup's exponentials run while the other's MMAs hold the tensor pipe.  The counts match: warpgroup 1 arrives once up
  // front and skips its arrival after the last tile.
  if (kSAhead && wg == 1 && n_ct > 0) named_bar_arrive(2, 256);
  for (int jl = 0; jl < n_ct; ++jl) {
    const uint32_t s = jl % NSTAGE;
    const uint32_t b0 = smem_u32(sB + s * kStage);
    // G = exp2(S log2e + offset) -> bf16 A fragments
    const int col0 = c_begin + jl * TN + fc;
    uint32_t pk[TN / 4];
    if constexpr (BCE) {
      // G = sigmoid(S + b) on the live columns (items before the split end / valid tokens), 0 elsewhere
      float pa = 1.f, pb = 1.f;   // MODE 3: products of (1 + e) over this tile's live columns
#pragma unroll
      for (int q = 0; q < TN / 8; ++q) {
        float g[4];
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int col = col0 + 8 * q + e;
          const bool in = col < c_end;
          float va = sacc[4 * q + e], vb = sacc[4 * q + 2 + e];
          if (HAS_BIAS) {
            const float ba = COLCONST ? brow_a : (in ? __ldg(bias + col) : 0.f);
            const float bb = COLCONST ? brow_b : ba;
            va += ba;
            vb += bb;
          }
          float oa, ob;
          const float sa = bce_sigmoid(va, oa), sb = bce_sigmoid(vb, ob);
          g[e] = in ? sa : 0.f;
          g[2 + e] = in ? sb : 0.f;
          if (FUSED) {
            za += in ? fmaxf(va, 0.f) : 0.f;
            zb += in ? fmaxf(vb, 0.f) : 0.f;
            pa *= in ? oa : 1.f;
            pb *= in ? ob : 1.f;
          }
        }
        if (COLCONST && HAS_BIAS) {
          za += g[0] + g[1];
          zb += g[2] + g[3];
        }
        pk[2 * q] = pack_bf16(g[0], g[1]);
        pk[2 * q + 1] = pack_bf16(g[2], g[3]);
      }
      if (FUSED) {
        za += __log2f(pa) * kLn2;
        zb += __log2f(pb) * kLn2;
      }
    } else {
      const float* off = sOff + s * TN + fc;   // COLCONST: offsets of this thread's columns, -inf beyond the valid tokens
      // Token rows: only a split's last column tile reaches past c_end, so every other tile runs without the per-column
      // compare and select (about one instruction per logit, on the path the other warpgroup's MMAs wait for)
      auto exps = [&](auto masked) {
        constexpr bool MASKED = decltype(masked)::value;
#pragma unroll
        for (int q = 0; q < TN / 8; ++q) {
          float g[4];
          float2 cq;
          // ld.shared: the aligned smem base goes through an integer, which hides the state space from the compiler and
          // made these generic loads (LD.E, about 0.2 ms of the dE pass at config 2).  volatile keeps it behind the tile's
          // mbarrier wait, which is what makes the offsets valid.
          if (COLCONST) asm volatile("ld.shared.v2.f32 {%0, %1}, [%2];" : "=f"(cq.x), "=f"(cq.y) : "r"(smem_u32(off + 8 * q)));
          // the same fragment columns of every tile take the polynomial, so a logit's value never depends on scheduling
          const bool poly = q % 8 < kPolyEighths;
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int col = col0 + 8 * q + e;
            float va = sacc[4 * q + e], vb = sacc[4 * q + 2 + e];
            if (COLCONST) {
              const float cc = e ? cq.y : cq.x;
              g[e] = poly ? ex2_poly(fmaf(va, kLog2e, cc)) : ex2f(fmaf(va, kLog2e, cc));
              g[2 + e] = poly ? ex2_poly(fmaf(vb, kLog2e, cc)) : ex2f(fmaf(vb, kLog2e, cc));
            } else {
              const bool in = !MASKED || col < c_end;
              if (HAS_BIAS && in) {
                const float bb = __ldg(bias + col);
                va += bb;
                vb += bb;
              }
              if (poly) {   // masked through the argument (2^-inf = 0): a select on the result would become a branch
                g[e] = ex2_poly(in ? fmaf(va, kLog2e, crow_a) : -INFINITY);
                g[2 + e] = ex2_poly(in ? fmaf(vb, kLog2e, crow_b) : -INFINITY);
              } else {
                g[e] = in ? ex2f(fmaf(va, kLog2e, crow_a)) : 0.f;
                g[2 + e] = in ? ex2f(fmaf(vb, kLog2e, crow_b)) : 0.f;
              }
            }
          }
          if (FUSED || (COLCONST && HAS_BIAS)) {
            za += g[0] + g[1];
            zb += g[2] + g[3];
          }
          pk[2 * q] = pack_bf16(g[0], g[1]);
          pk[2 * q + 1] = pack_bf16(g[2], g[3]);
        }
      };
      if (COLCONST || c_begin + (jl + 1) * TN > c_end) exps(std::true_type{});
      else exps(std::false_type{});
    }
    if constexpr (kSAhead && kPolyEighths > 0) {
      // G is complete before the turn: the barrier's thread count (256 whatever pk holds) depends on every pk word.  Without
      // it ptxas sinks the polynomial's arithmetic below the barrier, into the window where the other warpgroup waits.
      uint32_t all = 0;
#pragma unroll
      for (int i = 0; i < TN / 4; ++i) all |= pk[i];
      uint32_t n;
      asm volatile("{\n\t.reg .u32 t;\n\tor.b32 t, %1, 256;\n\tmin.u32 %0, t, 256;\n\t}" : "=r"(n) : "r"(all));
      named_bar_sync(2 + wg, (int)n);
    } else if (kSAhead) {
      named_bar_sync(2 + wg, 256);   // this warpgroup's turn
    }
    wg_fence();
#pragma unroll
    for (int kk = 0; kk < TN / 16; ++kk) {
      const uint32_t af[4] = {pk[4 * kk], pk[4 * kk + 1], pk[4 * kk + 2], pk[4 * kk + 3]};
      WgmmaRS<D>::template run<1>(acc, af, desc_mn(b0 + kk * 2048, kChunkB), 1);
    }
    wg_commit();
    // S of the next tile in its own commit group: wait<1> retires dH (the stage and pk are free again), wait<0> then S, whose
    // exponentials start the next iteration.  The waits are unconditional (the last tile commits an empty group instead of
    // S): ptxas follows both sides of a branch and would otherwise find S pending at the loop head and serialize every wgmma
    // of the kernel.
    const bool more = jl + 1 < n_ct;
    if constexpr (kSAhead) {
      if (more) issue_s(jl + 1);
      else wg_commit();
      if (wg == 0) named_bar_arrive(3, 256);   // the other warpgroup's turn
      else if (more) named_bar_arrive(2, 256);
      wg_wait<1>();
    } else {
      wg_wait<0>();
    }
    wg_fence_acc(acc);
    __syncwarp();
    // the counter's acq_rel orders every warp's completed wgmma reads of the stage before the TMA write that refills it
    if (lane == 0 && jl + NSTAGE < n_ct && smem_count_acq_rel(&s_released[s]) % 8 == 7) {
      fence_proxy_async();
      issue(jl + NSTAGE);
    }
    if (!kSAhead && more) issue_s(jl + 1);
    wg_wait<0>();
    wg_fence_acc(sacc);
  }
  // ---- row sums (the quad's threads share rows) and the accumulator stage
#pragma unroll
  for (int o = 1; o <= 2; o <<= 1) {
    za += __shfl_xor_sync(0xffffffffu, za, o);
    zb += __shfl_xor_sync(0xffffffffu, zb, o);
  }
  if (fc == 0) {
    s_row[rla] = za;
    s_row[rlb] = zb;
  }
  named_bar_sync(1, 256);   // both warpgroups are done with the ring
  float* stage = reinterpret_cast<float*>(sB);
  acc_to_stage(acc, stage, PITCH, 64 * wg, 0);
  named_bar_sync(1, 256);
  // ---- final: thread = row, warpgroup = slot of DW accumulator columns
  const int row = t, slot = wg;
  const int r = r0 + row;
  const float* arow = stage + row * PITCH + slot * DW;
  if constexpr (BCE) {
    const float inv_n = n_valid > 0 ? 1.f / (float)n_valid : 0.f;
    if (COLCONST) {
      // dE = G^T-part / T_v and d_bias = sum_t sigmoid / T_v; the one-hot part follows in ce_label_scatter_kernel
      if (r < n_items) {
        if (HAS_BIAS && slot == 0) d_bias[r] = s_row[row] * inv_n;
        float4* dst = reinterpret_cast<float4*>(reinterpret_cast<float*>(out) + (size_t)r * D + slot * DW);
#pragma unroll 4
        for (int c = 0; c < DW; c += 4) {
          const float4 v = *reinterpret_cast<const float4*>(arow + c);
          dst[c >> 2] = make_float4(v.x * inv_n, v.y * inv_n, v.z * inv_n, v.w * inv_n);
        }
      }
    } else if (direct.d_hc != nullptr) {
      // no column splits: dH = (sum_i sigmoid_i E_i - E[y]) / T_v, row loss = sum_i softplus - x_y
      const bool live = r < n_valid;
      const int y = live ? labels[r] : 0;
      float dot = 0.f;
      if (live) {
        const uint4* ey = reinterpret_cast<const uint4*>(table + (size_t)y * D + slot * DW);
        const uint4* hr = reinterpret_cast<const uint4*>(a_rows + (size_t)r * D + slot * DW);
        uint4* dst = reinterpret_cast<uint4*>(direct.d_hc + (size_t)r * D + slot * DW);
#pragma unroll 4
        for (int q = 0; q < DW / 8; ++q) {
          const uint4 e = __ldg(ey + q), hh = __ldg(hr + q);
          const __nv_bfloat162* e2 = reinterpret_cast<const __nv_bfloat162*>(&e);
          const __nv_bfloat162* h2 = reinterpret_cast<const __nv_bfloat162*>(&hh);
          uint4 w;
          uint32_t* w32 = reinterpret_cast<uint32_t*>(&w);
#pragma unroll
          for (int pp = 0; pp < 4; ++pp) {
            const float2 ef = __bfloat1622float2(e2[pp]), hf = __bfloat1622float2(h2[pp]);
            dot = fmaf(hf.x, ef.x, fmaf(hf.y, ef.y, dot));
            w32[pp] = pack_bf16((arow[8 * q + 2 * pp] - ef.x) * inv_n, (arow[8 * q + 2 * pp + 1] - ef.y) * inv_n);
          }
          dst[q] = w;
        }
      }
      s_dot[slot][row] = dot;
      named_bar_sync(1, 256);
      if (slot == 0 && live) {
        float zy = s_dot[0][row] + s_dot[1][row];
        if (HAS_BIAS) zy += bias[y];
        direct.row_loss[r] = s_row[row] - zy;
      }
    } else {
      // partial (this column split) sums; bce_finalize_kernel reduces the splits in a fixed order
      float* o = reinterpret_cast<float*>(out) + (size_t)split * capacity * D;
      if (r < n_valid) {
        if (slot == 0) zpart[(size_t)split * capacity + r] = s_row[row];
        float4* dst = reinterpret_cast<float4*>(o + (size_t)r * D + slot * DW);
#pragma unroll 4
        for (int c = 0; c < DW; c += 4) dst[c >> 2] = *reinterpret_cast<const float4*>(arow + c);
      }
    }
  } else if (COLCONST) {
    float* o = reinterpret_cast<float*>(out);
    // biased head: G carries a per-item factor e^{b_i}; it was left out of the loop and is applied to the row here
    const float rs = (HAS_BIAS && r < n_items) ? __expf(bias[r]) : 1.f;
    if (HAS_BIAS && slot == 0 && r < n_items) d_bias[r] = s_row[row] * rs;
    if (r < n_items) {
      float4* dst = reinterpret_cast<float4*>(o + (size_t)r * D + slot * DW);
#pragma unroll 4
      for (int c = 0; c < DW; c += 4) {
        const float4 v = *reinterpret_cast<const float4*>(arow + c);
        dst[c >> 2] = make_float4(v.x * rs, v.y * rs, v.z * rs, v.w * rs);
      }
    }
  } else if (FUSED && direct.d_hc != nullptr) {
    // ---- no column splits: finish here.  z_t = row sum of G~; dH = acc / (z T_v) - E[y] / T_v
    const float z = s_row[row];
    const bool live = r < n_valid;
    const float inv_n = n_valid > 0 ? 1.f / (float)n_valid : 0.f;
    const int y = live ? labels[r] : 0;
    float wg_ = (live && direct.row.w_ext) ? direct.row.w_ext[r] : 1.f;   // gradient weight of the row
    if (direct.row.kind == 1) {
      // LogInCE: the weight needs the target logit before the gradient can be scaled - one extra pass over h . E[y]
      float dp = 0.f;
      if (live) {
        const uint4* ey = reinterpret_cast<const uint4*>(table + (size_t)y * D + slot * DW);
        const uint4* hr = reinterpret_cast<const uint4*>(a_rows + (size_t)r * D + slot * DW);
#pragma unroll 4
        for (int q = 0; q < DW / 8; ++q) {
          const uint4 e = __ldg(ey + q), hh = __ldg(hr + q);
          const __nv_bfloat162* e2 = reinterpret_cast<const __nv_bfloat162*>(&e);
          const __nv_bfloat162* h2 = reinterpret_cast<const __nv_bfloat162*>(&hh);
#pragma unroll
          for (int pp = 0; pp < 4; ++pp) {
            const float2 ef = __bfloat1622float2(e2[pp]), hf = __bfloat1622float2(h2[pp]);
            dp = fmaf(hf.x, ef.x, fmaf(hf.y, ef.y, dp));
          }
        }
      }
      s_dot[slot][row] = dp;
      named_bar_sync(1, 256);
      float zy0 = s_dot[0][row] + s_dot[1][row];
      if (HAS_BIAS) zy0 += bias[y];
      named_bar_sync(1, 256);   // s_dot is written again below
      float rl_unused;
      if (live) ce_row_terms(direct.row, r, __logf(z) - crow_of(direct, r, n_valid) * kLn2, zy0, rl_unused, wg_);
    }
    const float scale = live ? wg_ * inv_n / z : 0.f;
    const float lab = wg_ * inv_n;
    float dot = 0.f;
    if (live) {
      const uint4* ey = reinterpret_cast<const uint4*>(table + (size_t)y * D + slot * DW);
      const uint4* hr = reinterpret_cast<const uint4*>(a_rows + (size_t)r * D + slot * DW);
      uint4* dst = reinterpret_cast<uint4*>(direct.d_hc + (size_t)r * D + slot * DW);
#pragma unroll 4
      for (int q = 0; q < DW / 8; ++q) {
        const uint4 e = __ldg(ey + q), hh = __ldg(hr + q);
        const __nv_bfloat162* e2 = reinterpret_cast<const __nv_bfloat162*>(&e);
        const __nv_bfloat162* h2 = reinterpret_cast<const __nv_bfloat162*>(&hh);
        uint4 w;
        uint32_t* w32 = reinterpret_cast<uint32_t*>(&w);
#pragma unroll
        for (int pp = 0; pp < 4; ++pp) {
          const float2 ef = __bfloat1622float2(e2[pp]), hf = __bfloat1622float2(h2[pp]);
          dot = fmaf(hf.x, ef.x, fmaf(hf.y, ef.y, dot));
          w32[pp] = pack_bf16(arow[8 * q + 2 * pp] * scale - lab * ef.x, arow[8 * q + 2 * pp + 1] * scale - lab * ef.y);
        }
        dst[q] = w;
      }
    }
    s_dot[slot][row] = dot;
    named_bar_sync(1, 256);
    if (slot == 0 && r < capacity) {
      if (live) {
        float zy = s_dot[0][row] + s_dot[1][row];
        if (HAS_BIAS) zy += bias[y];
        const float lse2 = log2f(z) - crow_of(direct, r, n_valid);   // (the offset is 0 unless the pass runs behind the two-pass forward)
        float rl, wg2;
        ce_row_terms(direct.row, r, lse2 * kLn2, zy, rl, wg2);
        direct.lse[r] = lse2 * kLn2;
        direct.cvec[r] = -lse2 + log2f(wg2 * inv_n);
        direct.row_loss[r] = rl;
        if (direct.row.roww) direct.row.roww[r] = wg2;
      } else {
        direct.cvec[r] = -INFINITY;  // rows beyond T_v contribute nothing to the dE pass
      }
    }
  } else if (FUSED) {
    // partial (this column split) un-normalised gradient and row sums; ce_fused_finalize_kernel reduces the splits
    float* o = reinterpret_cast<float*>(out) + (size_t)split * capacity * D;
    if (r < n_valid) {
      if (slot == 0) zpart[(size_t)split * capacity + r] = s_row[row];
      float4* dst = reinterpret_cast<float4*>(o + (size_t)r * D + slot * DW);
#pragma unroll 4
      for (int c = 0; c < DW; c += 4) dst[c >> 2] = *reinterpret_cast<const float4*>(arow + c);
    }
  } else {
    __nv_bfloat16* o = reinterpret_cast<__nv_bfloat16*>(out);
    if (r < n_valid) {
      const float inv_n = loss_inv[0] * (direct.row.roww ? direct.row.roww[r] : 1.f);
      const int y = labels[r];
      const uint4* ey = reinterpret_cast<const uint4*>(table + (size_t)y * D + slot * DW);
      uint4* dst = reinterpret_cast<uint4*>(o + (size_t)r * D + slot * DW);
#pragma unroll 4
      for (int q = 0; q < DW / 8; ++q) {
        const uint4 e = ey[q];
        const __nv_bfloat162* e2 = reinterpret_cast<const __nv_bfloat162*>(&e);
        uint4 w;
        uint32_t* w32 = reinterpret_cast<uint32_t*>(&w);
#pragma unroll
        for (int pp = 0; pp < 4; ++pp) {
          const float2 ef = __bfloat1622float2(e2[pp]);
          w32[pp] = pack_bf16(arow[8 * q + 2 * pp] - inv_n * ef.x, arow[8 * q + 2 * pp + 1] - inv_n * ef.y);
        }
        dst[q] = w;
      }
    }
  }
}

// dE[y_t, :] -= Hc[t, :] / T_v   (fp32 atomics; several tokens may share a label)
__global__ void ce_label_scatter_kernel(const __nv_bfloat16* __restrict__ hc, const int32_t* __restrict__ labels,
                                        const float* __restrict__ loss_inv, const int32_t* __restrict__ n_valid_ptr,
                                        int d, float* __restrict__ dE, float* __restrict__ d_bias,
                                        const float* __restrict__ roww) {
  const int n_valid = *n_valid_ptr;
  const float inv_n0 = loss_inv[0];
  if (d_bias)
    for (int t = blockIdx.x * blockDim.x + threadIdx.x; t < n_valid; t += gridDim.x * blockDim.x)
      atomicAdd(d_bias + labels[t], -inv_n0 * (roww ? roww[t] : 1.f));
  const int per_row = d / 4;   // one 16-byte vector reduction (red.global.add.v4.f32) per 4 columns
  const long long total = (long long)n_valid * per_row;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int t = (int)(i / per_row), c = (int)(i % per_row) * 4;
    const float inv_n = inv_n0 * (roww ? roww[t] : 1.f);
    const uint2 raw = *reinterpret_cast<const uint2*>(hc + (size_t)t * d + c);
    const float2 h0 = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&raw.x));
    const float2 h1 = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&raw.y));
    atomicAdd(reinterpret_cast<float4*>(dE + (size_t)labels[t] * d + c),
              make_float4(-inv_n * h0.x, -inv_n * h0.y, -inv_n * h1.x, -inv_n * h1.y));
  }
}

// ---- safety bound of the fused (single-reference-max) path: |s_ti + b_i| <= max_t||h_t|| * max_i||e_i|| + max|b|
__global__ void ce_bound_kernel(const __nv_bfloat16* __restrict__ hc, const __nv_bfloat16* __restrict__ table,
                                const float* __restrict__ bias, const int32_t* __restrict__ n_valid_ptr, int n_items, int d,
                                unsigned int* __restrict__ bound /* [3] float bits, zeroed */) {
  // G = min(32, d/8) lanes share one row with 16-byte loads (d/8 chunks per row, d in {64,128,256,512}); every thread keeps
  // 4 rows in flight, so the 20 MB of operands stream instead of waiting on one shuffle chain per row.
  const int n_valid = *n_valid_ptr;
  const int lane = threadIdx.x & 31;
  const int cpr = d >> 3, G = cpr < 32 ? cpr : 32, per_lane = cpr / G;     // chunks per row / lanes per row / chunks per lane
  const int rows_per_warp = 32 / G;
  const int sub = lane / G, gl = lane % G;
  const long long warp_id = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const long long n_warps = (long long)gridDim.x * (blockDim.x >> 5);
  const int total = n_valid + n_items;
  float mh = 0.f, me = 0.f, mb = 0.f;
  for (long long r0 = warp_id * rows_per_warp * 4; r0 < total; r0 += n_warps * rows_per_warp * 4) {
    float ss[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const long long r = r0 + u * rows_per_warp + sub;
      if (r < total) {
        const __nv_bfloat16* row = r < n_valid ? hc + (size_t)r * d : table + (size_t)(r - n_valid) * d;
        for (int k = 0; k < per_lane; ++k) {
          const uint4 v = __ldg(reinterpret_cast<const uint4*>(row) + gl + k * G);
          const __nv_bfloat162* h2 = reinterpret_cast<const __nv_bfloat162*>(&v);
#pragma unroll
          for (int q = 0; q < 4; ++q) {
            const float2 f = __bfloat1622float2(h2[q]);
            ss[u] = fmaf(f.x, f.x, fmaf(f.y, f.y, ss[u]));
          }
        }
      }
    }
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      for (int o = G >> 1; o > 0; o >>= 1) ss[u] += __shfl_xor_sync(0xffffffffu, ss[u], o);
      const long long r = r0 + u * rows_per_warp + sub;
      if (r < total) {
        if (r < n_valid) mh = fmaxf(mh, ss[u]); else me = fmaxf(me, ss[u]);
        if (r >= n_valid && bias && gl == 0) mb = fmaxf(mb, fabsf(bias[r - n_valid]));
      }
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    mh = fmaxf(mh, __shfl_xor_sync(0xffffffffu, mh, o));
    me = fmaxf(me, __shfl_xor_sync(0xffffffffu, me, o));
    mb = fmaxf(mb, __shfl_xor_sync(0xffffffffu, mb, o));
  }
  if (lane == 0) {  // non-negative floats order like their bit patterns
    atomicMax(bound + 0, __float_as_uint(mh));
    atomicMax(bound + 1, __float_as_uint(me));
    atomicMax(bound + 2, __float_as_uint(mb));
  }
}

__global__ void ce_flag_kernel(const unsigned int* __restrict__ bound, int32_t* __restrict__ safe_flag) {
  const float b = sqrtf(__uint_as_float(bound[0]) * __uint_as_float(bound[1])) + __uint_as_float(bound[2]);
  // exp2(b * log2e) and its reciprocal must stay far inside the fp32 / bf16 exponent range
  *safe_flag = (b * kLog2e < 100.f) ? 1 : 0;
}

// reduce the column splits of the fused pass: lse, loss, exponent offsets for the dE pass, and
//   dHc[t] = sum_p dH~_p[t] / (z_t * T_v) - E[y_t] / T_v
__global__ void ce_fused_finalize_kernel(const float* __restrict__ part_dh, const float* __restrict__ zpart,
                                         const __nv_bfloat16* __restrict__ hc, const __nv_bfloat16* __restrict__ table,
                                         const int32_t* __restrict__ labels, const float* __restrict__ bias,
                                         const int32_t* __restrict__ n_valid_ptr, const int32_t* __restrict__ safe_flag,
                                         int n_splits, int z_slots, int capacity, int d, float* __restrict__ lse_out,
                                         float* __restrict__ cvec, __nv_bfloat16* __restrict__ d_hc,
                                         float* __restrict__ block_sums, unsigned int* __restrict__ ticket,
                                         float* __restrict__ loss_out, const CeRowOpts row, int use_lse_off, int run_if_safe) {
  if ((*safe_flag != 0) != (run_if_safe != 0)) return;
  const int n_valid = *n_valid_ptr;
  const float inv_n = n_valid > 0 ? 1.f / (float)n_valid : 0.f;
  const int lane = threadIdx.x & 31, wpb = blockDim.x >> 5;
  float local = 0.f;
  for (int t = blockIdx.x * wpb + (threadIdx.x >> 5); t < capacity; t += gridDim.x * wpb) {
    if (t >= n_valid) {
      if (lane == 0) cvec[t] = -INFINITY;
      continue;
    }
    float z = 0.f;
    for (int i = lane; i < n_splits * z_slots; i += 32) z += zpart[(size_t)i * capacity + t];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) z += __shfl_xor_sync(0xffffffffu, z, o);
    const int y = labels[t];
    const __nv_bfloat16* hr = hc + (size_t)t * d;
    const __nv_bfloat16* er = table + (size_t)y * d;
    // target logit first: the per-row variants (CeRowOpts) scale the gradient with a weight that may depend on it
    float dot = 0.f;
    for (int c = lane * 4; c < d; c += 128) {
      const uint2 hraw = *reinterpret_cast<const uint2*>(hr + c), eraw = *reinterpret_cast<const uint2*>(er + c);
      const float2 h0 = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&hraw.x));
      const float2 h1 = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&hraw.y));
      const float2 e0 = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&eraw.x));
      const float2 e1 = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&eraw.y));
      dot = fmaf(h0.x, e0.x, fmaf(h0.y, e0.y, fmaf(h1.x, e1.x, fmaf(h1.y, e1.y, dot))));
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) dot += __shfl_xor_sync(0xffffffffu, dot, o);
    if (bias) dot += bias[y];
    const float lse2 = log2f(z) + (use_lse_off ? lse_out[t] * kLog2e : 0.f);   // behind the two-pass forward: offsets -lse
    float rl, wg;
    ce_row_terms(row, t, lse2 * kLn2, dot, rl, wg);
    const float scale = wg * inv_n / z, lab = wg * inv_n;
    for (int c = lane * 4; c < d; c += 128) {  // 16-byte loads of the partials, all splits in flight
      const uint2 eraw = *reinterpret_cast<const uint2*>(er + c);
      const float2 e0 = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&eraw.x));
      const float2 e1 = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&eraw.y));
      float4 a = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll 8
      for (int p = 0; p < n_splits; ++p) {
        const float4 v = __ldg(reinterpret_cast<const float4*>(part_dh + ((size_t)p * capacity + t) * d + c));
        a.x += v.x; a.y += v.y; a.z += v.z; a.w += v.w;
      }
      uint2 o;
      o.x = pack_bf16(a.x * scale - lab * e0.x, a.y * scale - lab * e0.y);
      o.y = pack_bf16(a.z * scale - lab * e1.x, a.w * scale - lab * e1.y);
      *reinterpret_cast<uint2*>(d_hc + (size_t)t * d + c) = o;
    }
    if (lane == 0) {
      lse_out[t] = lse2 * kLn2;
      cvec[t] = -lse2 + log2f(wg * inv_n);
      if (row.roww) row.roww[t] = wg;
      local += rl;
    }
  }
  __shared__ float red[32];
  __shared__ bool last;
  if (lane == 0) red[threadIdx.x >> 5] = local;
  __syncthreads();
  if (threadIdx.x == 0) {
    float sum = 0.f;
    for (int i = 0; i < wpb; ++i) sum += red[i];
    block_sums[blockIdx.x] = sum;
    __threadfence();
    last = (atomicAdd(ticket, 1u) == gridDim.x - 1);
  }
  __syncthreads();
  if (last && threadIdx.x == 0) {
    __threadfence();
    float sum = 0.f;
    for (int i = 0; i < (int)gridDim.x; ++i) sum += reinterpret_cast<volatile float*>(block_sums)[i];
    loss_out[0] = sum * inv_n;
    loss_out[1] = inv_n;
  }
}

// d = 512 path: dH[c0 + r, :] = sum_s part[s][r, :] - E[y, :] / T_v   (split-K partials of softmax . E / T_v; the one-hot
// part of softmax - onehot is subtracted here), rows c0 + r < *n_valid.  One warp per row.
__global__ void ce_dh_reduce_kernel(const float* __restrict__ part, int n_splits, long long split_stride, int rows, int c0,
                                    __nv_bfloat16* __restrict__ d_hc, const __nv_bfloat16* __restrict__ table,
                                    const int32_t* __restrict__ labels, const float* __restrict__ loss_inv,
                                    const int32_t* __restrict__ n_valid_ptr, int d, const float* __restrict__ roww) {
  const int n_valid = *n_valid_ptr;
  const int lane = threadIdx.x & 31, wpb = blockDim.x >> 5;
  for (int r = blockIdx.x * wpb + (threadIdx.x >> 5); r < rows && c0 + r < n_valid; r += gridDim.x * wpb) {
    const int t = c0 + r;
    const float inv_n = loss_inv[0] * (roww ? roww[t] : 1.f);
    const __nv_bfloat16* e = table + (size_t)labels[t] * d;
    for (int c = lane * 4; c < d; c += 128) {
      float4 a = make_float4(0.f, 0.f, 0.f, 0.f);
      for (int sp = 0; sp < n_splits; ++sp) {
        const float4 v = *reinterpret_cast<const float4*>(part + (size_t)sp * split_stride + (size_t)r * d + c);
        a.x += v.x; a.y += v.y; a.z += v.z; a.w += v.w;
      }
      const uint2 ev = *reinterpret_cast<const uint2*>(e + c);
      const float2 e0 = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&ev.x));
      const float2 e1 = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&ev.y));
      uint2 o;
      o.x = pack_bf16(a.x - inv_n * e0.x, a.y - inv_n * e0.y);
      o.y = pack_bf16(a.z - inv_n * e1.x, a.w - inv_n * e1.y);
      *reinterpret_cast<uint2*>(d_hc + (size_t)t * d + c) = o;
    }
  }
}

// BCE: reduce the column splits.  zrow: softplus row sums, element (t, p) at zrow[p * zsp + t * zst]; loss_out (if given)
// = {mean_t (sum_p zrow - x_t,y), 1 / T_v}, deterministic (fixed partition, the last block adds the block sums in order).
// part_dh (if given): the fused pass's split partials of sum_i sigmoid_ti E_i -> d_hc[t] = (sum_p part_dh[p][t] - E[y]) / T_v.
__global__ void bce_finalize_kernel(const float* __restrict__ zrow, long long zsp, int zst, const float* __restrict__ part_dh,
                                    int n_splits, const __nv_bfloat16* __restrict__ hc, const __nv_bfloat16* __restrict__ table,
                                    const int32_t* __restrict__ labels, const float* __restrict__ bias,
                                    const int32_t* __restrict__ n_valid_ptr, int capacity, int d,
                                    __nv_bfloat16* __restrict__ d_hc, float* __restrict__ block_sums,
                                    unsigned int* __restrict__ ticket, float* __restrict__ loss_out) {
  const int n_valid = *n_valid_ptr;
  const float inv_n = n_valid > 0 ? 1.f / (float)n_valid : 0.f;
  const int lane = threadIdx.x & 31, wpb = blockDim.x >> 5;
  float local = 0.f;
  for (int t = blockIdx.x * wpb + (threadIdx.x >> 5); t < n_valid; t += gridDim.x * wpb) {
    const int y = labels[t];
    const __nv_bfloat16* er = table + (size_t)y * d;
    if (loss_out) {
      float z = 0.f;
      for (int p = lane; p < n_splits; p += 32) z += zrow[(size_t)p * zsp + (size_t)t * zst];
      const __nv_bfloat16* hr = hc + (size_t)t * d;
      float dot = 0.f;
      for (int c = lane * 2; c < d; c += 64) {
        const float2 a = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(hr + c));
        const float2 b = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(er + c));
        dot = fmaf(a.x, b.x, fmaf(a.y, b.y, dot));
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        z += __shfl_xor_sync(0xffffffffu, z, o);
        dot += __shfl_xor_sync(0xffffffffu, dot, o);
      }
      if (bias) dot += bias[y];
      if (lane == 0) local += z - dot;
    }
    if (d_hc) {
      for (int c = lane * 4; c < d; c += 128) {
        const uint2 eraw = *reinterpret_cast<const uint2*>(er + c);
        const float2 e0 = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&eraw.x));
        const float2 e1 = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&eraw.y));
        float4 a = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll 8
        for (int p = 0; p < n_splits; ++p) {
          const float4 v = __ldg(reinterpret_cast<const float4*>(part_dh + ((size_t)p * capacity + t) * d + c));
          a.x += v.x; a.y += v.y; a.z += v.z; a.w += v.w;
        }
        uint2 o;
        o.x = pack_bf16((a.x - e0.x) * inv_n, (a.y - e0.y) * inv_n);
        o.y = pack_bf16((a.z - e1.x) * inv_n, (a.w - e1.y) * inv_n);
        *reinterpret_cast<uint2*>(d_hc + (size_t)t * d + c) = o;
      }
    }
  }
  if (!loss_out) return;
  __shared__ float red[32];
  __shared__ bool last;
  if (lane == 0) red[threadIdx.x >> 5] = local;
  __syncthreads();
  if (threadIdx.x == 0) {
    float s = 0.f;
    for (int i = 0; i < wpb; ++i) s += red[i];
    block_sums[blockIdx.x] = s;
    __threadfence();
    last = (atomicAdd(ticket, 1u) == gridDim.x - 1);
  }
  __syncthreads();
  if (last && threadIdx.x == 0) {
    __threadfence();
    float s = 0.f;
    for (int i = 0; i < (int)gridDim.x; ++i) s += reinterpret_cast<volatile float*>(block_sums)[i];
    loss_out[0] = s * inv_n;
    loss_out[1] = inv_n;
  }
}

// BCE at d = 512: per-row exponent offsets of rp_gemm's sigmoid epilogue (act 4): log2(1 / T_v) on the valid rows, -inf past
// them, so G = sigmoid / T_v there and exactly 0 on stale rows
__global__ void bce_row_offset_kernel(const int32_t* __restrict__ n_valid_ptr, int capacity, float* __restrict__ off) {
  const int n_valid = *n_valid_ptr;
  const float l = n_valid > 0 ? -log2f((float)n_valid) : 0.f;
  for (int t = blockIdx.x * blockDim.x + threadIdx.x; t < capacity; t += gridDim.x * blockDim.x) off[t] = t < n_valid ? l : -INFINITY;
}

// Biased head at d = 512: d_bias[i] = (first chunk) / += (later chunks) sum_t G[t, i] over the chunk's rows below *n_valid
// (G already carries 1 / T_v; the one-hot part follows in ce_label_scatter_kernel).  Rows at or past *n_valid are not read:
// the G GEMM skips whole row tiles there, which keep an earlier chunk's values.  A block owns 256 columns, a lane 8 of them
// (one 16-byte load per row), the 8 warps take every 8th row and their sums are added in warp order: deterministic, no
// atomics.  Columns >= n_items are never written (a lane's last vector may load a few; their sums are dropped).
__global__ void __launch_bounds__(256) ce_bias_colsum_kernel(const __nv_bfloat16* __restrict__ G, long long ldg, int rows, int c0,
                                                             const int32_t* __restrict__ n_valid_ptr, int n_items,
                                                             float* __restrict__ d_bias, int accumulate) {
  __shared__ float part[8][256];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int col0 = blockIdx.x * 256 + lane * 8;
  int n = *n_valid_ptr - c0;
  n = n < 0 ? 0 : (n > rows ? rows : n);
  float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  if (col0 < n_items) {   // col0 + 8 <= round_up(n_items, 8) <= ldg: the load stays inside the row
    const __nv_bfloat16* g = G + col0;
    int t = warp;
    for (; t + 24 < n; t += 32) {   // four rows in flight per lane
      uint4 v[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) v[u] = __ldg(reinterpret_cast<const uint4*>(g + (size_t)(t + 8 * u) * ldg));
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const __nv_bfloat162* h2 = reinterpret_cast<const __nv_bfloat162*>(&v[u]);
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const float2 f = __bfloat1622float2(h2[q]);
          acc[2 * q] += f.x;
          acc[2 * q + 1] += f.y;
        }
      }
    }
    for (; t < n; t += 8) {
      const uint4 v = __ldg(reinterpret_cast<const uint4*>(g + (size_t)t * ldg));
      const __nv_bfloat162* h2 = reinterpret_cast<const __nv_bfloat162*>(&v);
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const float2 f = __bfloat1622float2(h2[q]);
        acc[2 * q] += f.x;
        acc[2 * q + 1] += f.y;
      }
    }
  }
#pragma unroll
  for (int q = 0; q < 8; ++q) part[warp][lane * 8 + q] = acc[q];
  __syncthreads();
  const int c = blockIdx.x * 256 + threadIdx.x;
  if (c < n_items) {
    float s = 0.f;
#pragma unroll
    for (int w = 0; w < 8; ++w) s += part[w][threadIdx.x];
    d_bias[c] = accumulate ? d_bias[c] + s : s;
  }
}

// d = 512 backward (wide_bwd): the materialised G is bf16 [chunk rows, wide_ldg]; chunk rows: as many as fit the G budget
// (RP_CE_WIDE_G_BYTES, default 8 GiB), multiple of 128.
static long long wide_ldg(int n_items) { return ((long long)n_items + 63) / 64 * 64; }
static int wide_chunk_rows(int cap, int n_items) {
  const char* env = getenv("RP_CE_WIDE_G_BYTES");  // read per call: the workspace query and the launch must agree
  const long long budget = env ? atoll(env) : (8ll << 30);
  long long rows = budget / (wide_ldg(n_items) * 2) / 128 * 128;
  const long long cap128 = ((long long)cap + 127) / 128 * 128;
  if (rows < 128) rows = 128;
  if (rows > cap128) rows = cap128;
  return (int)rows;
}

static int pick_splits(int n_row_tiles, int n_col_tiles, int max_splits = 8) {
  const int sms = sm_count();
  int best = 1;
  double best_eff = 0.0;
  for (int p = 1; p <= max_splits && p <= n_col_tiles; ++p) {
    const long long ctas = (long long)n_row_tiles * p;
    const double eff = (double)ctas / (double)(((ctas + sms - 1) / sms) * sms);
    if (eff > best_eff + 0.02) {
      best_eff = eff;
      best = p;
    }
  }
  return best;
}

}  // namespace rp

using namespace rp;

// Workspace of the CE and BCE heads (cap = capacity; ops.ce_head_fused_taken reads `flag` at this layout):
//   part        float2 [cap * kMaxSplitsFwd * 2]   (max, sum) per row and column split of the two-pass forward
//   block_sums  float [1024]                        per-block sums of the deterministic loss reductions
//   ticket, bound[3], flag, pad -> 64 B            zeroed by every CE forward
//   zpart       float [kMaxSplits * cap]            row sums / row losses per column split (BCE's un-fused forward: its
//                                                   softplus row sums)
//   roww        float [round_up(cap, 4)]            gradient weight per row (BCE at d = 512: the sigmoid's exponent offsets)
//   part_dh     float [kMaxSplits * cap * d]        partial dH per column split, d <= 256 only
// then 256 B of slack; at d = 512, from the next 1 KiB boundary, the G chunk and the split-K partials of dH (ce_ws_bytes).
struct CeWs {
  float2* part; float* block_sums; unsigned int* ticket; unsigned int* bound; int32_t* flag; float* zpart; float* roww; float* part_dh;
};
static const int kMaxSplits = 8;       // fused forward + dH: partial gradients per split
static const int kMaxSplitsFwd = 32;   // two-pass forward: only (max, sum) pairs per split
static const int kWideSplitK = 16;     // d = 512 backward: split-K partials of the dH GEMM

static size_t ce_ws_base_bytes(int cap, int d) {
  return (size_t)cap * kMaxSplitsFwd * 2 * sizeof(float2) + 4096 + 64 + (size_t)kMaxSplits * cap * 4 +
         (size_t)(cap + 3) / 4 * 16 + (d <= 256 ? (size_t)kMaxSplits * cap * d * 4 : 0) + 256;
}
static size_t ce_ws_bytes(int cap, int n_items, int d) {
  size_t b = (ce_ws_base_bytes(cap, d) + 1023) / 1024 * 1024;
  if (d > 256) {
    const size_t rows = (size_t)wide_chunk_rows(cap, n_items);
    b += rows * wide_ldg(n_items) * 2;              // G chunk (bf16)
    b += (size_t)kWideSplitK * rows * d * 4;        // split-K partials of dH (fp32)
  }
  return b;
}
static CeWs ce_ws(void* workspace, int cap) {
  uint8_t* w = reinterpret_cast<uint8_t*>(workspace);
  CeWs r;
  r.part = reinterpret_cast<float2*>(w);
  w += (size_t)cap * kMaxSplitsFwd * 2 * sizeof(float2);
  r.block_sums = reinterpret_cast<float*>(w);
  w += 4096;
  r.ticket = reinterpret_cast<unsigned int*>(w);
  r.bound = r.ticket + 1;
  r.flag = reinterpret_cast<int32_t*>(r.ticket + 4);
  w += 64;
  r.zpart = reinterpret_cast<float*>(w);
  w += (size_t)kMaxSplits * cap * 4;
  r.roww = reinterpret_cast<float*>(w);   // gradient weight per row (CeRowOpts), written by every forward finalisation
  w += (size_t)(cap + 3) / 4 * 16;
  r.part_dh = reinterpret_cast<float*>(w);
  return r;
}

RP_API size_t rp_ce_head_workspace(int capacity_tokens, int n_items, int d) {
  if (capacity_tokens <= 0 || n_items <= 0 || d <= 0) return 0;
  return ce_ws_bytes(capacity_tokens, n_items, d);
}

// Argument checks of the five head entry points, in the order their error codes take precedence.  `args_ok`: the entry
// point's own required arguments are valid (an entry point that always reads the workspace counts it here, so a null one is
// RP_EINVAL there); `needs_ws`: this call reads the workspace, which must then be present and large enough.
static int check_head_args(const void* hc, const void* table, const int32_t* labels, const int32_t* n_valid,
                           const float* loss_out, bool args_ok, int capacity, int n_items, int d, bool needs_ws,
                           const void* workspace, size_t workspace_bytes) {
  if (!hc || !table || !labels || !n_valid || !loss_out || !args_ok) return RP_EINVAL;
  if (capacity <= 0 || n_items <= 0) return RP_ESHAPE;
  if (d != 64 && d != 128 && d != 256 && d != 512) return RP_ESHAPE;
  if (needs_ws && (!workspace || workspace_bytes < ce_ws_bytes(capacity, n_items, d))) return RP_EWORKSPACE;
  return RP_OK;
}

// row tiles the column splits are balanced over: those the host expects to hold valid targets, else all of them
static int hint_row_tiles(int n_valid_hint, int capacity) {
  const int rows = (n_valid_hint > 0 && n_valid_hint <= capacity) ? n_valid_hint : capacity;
  return (rows + kT - 1) / kT;
}

// grid of the finalisation kernels (one warp per row, 8 per CTA)
static int finalize_blocks(int capacity) {
  const int blocks = (capacity + 7) / 8;
  return blocks > 1024 ? 1024 : blocks;
}

template <int KCH, int NSTAGE, bool BCE>
static int launch_ce_fwd(const CUtensorMap& tmA, const CUtensorMap& tmB, const int32_t* n_valid, int n_items,
                         int n_splits, int n_tok_tiles, const float* bias, float2* part, const int32_t* skip,
                         cudaStream_t stream) {
  const int smem = (KCH + NSTAGE) * kChunk + 1024;
  auto kern = ce_fwd_kernel<KCH, NSTAGE, BCE>;
  RP_CUDA_CHECK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  kern<<<n_tok_tiles * n_splits, kThreads, smem, stream>>>(tmA, tmB, n_valid, n_items, n_splits, bias, part, skip);
  RP_LAUNCH_CHECK();
  return RP_OK;
}

// CE's two-pass forward and BCE's un-fused forward: (max, sum) or softplus row sums per (row, column split)
template <bool BCE>
static int dispatch_ce_fwd(int d, const CUtensorMap& tmA, const CUtensorMap& tmB, const int32_t* n_valid, int n_items,
                           int n_splits, int n_tok_tiles, const float* bias, float2* part, const int32_t* skip,
                           cudaStream_t stream) {
  switch (d) {
    case 64: return launch_ce_fwd<1, 8, BCE>(tmA, tmB, n_valid, n_items, n_splits, n_tok_tiles, bias, part, skip, stream);
    case 128: return launch_ce_fwd<2, 8, BCE>(tmA, tmB, n_valid, n_items, n_splits, n_tok_tiles, bias, part, skip, stream);
    case 256: return launch_ce_fwd<4, 8, BCE>(tmA, tmB, n_valid, n_items, n_splits, n_tok_tiles, bias, part, skip, stream);
    default: return launch_ce_fwd<8, 5, BCE>(tmA, tmB, n_valid, n_items, n_splits, n_tok_tiles, bias, part, skip, stream);
  }
}

template <int KCH, int NSTAGE, int TN, int MODE>
static int launch_ce_bwd(const CUtensorMap& tmA, const void* b_mat, int b_rows, const void* a_rows, const float* cvec,
                         const int32_t* labels,
                         const void* table, const float* loss_inv, const int32_t* n_valid, int n_items, const float* bias,
                         float* d_bias, void* out, int grid, const int32_t* safe_flag, int run_if_safe, int n_splits,
                         int capacity, float* zpart, cudaStream_t stream, const CeDirect& direct) {
  // row tile + a ring of NSTAGE column tiles; the fp32 accumulator stage reuses the ring at the end.  MODE 1 adds the ring's
  // slots of exponent offsets, which the bulk copy fills from a 16-byte aligned cvec
  const int ring = NSTAGE * KCH * TN * 128, stage = 128 * (KCH * 64 + 4) * 4;
  const int offsets = MODE == 1 ? NSTAGE * TN * 4 : 0;
  if (MODE == 1 && (reinterpret_cast<uintptr_t>(cvec) & 15) != 0) return RP_EALIGN;
  const int smem = KCH * kChunk + (ring > stage ? ring : stage) + offsets + 1024;
  CUtensorMap tmB;   // column-side matrix, one [TN rows x 64 columns] box per chunk
  {
    const int rc = make_tmap_bf16(&tmB, b_mat, b_rows, KCH * 64, KCH * 64, TN);
    if (rc != RP_OK) return rc;
  }
  // the biased head (BERT4Rec) is a separate instantiation: its per-column adds / row sums cost an instruction per logit
  auto kern = bias ? ce_bwd_kernel<KCH, NSTAGE, TN, MODE, true> : ce_bwd_kernel<KCH, NSTAGE, TN, MODE, false>;
  RP_CUDA_CHECK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  kern<<<grid, kThreads, smem, stream>>>(tmA, tmB, reinterpret_cast<const __nv_bfloat16*>(a_rows), cvec, labels,
                                         reinterpret_cast<const __nv_bfloat16*>(table), loss_inv,
                                         n_valid, n_items, bias, d_bias, out, safe_flag, run_if_safe, n_splits, capacity, zpart, direct);
  RP_LAUNCH_CHECK();
  return RP_OK;
}

template <int MODE>
static int dispatch_ce_bwd(int d, const CUtensorMap& tmA, const void* b_mat, int b_rows, const void* a_rows, const float* cvec,
                           const int32_t* labels,
                           const void* table, const float* loss_inv, const int32_t* n_valid, int n_items, const float* bias,
                           float* d_bias, void* out, int grid, const int32_t* safe_flag, int run_if_safe, int n_splits,
                           int capacity, float* zpart, cudaStream_t stream, const CeDirect& direct = CeDirect{}) {
  switch (d) {
    case 64:
      return launch_ce_bwd<1, 8, 128, MODE>(tmA, b_mat, b_rows, a_rows, cvec, labels, table, loss_inv, n_valid, n_items, bias, d_bias, out, grid,
                                       safe_flag, run_if_safe, n_splits, capacity, zpart, stream, direct);
    case 128:
      return launch_ce_bwd<2, 4, 128, MODE>(tmA, b_mat, b_rows, a_rows, cvec, labels, table, loss_inv, n_valid, n_items, bias, d_bias, out, grid,
                                       safe_flag, run_if_safe, n_splits, capacity, zpart, stream, direct);
    case 256:
      return launch_ce_bwd<4, 4, 64, MODE>(tmA, b_mat, b_rows, a_rows, cvec, labels, table, loss_inv, n_valid, n_items, bias, d_bias, out, grid,
                                       safe_flag, run_if_safe, n_splits, capacity, zpart, stream, direct);
    default:
      return RP_ESHAPE;
  }
}

// The BCE token pass (MODE 3) keeps softplus's product and max terms beside the sigmoid: with 128-column tiles at d = 128 it
// spills, so there it walks 64-column tiles with a ring twice as deep.  The dE pass (MODE 4) uses dispatch_ce_bwd's table.
static int dispatch_bce_rows(int d, const CUtensorMap& tmA, const void* table, int n_items, const void* hc, const int32_t* labels,
                             const int32_t* n_valid, const float* bias, float* part_dh, int grid, int n_splits, int capacity,
                             float* zpart, cudaStream_t stream, const CeDirect& direct) {
  switch (d) {
    case 64:
      return launch_ce_bwd<1, 8, 128, 3>(tmA, table, n_items, hc, nullptr, labels, table, nullptr, n_valid, n_items, bias, nullptr,
                                         part_dh, grid, nullptr, 0, n_splits, capacity, zpart, stream, direct);
    case 128:
      return launch_ce_bwd<2, 8, 64, 3>(tmA, table, n_items, hc, nullptr, labels, table, nullptr, n_valid, n_items, bias, nullptr,
                                        part_dh, grid, nullptr, 0, n_splits, capacity, zpart, stream, direct);
    case 256:
      return launch_ce_bwd<4, 4, 64, 3>(tmA, table, n_items, hc, nullptr, labels, table, nullptr, n_valid, n_items, bias, nullptr,
                                        part_dh, grid, nullptr, 0, n_splits, capacity, zpart, stream, direct);
    default:
      return RP_ESHAPE;
  }
}

// The fused CE pass (MODE 2: row sums of exp(s) and the un-normalised dH in one sweep) and its completion.  With one column
// split every CTA sees the whole catalog: lse / cvec / dH / row losses come straight out of the pass and
// ce_loss_reduce_kernel sums the losses.  With several, ce_fused_finalize_kernel reduces the split partials.
// behind == false: runs when the device-side bound held, exponent offset 0.  behind == true: the pass behind the two-pass
// forward, runs when the bound failed, exponent offset -lse[t] (G = softmax, z ~ 1, whatever |logit| is).
static int ce_fused_pass(bool behind, const CUtensorMap& tmA, const void* hc, const void* table, const float* bias,
                         const int32_t* labels, const int32_t* n_valid, int capacity, int n_items, int d, float* loss_out,
                         float* lse, float* cvec, void* d_hc, int n_valid_hint, const CeRowOpts& row, const CeWs& ws,
                         cudaStream_t stream) {
  const int run_if_safe = behind ? 0 : 1, use_lse_off = behind ? 1 : 0;
  const int hint_tiles = hint_row_tiles(n_valid_hint, capacity), n_item_tiles = (n_items + kT - 1) / kT;
  const int P = pick_splits(hint_tiles, n_item_tiles);
  CeDirect direct{nullptr, lse, nullptr, nullptr, row, use_lse_off};
  if (P == 1) {
    direct.d_hc = reinterpret_cast<__nv_bfloat16*>(d_hc);
    direct.cvec = cvec;
    direct.row_loss = ws.zpart;  // the row-sum partials are not needed in this mode: reuse their buffer
  }
  const int rc = dispatch_ce_bwd<2>(d, tmA, table, n_items, hc, cvec, labels, table, loss_out + 1, n_valid, n_items, bias, nullptr,
                                    ws.part_dh, (capacity + kT - 1) / kT * P, ws.flag, run_if_safe, P, capacity, ws.zpart, stream,
                                    direct);
  if (rc != RP_OK) return rc;
  if (P == 1)
    ce_loss_reduce_kernel<<<1, 1024, 0, stream>>>(ws.zpart, n_valid, ws.flag, loss_out, run_if_safe);
  else
    ce_fused_finalize_kernel<<<finalize_blocks(capacity), 256, 0, stream>>>(
        ws.part_dh, ws.zpart, reinterpret_cast<const __nv_bfloat16*>(hc), reinterpret_cast<const __nv_bfloat16*>(table), labels,
        bias, n_valid, ws.flag, P, 1, capacity, d, lse, cvec, reinterpret_cast<__nv_bfloat16*>(d_hc), ws.block_sums, ws.ticket,
        loss_out, row, use_lse_off, run_if_safe);
  RP_LAUNCH_CHECK();
  return RP_OK;
}

// d = 512 backward of both heads.  The [128 x 512] fp32 gradient accumulator does not fit the registers of the two
// warpgroups, so per token chunk (wide_chunk_rows) three plain GEMMs run on the materialised G (bf16):
//   G = act(hc . E^T + b) with per-row exponent offsets `off`:  act 3 (CE): exp2(x log2e + cvec[t]), the weighted softmax
//       / T_v;  act 4 (BCE): sigmoid / T_v, 0 on rows past T_v (bce_row_offset_kernel)
//   d_bias (+)= colsum G (iff bias);  dH = G . E - roww[t] E[y_t] / T_v (roww null = 1);  dE (+)= G^T . hc
// The one-hot part of dE and d_bias is the caller's ce_label_scatter_kernel.
static int wide_bwd(int act, const float* off, const float* roww, const void* hc, const void* table, const float* bias,
                    const int32_t* labels, const int32_t* n_valid, int capacity, int n_items, int d, const float* loss_inv,
                    void* d_hc, float* d_table, float* d_bias, int n_valid_hint, void* workspace, cudaStream_t stream) {
  const long long ldg = wide_ldg(n_items);
  const int chunk = wide_chunk_rows(capacity, n_items);
  uint8_t* G = reinterpret_cast<uint8_t*>(workspace) + (ce_ws_base_bytes(capacity, d) + 1023) / 1024 * 1024;
  float* part = reinterpret_cast<float*>(G + (size_t)chunk * ldg * 2);
  const long long part_stride = (long long)chunk * d;
  const int hint = (n_valid_hint > 0 && n_valid_hint < capacity) ? n_valid_hint : capacity;
  int rc;
  for (int c0 = 0, it = 0; c0 < capacity; c0 += chunk, ++it) {
    const int rows = (capacity - c0 < chunk) ? capacity - c0 : chunk;
    // G [rows, n_items] = act((hc[c0:c0+rows] . E^T + b), off[c0:c0+rows])   (the epilogue adds the bias before the act)
    rp_gemm_desc g = rp_gemm_default();
    g.A = reinterpret_cast<const __nv_bfloat16*>(hc) + (size_t)c0 * d; g.a_rows = rows; g.a_cols = d; g.lda = d; g.a_mn = 0;
    g.B = table; g.b_rows = n_items; g.b_cols = d; g.ldb = d; g.b_mn = 0;
    g.M = rows; g.N = n_items; g.K = d;
    g.C = G; g.ldc = ldg; g.out_mode = 0; g.act = act; g.row_exp2_offset = off + c0; g.bias = bias;
    g.m_limit_dev = n_valid; g.m_limit_base = c0;
    if ((rc = rp_gemm(&g, stream)) != RP_OK) return rc;
    if (bias) {
      ce_bias_colsum_kernel<<<(n_items + 255) / 256, 256, 0, stream>>>(reinterpret_cast<const __nv_bfloat16*>(G), ldg, rows, c0,
                                                                       n_valid, n_items, d_bias, it != 0);
      RP_LAUNCH_CHECK();
    }
    // dH[c0:c0+rows] = G . E - label term   (A = G K-major over the items, B = E read MN-major).  Few row tiles against a
    // contraction over the whole catalog: split-K partials (fp32, deterministic), reduced together with the label term
    int live = hint - c0;
    live = live < 128 ? 128 : (live > rows ? rows : live);
    int split = (2 * sm_count()) / (((live + 127) / 128) * (d / 128));
    split = split < 1 ? 1 : (split > kWideSplitK ? kWideSplitK : split);
    g = rp_gemm_default();
    g.split_k = split;
    g.A = G; g.a_rows = rows; g.a_cols = n_items; g.lda = ldg; g.a_mn = 0;
    g.B = table; g.b_rows = n_items; g.b_cols = d; g.ldb = d; g.b_mn = 1;
    g.M = rows; g.N = d; g.K = n_items;
    g.C = part; g.ldc = d; g.out_mode = 3; g.c_split_stride = part_stride;
    g.m_limit_dev = n_valid; g.m_limit_base = c0;
    if ((rc = rp_gemm(&g, stream)) != RP_OK) return rc;
    ce_dh_reduce_kernel<<<sm_count() * 4, 256, 0, stream>>>(part, split, part_stride, rows, c0,
                                                             reinterpret_cast<__nv_bfloat16*>(d_hc),
                                                             reinterpret_cast<const __nv_bfloat16*>(table), labels, loss_inv,
                                                             n_valid, d, roww);
    RP_LAUNCH_CHECK();
    // dE (+)= G^T . hc[c0:c0+rows]      (A = G read MN-major, contraction over the chunk's valid tokens)
    g = rp_gemm_default();
    g.A = G; g.a_rows = rows; g.a_cols = n_items; g.lda = ldg; g.a_mn = 1;
    g.B = reinterpret_cast<const __nv_bfloat16*>(hc) + (size_t)c0 * d; g.b_rows = rows; g.b_cols = d; g.ldb = d; g.b_mn = 1;
    g.M = n_items; g.N = d; g.K = rows;
    g.C = d_table; g.ldc = d; g.out_mode = it == 0 ? 2 : 4;
    g.k_limit_dev = n_valid; g.k_limit_base = c0;
    if ((rc = rp_gemm(&g, stream)) != RP_OK) return rc;
  }
  return RP_OK;
}

// Forward of the CE head.  hc bf16 [capacity, d] (rows >= *n_valid ignored), table bf16 [n_items, d], labels int32
// [capacity], n_valid int32 [1] (device).  Outputs: loss_out fp32 [2] = {mean CE, 1/T_v}; lse fp32 [capacity]; cvec fp32
// (exponent offsets consumed by rp_ce_head_bwd).
// d_hc != NULL (training, d <= 256) enables the FUSED path: one pass computes the row sums of exp(s) against a fixed
// reference maximum of 0 together with the un-normalised gradient sum_i exp(s_i) E_i, so the separate log-sum-exp pass
// disappears and d_hc is already final after this call.  A device-side Cauchy-Schwarz bound on |s| guards the trick; if
// it fails the two-pass kernels run instead (both variants are launched, the losing one exits at once), so the call
// stays CUDA-graph capturable.  n_valid_hint (host estimate of *n_valid, 0 = unknown) only tunes the load balance.
RP_API int rp_ce_head_fwd_w(const void* hc, const void* table, const float* bias, const int32_t* labels,
                            const int32_t* n_valid, int capacity, int n_items, int d, float* loss_out, float* lse, float* cvec,
                            void* d_hc, int n_valid_hint, const float* row_weight, int loss_kind, float log_eps, float clamp,
                            void* workspace, size_t workspace_bytes, void* stream_);
RP_API int rp_ce_head_fwd(const void* hc, const void* table, const float* bias, const int32_t* labels,
                          const int32_t* n_valid, int capacity, int n_items, int d, float* loss_out, float* lse, float* cvec,
                          void* d_hc, int n_valid_hint, void* workspace, size_t workspace_bytes, void* stream_) {
  return rp_ce_head_fwd_w(hc, table, bias, labels, n_valid, capacity, n_items, d, loss_out, lse, cvec, d_hc, n_valid_hint, nullptr,
                          0, 0.f, 0.f, workspace, workspace_bytes, stream_);
}

// Per-row variants of the head (CeRowOpts): row_weight fp32 [capacity] (>= 0, compacted order of the valid targets, NULL = 1),
// loss_kind 0 = CE, 1 = LogInCE with (log_eps, clamp).  The backward must be rp_ce_head_bwd with the SAME workspace (the
// per-row gradient weights live there); everything else as rp_ce_head_fwd.
RP_API int rp_ce_head_fwd_w(const void* hc, const void* table, const float* bias, const int32_t* labels,
                            const int32_t* n_valid, int capacity, int n_items, int d, float* loss_out, float* lse, float* cvec,
                            void* d_hc, int n_valid_hint, const float* row_weight, int loss_kind, float log_eps, float clamp,
                            void* workspace, size_t workspace_bytes, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  int rc = check_head_args(hc, table, labels, n_valid, loss_out, (loss_kind == 0 || loss_kind == 1) && lse && cvec && workspace,
                           capacity, n_items, d, true, workspace, workspace_bytes);
  if (rc != RP_OK) return rc;
  const bool fused = d_hc != nullptr && d <= 256;
  const int n_tok_tiles = (capacity + kT - 1) / kT, n_item_tiles = (n_items + kT - 1) / kT;
  const CeWs ws = ce_ws(workspace, capacity);
  const CeRowOpts row{row_weight, ws.roww, loss_kind, log_eps, clamp};
  CUtensorMap tmA, tmB;
  if ((rc = make_tmap_bf16(&tmA, hc, capacity, d, d, 128)) != RP_OK) return rc;
  if ((rc = make_tmap_bf16(&tmB, table, n_items, d, d, 128)) != RP_OK) return rc;
  RP_CUDA_CHECK(cudaMemsetAsync(ws.ticket, 0, 64, stream));  // ticket, bound[3], flag
  if (fused) {
    ce_bound_kernel<<<sm_count() * 8, 256, 0, stream>>>(reinterpret_cast<const __nv_bfloat16*>(hc),
                                                        reinterpret_cast<const __nv_bfloat16*>(table), bias, n_valid, n_items, d,
                                                        ws.bound);
    RP_LAUNCH_CHECK();
    ce_flag_kernel<<<1, 1, 0, stream>>>(ws.bound, ws.flag);
    RP_LAUNCH_CHECK();
    if ((rc = ce_fused_pass(false, tmA, hc, table, bias, labels, n_valid, capacity, n_items, d, loss_out, lse, cvec, d_hc,
                            n_valid_hint, row, ws, stream)) != RP_OK)
      return rc;
  }
  int P2 = pick_splits(hint_row_tiles(n_valid_hint, capacity), n_item_tiles, kMaxSplitsFwd);
  if (fused) {  // two-pass fallback behind the fused pass: it only runs when the bound failed; launching (and retiring) tens of
                // thousands of CTAs that exit at once is not free, so keep it at about two waves
    const int cap = (2 * sm_count() + n_tok_tiles - 1) / n_tok_tiles;
    if (P2 > cap) P2 = cap;
  }
  const int32_t* skip = fused ? ws.flag : nullptr;
  if ((rc = dispatch_ce_fwd<false>(d, tmA, tmB, n_valid, n_items, P2, n_tok_tiles, bias, ws.part, skip, stream)) != RP_OK) return rc;
  ce_finalize_kernel<<<finalize_blocks(capacity), 256, 0, stream>>>(ws.part, reinterpret_cast<const __nv_bfloat16*>(hc),
                                                                    reinterpret_cast<const __nv_bfloat16*>(table), labels, bias,
                                                                    n_valid, P2, capacity, d, lse, cvec, ws.block_sums,
                                                                    ws.ticket, loss_out, skip, row);
  RP_LAUNCH_CHECK();
  if (fused) {
    // The bound failed (these launches exit at once otherwise): the two-pass forward above has produced lse; the gradient
    // dH comes from the SAME fused kernel, now with the exponent offset -lse[t] per row (G = softmax, z ~ 1) - with its column
    // splits and all SMs busy, where the row-tile-per-CTA MODE 0 pass ran 32 CTAs at BERT4Rec's ~4000 masked positions
    // (2.2 ms of a 4.3 ms step at config 3, whose un-normalised outputs outgrow the bound within a few hundred steps).
    RP_CUDA_CHECK(cudaMemsetAsync(ws.ticket, 0, 4, stream));   // the deterministic loss reduction's ticket was used above
    if ((rc = ce_fused_pass(true, tmA, hc, table, bias, labels, n_valid, capacity, n_items, d, loss_out, lse, cvec, d_hc,
                            n_valid_hint, row, ws, stream)) != RP_OK)
      return rc;
  }
  return RP_OK;
}

// Backward of rp_ce_head_fwd for d(loss) = 1:
//   d_hc   bf16 [capacity, d]  (rows < *n_valid) - already written by the forward when it ran fused (`fused` != 0 and the
//          device-side bound held); otherwise computed here from the stored lse.  d = 512: chunked materialised-G path
//          (three GEMMs per token chunk, see wide_bwd), workspace required
//   d_table fp32 [n_items, d]  OVERWRITTEN with softmax^T . hc / T_v, then the one-hot part is atomically subtracted
//   d_bias  fp32 [n_items] (iff bias)  OVERWRITTEN likewise.        d in {64,128,256,512}.
RP_API int rp_ce_head_bwd(const void* hc, const void* table, const float* bias, const int32_t* labels,
                          const int32_t* n_valid, int capacity, int n_items, int d, const float* loss_out /* from fwd */,
                          const float* cvec /* from fwd */, void* d_hc, float* d_table, float* d_bias, int fused,
                          int n_valid_hint, void* workspace, size_t workspace_bytes, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  int rc = check_head_args(hc, table, labels, n_valid, loss_out, cvec && d_hc && d_table && (bias == nullptr) == (d_bias == nullptr),
                           capacity, n_items, d, fused || d == 512, workspace, workspace_bytes);
  if (rc != RP_OK) return rc;
  // gradient weight per row, written by the forward (all ones for the plain CE head); without a workspace: plain head
  const float* roww = (workspace && workspace_bytes >= ce_ws_bytes(capacity, n_items, d)) ? ce_ws(workspace, capacity).roww : nullptr;
  const float* loss_inv = loss_out + 1;
  if (d == 512) {
    if ((rc = wide_bwd(3, cvec, roww, hc, table, bias, labels, n_valid, capacity, n_items, d, loss_inv, d_hc, d_table, d_bias,
                       n_valid_hint, workspace, stream)) != RP_OK)
      return rc;
  } else {
    CUtensorMap tmH, tmE;
    if ((rc = make_tmap_bf16(&tmH, hc, capacity, d, d, 128)) != RP_OK) return rc;
    if ((rc = make_tmap_bf16(&tmE, table, n_items, d, d, 128)) != RP_OK) return rc;
    const int n_tok_tiles = (capacity + kT - 1) / kT, n_item_tiles = (n_items + kT - 1) / kT;
    // token-major pass: only when the forward did not already produce d_hc (a fused forward always does: from the fused pass
    // itself, or - bound failed - from its second launch behind the two-pass forward)
    if (!fused && (rc = dispatch_ce_bwd<0>(d, tmH, table, n_items, hc, cvec, labels, table, loss_inv, n_valid, n_items, bias, nullptr,
                                           d_hc, n_tok_tiles, nullptr, 0, 1, capacity, nullptr, stream,
                                           CeDirect{nullptr, nullptr, nullptr, nullptr,
                                                    CeRowOpts{nullptr, const_cast<float*>(roww), 0, 0.f, 0.f}})) != RP_OK)
      return rc;
    rc = dispatch_ce_bwd<1>(d, tmE, hc, capacity, table, cvec, labels, table, loss_inv, n_valid, n_items, bias, d_bias, d_table,
                            n_item_tiles, nullptr, 0, 1, capacity, nullptr, stream);
    if (rc != RP_OK) return rc;
  }
  ce_label_scatter_kernel<<<sm_count() * 4, 256, 0, stream>>>(reinterpret_cast<const __nv_bfloat16*>(hc), labels, loss_inv,
                                                               n_valid, d, d_table, d_bias, roww);
  RP_LAUNCH_CHECK();
  return RP_OK;
}

// ---------------------------------------------------------------------------------------------------------------- BCE head
// the token-major BCE pass (MODE 3) over the catalog: d_hc, and the row losses when `loss_out` is given.  Without column
// splits both come out of the pass itself; otherwise bce_finalize_kernel reduces the split partials.
static int bce_rows_pass(const void* hc, const void* table, const float* bias, const int32_t* labels, const int32_t* n_valid,
                         int capacity, int n_items, int d, float* loss_out, void* d_hc, int n_valid_hint, const CeWs& ws,
                         cudaStream_t stream) {
  const int n_tok_tiles = (capacity + kT - 1) / kT, n_item_tiles = (n_items + kT - 1) / kT;
  CUtensorMap tmA;
  int rc;
  if ((rc = make_tmap_bf16(&tmA, hc, capacity, d, d, 128)) != RP_OK) return rc;
  const int P = pick_splits(hint_row_tiles(n_valid_hint, capacity), n_item_tiles);
  CeDirect direct{};
  if (P == 1) {
    direct.d_hc = reinterpret_cast<__nv_bfloat16*>(d_hc);
    direct.row_loss = ws.zpart;
  }
  rc = dispatch_bce_rows(d, tmA, table, n_items, hc, labels, n_valid, bias, ws.part_dh, n_tok_tiles * P, P, capacity, ws.zpart,
                         stream, direct);
  if (rc != RP_OK) return rc;
  if (P == 1) {
    if (loss_out) {
      ce_loss_reduce_kernel<<<1, 1024, 0, stream>>>(ws.zpart, n_valid, nullptr, loss_out, 0);
      RP_LAUNCH_CHECK();
    }
    return RP_OK;
  }
  bce_finalize_kernel<<<finalize_blocks(capacity), 256, 0, stream>>>(ws.zpart, capacity, 1, ws.part_dh, P,
                                                                     reinterpret_cast<const __nv_bfloat16*>(hc),
                                                                     reinterpret_cast<const __nv_bfloat16*>(table), labels, bias,
                                                                     n_valid, capacity, d, reinterpret_cast<__nv_bfloat16*>(d_hc),
                                                                     ws.block_sums, ws.ticket, loss_out);
  RP_LAUNCH_CHECK();
  return RP_OK;
}

// Forward of the full-catalog BCE head: loss_out fp32 [2] = {sum_t [sum_i softplus(x_ti) - x_t,y_t] / T_v, 1 / T_v}.  Buffers
// as rp_ce_head_fwd (workspace: rp_ce_head_workspace).  d_hc != NULL (d <= 256): one fused pass also writes the final d_hc.
RP_API int rp_bce_head_fwd(const void* hc, const void* table, const float* bias, const int32_t* labels, const int32_t* n_valid,
                           int capacity, int n_items, int d, float* loss_out, void* d_hc, int n_valid_hint, void* workspace,
                           size_t workspace_bytes, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  int rc = check_head_args(hc, table, labels, n_valid, loss_out, workspace != nullptr, capacity, n_items, d, true, workspace,
                           workspace_bytes);
  if (rc != RP_OK) return rc;
  const CeWs ws = ce_ws(workspace, capacity);
  RP_CUDA_CHECK(cudaMemsetAsync(ws.ticket, 0, 4, stream));
  if (d_hc != nullptr && d <= 256) return bce_rows_pass(hc, table, bias, labels, n_valid, capacity, n_items, d, loss_out, d_hc,
                                                        n_valid_hint, ws, stream);
  // un-fused: softplus row sums per (row, split), then the loss
  const int n_tok_tiles = (capacity + kT - 1) / kT, n_item_tiles = (n_items + kT - 1) / kT;
  const int P = pick_splits(hint_row_tiles(n_valid_hint, capacity), n_item_tiles);   // <= kMaxSplits: the partials live in ws.zpart
  CUtensorMap tmA, tmB;
  if ((rc = make_tmap_bf16(&tmA, hc, capacity, d, d, 128)) != RP_OK) return rc;
  if ((rc = make_tmap_bf16(&tmB, table, n_items, d, d, 128)) != RP_OK) return rc;
  rc = dispatch_ce_fwd<true>(d, tmA, tmB, n_valid, n_items, P, n_tok_tiles, bias, reinterpret_cast<float2*>(ws.zpart), nullptr, stream);
  if (rc != RP_OK) return rc;
  bce_finalize_kernel<<<finalize_blocks(capacity), 256, 0, stream>>>(ws.zpart, 1, P, nullptr, P,
                                                                     reinterpret_cast<const __nv_bfloat16*>(hc),
                                                                     reinterpret_cast<const __nv_bfloat16*>(table), labels, bias,
                                                                     n_valid, capacity, d, nullptr, ws.block_sums, ws.ticket,
                                                                     loss_out);
  RP_LAUNCH_CHECK();
  return RP_OK;
}

// Backward of rp_bce_head_fwd for d(loss) = 1 (same workspace): d_hc bf16 [capacity, d] (rows < *n_valid; already final when
// the forward ran fused, `fused` != 0), d_table fp32 [n_items, d] and d_bias fp32 [n_items] (iff bias) OVERWRITTEN with
// (sigmoid - onehot)^T . hc / T_v and its column sums.  d = 512: sigmoid / T_v of a token chunk is materialised in bf16
// (rp_gemm act 4, the bias inside the sigmoid) and three GEMMs per chunk produce dH and dE, as rp_ce_head_bwd does; with a
// bias, ce_bias_colsum_kernel sums the chunk's columns into d_bias.
RP_API int rp_bce_head_bwd(const void* hc, const void* table, const float* bias, const int32_t* labels, const int32_t* n_valid,
                           int capacity, int n_items, int d, const float* loss_out, void* d_hc, float* d_table, float* d_bias,
                           int fused, int n_valid_hint, void* workspace, size_t workspace_bytes, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  int rc = check_head_args(hc, table, labels, n_valid, loss_out, workspace != nullptr, capacity, n_items, d, true, workspace,
                           workspace_bytes);
  if (rc != RP_OK) return rc;
  if (!d_hc || !d_table || (bias == nullptr) != (d_bias == nullptr)) return RP_EINVAL;
  const CeWs ws = ce_ws(workspace, capacity);
  const float* loss_inv = loss_out + 1;
  if (d == 512) {
    float* off = ws.roww;   // per-row exponent offsets of the sigmoid epilogue (the CE row weights are not used here)
    bce_row_offset_kernel<<<(capacity + 255) / 256 < 1024 ? (capacity + 255) / 256 : 1024, 256, 0, stream>>>(n_valid, capacity, off);
    RP_LAUNCH_CHECK();
    if ((rc = wide_bwd(4, off, nullptr, hc, table, bias, labels, n_valid, capacity, n_items, d, loss_inv, d_hc, d_table, d_bias,
                       n_valid_hint, workspace, stream)) != RP_OK)
      return rc;
  } else {
    if (!fused && (rc = bce_rows_pass(hc, table, bias, labels, n_valid, capacity, n_items, d, nullptr, d_hc, n_valid_hint, ws,
                                      stream)) != RP_OK)
      return rc;
    CUtensorMap tmE;
    if ((rc = make_tmap_bf16(&tmE, table, n_items, d, d, 128)) != RP_OK) return rc;
    rc = dispatch_ce_bwd<4>(d, tmE, hc, capacity, table, nullptr, labels, table, loss_inv, n_valid, n_items, bias, d_bias, d_table,
                            (n_items + kT - 1) / kT, nullptr, 0, 1, capacity, nullptr, stream);
    if (rc != RP_OK) return rc;
  }
  ce_label_scatter_kernel<<<sm_count() * 4, 256, 0, stream>>>(reinterpret_cast<const __nv_bfloat16*>(hc), labels, loss_inv,
                                                               n_valid, d, d_table, d_bias, nullptr);
  RP_LAUNCH_CHECK();
  return RP_OK;
}
