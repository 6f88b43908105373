// rp_sampled_head.cu - sampled-softmax / sampled-BCE training heads (SURVEY.md §8 a9, f.2): logits only for the positive item
// and N sampled negatives per target token, loss and gradients.  Replaces
//   SampledLossBase.get_sampled_logits + mask_negative_logits      replay/nn/loss/base.py:40-154,157-196
//   CESampled.forward                                             replay/nn/loss/ce.py:199-249
//   BCESampled.forward                                            replay/nn/loss/bce.py:154-218
//   LogInCESampled.forward                                        replay/nn/loss/login_ce.py:240-375
//   CESampledWeighted.forward                                     replay/nn/loss/ce.py:252-330
//   legacy _compute_loss_ce_sampled / _compute_loss_bce_sampled    replay/models/nn/sequential/sasrec/lightning.py:310-376
// (the negatives are an INPUT, as in the reference's new path).  Multi-positive rows (num_positives P > 1, new-path CE / BCE /
// weighted CE only): row t carries P raw labels [t*P, t*P+P) and a slot mask; every masked-in slot is a (position, positive)
// pair scored against the row's negatives, and the mean runs over the pairs.
//
// Layout: hc bf16 [capacity, d] = hidden rows of the valid targets (compacted, rows >= *n_valid ignored); labels int32
// [capacity]; negatives int64 in one of three shapes: 0 = [N] shared by the whole batch, 1 = [B*L, N] per position,
// 2 = [B, N] per sequence (rows addressed through valid_idx = flat b*L+l index of every compacted row).
// Shared negatives run on the tensor cores (z = hc . E_neg^T, dH = dz . E_neg, dE_neg = dz^T . hc through rp_gemm, then N
// rows are scattered into the table gradient); per-position / per-sequence negatives are gather-dot kernels (HBM/L2
// bound: each (token, negative) pair reads one table row) whose backward scatters with fp32 atomics.
#include "rp_host.h"
#include "rp_gemm_desc.h"
#include "rp_sm90.cuh"

namespace rp {

enum { kCESampled = 0, kBCESampled = 1, kLegacyCE = 2, kLegacyBCE = 3, kLogInCESampled = 4, kCESampledWeighted = 5 };

struct SampledArgs {
  const __nv_bfloat16* hc;
  const __nv_bfloat16* table;
  const int32_t* labels;
  const int32_t* valid_idx;
  const int64_t* negatives;
  const int32_t* n_valid;
  const float* row_weight;  // [capacity] sample weight of each compacted row (kCESampledWeighted only)
  int capacity, n_items, d, N, neg_mode, L, kind, ignore_index, vocab_size;
  float log_eps, clamp;
  float* loss_out;
  // workspace
  float* zpos;            // [capacity]           positive logits -> d(loss)/d(z_pos)
  float* zneg;            // [capacity, ldz]      negative logits -> d(loss)/d(z_neg)
  __nv_bfloat16* dz16;    // [capacity128, ldn]   bf16 copy of d(loss)/d(z_neg) for the GEMMs (shared negatives)
  __nv_bfloat16* e_neg;   // [N, d]               gathered negative rows (shared negatives)
  float* de_neg;          // [N, d]
  float* block_sums;      // [1024]
  unsigned int* ticket;
  int ldz, ldn;
};

// multi-positive rows (P > 1): labels / row_weight are [capacity, P], slot_mask [capacity, P], *n_pairs = masked-in slots.
// A kernel parameter of its own, after SampledArgs, so that the single-positive kernels keep their parameter layout.
struct MultiPos {
  int P;
  const uint8_t* slot_mask;
  const int32_t* n_pairs;
};

__device__ __forceinline__ long long neg_row(const SampledArgs& a, int t) {
  if (a.neg_mode == 0) return 0;
  const int flat = a.valid_idx[t];
  return a.neg_mode == 1 ? (long long)flat : (long long)(flat / a.L);
}
__device__ __forceinline__ int clamp_item(long long id, int n_items) {
  return (id >= 0 && id < n_items) ? (int)id : 0;  // out-of-range ids (padding / ignore_index) are masked by the loss
}

// shared negatives: E_neg[j, :] = table[neg[j], :]
__global__ void sampled_gather_neg_kernel(const SampledArgs a) {
  const int lane = threadIdx.x & 31, wpb = blockDim.x >> 5;
  for (int j = blockIdx.x * wpb + (threadIdx.x >> 5); j < a.N; j += gridDim.x * wpb) {
    const uint4* src = reinterpret_cast<const uint4*>(a.table + (size_t)clamp_item(a.negatives[j], a.n_items) * a.d);
    uint4* dst = reinterpret_cast<uint4*>(a.e_neg + (size_t)j * a.d);
    for (int c = lane; c < a.d / 8; c += 32) dst[c] = src[c];
  }
}

template <int D>
__device__ __forceinline__ float warp_dot(const float (&h)[D / 32], const __nv_bfloat16* __restrict__ row, int lane) {
  // lane owns elements [lane*2 + 64*k, +2)
  float acc = 0.f;
#pragma unroll
  for (int k = 0; k < D / 64; ++k) {
    const float2 e = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(row + k * 64 + lane * 2));
    acc = fmaf(h[2 * k], e.x, fmaf(h[2 * k + 1], e.y, acc));
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  return acc;
}

// one warp per valid token: z_pos = h . E[y] (MP: one per masked-in slot); (modes 1, 2) z_neg[j] = h . E[neg(t, j)]
template <int D, bool MP>
__global__ void sampled_logits_kernel(const SampledArgs a, const MultiPos mp) {
  const int n_valid = *a.n_valid;
  const int lane = threadIdx.x & 31, wpb = blockDim.x >> 5;
  for (int t = blockIdx.x * wpb + (threadIdx.x >> 5); t < n_valid; t += gridDim.x * wpb) {
    float h[D / 32];
#pragma unroll
    for (int k = 0; k < D / 64; ++k) {
      const float2 v = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(a.hc + (size_t)t * D + k * 64 + lane * 2));
      h[2 * k] = v.x;
      h[2 * k + 1] = v.y;
    }
    if constexpr (MP) {
      for (int k = 0; k < mp.P; ++k) {
        const size_t s = (size_t)t * mp.P + k;
        const float zp = mp.slot_mask[s] ? warp_dot<D>(h, a.table + (size_t)a.labels[s] * D, lane) : 0.f;
        if (lane == 0) a.zpos[s] = zp;
      }
    } else {
      const float zp = warp_dot<D>(h, a.table + (size_t)a.labels[t] * D, lane);
      if (lane == 0) a.zpos[t] = zp;
    }
    if (a.neg_mode != 0) {
      const int64_t* nr = a.negatives + neg_row(a, t) * a.N;
      for (int j = 0; j < a.N; ++j) {
        const float z = warp_dot<D>(h, a.table + (size_t)clamp_item(nr[j], a.n_items) * D, lane);
        if (lane == 0) a.zneg[(size_t)t * a.ldz + j] = z;
      }
    }
  }
}

// loss_out = {sum of the warps' `local` * inv_n, inv_n}: deterministic (block partials in a fixed order, the last block adds)
__device__ __forceinline__ void sampled_mean(const SampledArgs& a, float local, float inv_n) {
  const int lane = threadIdx.x & 31, wpb = blockDim.x >> 5;
  __shared__ float red[32];
  __shared__ bool last;
  if (lane == 0) red[threadIdx.x >> 5] = local;
  __syncthreads();
  if (threadIdx.x == 0) {
    float s = 0.f;
    for (int i = 0; i < wpb; ++i) s += red[i];
    a.block_sums[blockIdx.x] = s;
    __threadfence();
    last = (atomicAdd(a.ticket, 1u) == gridDim.x - 1);
  }
  __syncthreads();
  if (last && threadIdx.x == 0) {
    __threadfence();
    float s = 0.f;
    for (int i = 0; i < (int)gridDim.x; ++i) s += reinterpret_cast<volatile float*>(a.block_sums)[i];
    a.loss_out[0] = s * inv_n;
    a.loss_out[1] = inv_n;
    *a.ticket = 0u;
  }
}

// one warp per token: masks, loss, d(loss)/d(logits) in place; deterministic mean (block partials, last block adds)
__global__ void sampled_loss_kernel(const SampledArgs a) {
  const int n_valid = *a.n_valid;
  const float inv_n = n_valid > 0 ? __frcp_rn((float)n_valid) : 0.f;   // loss_out[1] = 1/T_v rounded once (fast-math safe)
  const int lane = threadIdx.x & 31, wpb = blockDim.x >> 5;
  // shared negatives: the GEMMs read dz16 in whole 128-row M tiles (dH) and 64-row K chunks (dE_neg), past the capacity when
  // it is not a multiple of 64 - zero every row they can reach (dz16 has round_up(capacity, 128) rows), so that a stale
  // workspace cannot reach dE_neg as 0 x NaN
  const int t_end = a.neg_mode == 0 ? ((n_valid + 127) / 128) * 128 : n_valid;
  const int n_neg_drawn = min(a.N, a.vocab_size);   // legacy CE: the reference corrects by min(N, vocab_size) - #reject
  const bool ce = a.kind == kCESampled || a.kind == kLegacyCE || a.kind == kLogInCESampled || a.kind == kCESampledWeighted;
  const bool masked = a.kind == kCESampled || a.kind == kBCESampled || a.kind == kLogInCESampled || a.kind == kCESampledWeighted;
  float local = 0.f;
  for (int t = blockIdx.x * wpb + (threadIdx.x >> 5); t < t_end; t += gridDim.x * wpb) {
    float* zr = a.zneg + (size_t)t * a.ldz;
    __nv_bfloat16* gr = a.dz16 ? a.dz16 + (size_t)t * a.ldn : nullptr;
    if (t >= n_valid) {
      if (gr)
        for (int j = lane; j < a.ldn; j += 32) gr[j] = __float2bfloat16(0.f);
      continue;
    }
    const int y = a.labels[t];
    const int64_t* nr = a.negatives + neg_row(a, t) * a.N;
    const float zp = a.zpos[t];
    // pass 1: masks / corrections, row statistics
    int n_reject = 0;
    if (a.kind == kLegacyCE) {
      for (int j = lane; j < a.N; j += 32) n_reject += (nr[j] == (int64_t)y) ? 1 : 0;
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) n_reject += __shfl_xor_sync(0xffffffffu, n_reject, o);
    }
    float mx = ce ? zp : 0.f;
    for (int j = lane; j < a.N; j += 32) {
      const int64_t nj = nr[j];
      float z = zr[j];
      if (masked && (nj == (int64_t)y || (a.ignore_index >= 0 && nj == (int64_t)a.ignore_index))) z = -1e9f;
      if (a.kind == kLegacyCE) z = z + logf((float)(a.vocab_size - 1)) - (nj == (int64_t)y ? 1e6f : 0.f) - logf((float)(n_neg_drawn - n_reject));
      zr[j] = z;
      mx = fmaxf(mx, z);
    }
    if (ce) {
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
      float s = 0.f;
      for (int j = lane; j < a.N; j += 32) s += __expf(zr[j] - mx);
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
      const float ep = __expf(zp - mx);
      const float s_neg = s;
      s += ep;
      const float lse = mx + logf(s);
      const float inv_s = 1.f / s;
      // every CE kind's gradient is wg * (softmax - onehot) / T_v with a per-row factor wg (1 for CE / legacy CE)
      float row_loss = lse - zp, wg = 1.f, dpos = ep * inv_s - 1.f;
      if (a.kind == kCESampledWeighted) {
        // (row CE * w_t).mean() over the valid targets (replay/nn/loss/ce.py:252-330)
        wg = a.row_weight[t];
        row_loss *= wg;
      } else if (a.kind == kLogInCESampled) {
        // -clamp(log(p + eps), -c, c) of the positive's softmax share p: d/dz = p / (p + eps) x the CE gradient inside the
        // clamp, 0 outside (same edge rule as the catalog LogInCE); 1 - p from the negatives' sum, not from p
        const float p = ep * inv_s;
        const float lg = logf(p + a.log_eps);
        row_loss = -fminf(fmaxf(lg, -a.clamp), a.clamp);
        wg = (lg > -a.clamp && lg < a.clamp) ? p / (p + a.log_eps) : 0.f;
        dpos = -s_neg * inv_s;
      }
      const float gs = wg * inv_n;
      for (int j = lane; j < a.N; j += 32) {
        const float g = __expf(zr[j] - mx) * inv_s * gs;
        zr[j] = g;
        if (gr) gr[j] = __float2bfloat16(g);
      }
      if (lane == 0) {
        a.zpos[t] = dpos * gs;
        local += row_loss;
      }
    } else {
      // BCE: -( clamp(log(sigmoid(z_pos) + eps)) + sum_j clamp(log(1 - sigmoid(z_j) + eps)) ), fp32 as the reference
      float acc = 0.f;
      for (int j = lane; j < a.N; j += 32) {
        const float z = zr[j];
        const float sg = 1.f / (1.f + __expf(-z));
        const float arg = (1.f - sg) + a.log_eps;
        const float lg = logf(arg);
        const bool in = lg > -a.clamp && lg < a.clamp;
        acc += fminf(fmaxf(lg, -a.clamp), a.clamp);
        const float g = in ? (sg * (1.f - sg) / arg) * inv_n : 0.f;   // d(-log(1 - s + eps))/dz = s(1-s)/(1-s+eps)
        zr[j] = g;
        if (gr) gr[j] = __float2bfloat16(g);
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
      if (lane == 0) {
        const float sg = 1.f / (1.f + __expf(-zp));
        const float arg = sg + a.log_eps;
        const float lg = logf(arg);
        const bool in = lg > -a.clamp && lg < a.clamp;
        a.zpos[t] = in ? -(sg * (1.f - sg) / arg) * inv_n : 0.f;
        local += -(fminf(fmaxf(lg, -a.clamp), a.clamp) + acc);
      }
    }
    if (gr)
      for (int j = a.N + lane; j < a.ldn; j += 32) gr[j] = __float2bfloat16(0.f);
  }
  sampled_mean(a, local, inv_n);
}

// multi-positive rows (kCESampled / kBCESampled / kCESampledWeighted), one warp per row, lane k < P owns slot k.  A negative
// is masked when it equals any of the row's P raw labels (masked-out slots included: replay/nn/loss/base.py:139-154 hands
// every pair the whole label row) or ignore_index, so the masked row is shared by the row's pairs.  CE pair k:
// lse([z_k, z_neg]) - z_k; BCE pair k: its positive term plus the whole negative row.  Both times w_k (weighted CE), mean
// over the *n_pairs pairs.  d(loss)/d(z_neg[j]) sums the pairs: exp(z_j - m) sum_k w_k exp(m - m_k) / S_k (CE, m = max of
// the negatives, m_k = max(m, z_k)), n_pairs(row) x the BCE term.
__global__ void sampled_loss_multi_kernel(const SampledArgs a, const MultiPos mp) {
  const int n_valid = *a.n_valid, n_pairs = *mp.n_pairs;
  const float inv_n = n_pairs > 0 ? __frcp_rn((float)n_pairs) : 0.f;
  const int lane = threadIdx.x & 31, wpb = blockDim.x >> 5;
  const int t_end = a.neg_mode == 0 ? ((n_valid + 127) / 128) * 128 : n_valid;   // see sampled_loss_kernel
  const bool ce = a.kind != kBCESampled;
  float local = 0.f;
  for (int t = blockIdx.x * wpb + (threadIdx.x >> 5); t < t_end; t += gridDim.x * wpb) {
    float* zr = a.zneg + (size_t)t * a.ldz;
    __nv_bfloat16* gr = a.dz16 ? a.dz16 + (size_t)t * a.ldn : nullptr;
    if (t >= n_valid) {
      if (gr)
        for (int j = lane; j < a.ldn; j += 32) gr[j] = __float2bfloat16(0.f);
      continue;
    }
    const int64_t* nr = a.negatives + neg_row(a, t) * a.N;
    const int32_t* yr = a.labels + (size_t)t * mp.P;
    const size_t sk = (size_t)t * mp.P + lane;
    const bool live = lane < mp.P && mp.slot_mask[sk] != 0;
    const float zk = live ? a.zpos[sk] : 0.f;
    const float wk = live ? (a.row_weight ? a.row_weight[sk] : 1.f) : 0.f;
    const int n_row = __popc(__ballot_sync(0xffffffffu, live));
    float mx = -3.0e38f;   // max of the masked negatives (each CE pair adds its own positive below)
    for (int j = lane; j < a.N; j += 32) {
      const int64_t nj = nr[j];
      bool hit = a.ignore_index >= 0 && nj == (int64_t)a.ignore_index;
      for (int k = 0; k < mp.P; ++k) hit |= nj == (int64_t)yr[k];
      const float z = hit ? -1e9f : zr[j];
      zr[j] = z;
      mx = fmaxf(mx, z);
    }
    if (ce) {
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
      float s = 0.f;
      for (int j = lane; j < a.N; j += 32) s += __expf(zr[j] - mx);
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
      // pair k: its own log-sum-exp over [z_k | negatives] with m_k = max(mx, z_k), so that another positive of the row far
      // above z_k cannot flush the sum to 0; S_k >= 1
      float c = 0.f, row_loss = 0.f;
      if (live) {
        const float mk = fmaxf(mx, zk);
        const float en = __expf(mx - mk), ep = __expf(zk - mk);
        const float S = s * en + ep;
        const float inv_s = 1.f / S;
        row_loss = wk * (mk + logf(S) - zk);
        c = wk * en * inv_s;
        a.zpos[sk] = wk * (ep * inv_s - 1.f) * inv_n;
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        c += __shfl_xor_sync(0xffffffffu, c, o);
        row_loss += __shfl_xor_sync(0xffffffffu, row_loss, o);
      }
      const float gs = c * inv_n;
      for (int j = lane; j < a.N; j += 32) {
        const float g = __expf(zr[j] - mx) * gs;
        zr[j] = g;
        if (gr) gr[j] = __float2bfloat16(g);
      }
      if (lane == 0) local += row_loss;
    } else {
      float acc = 0.f;
      const float gs = (float)n_row * inv_n;
      for (int j = lane; j < a.N; j += 32) {
        const float z = zr[j];
        const float sg = 1.f / (1.f + __expf(-z));
        const float arg = (1.f - sg) + a.log_eps;
        const float lg = logf(arg);
        const bool in = lg > -a.clamp && lg < a.clamp;
        acc += fminf(fmaxf(lg, -a.clamp), a.clamp);
        const float g = in ? (sg * (1.f - sg) / arg) * gs : 0.f;
        zr[j] = g;
        if (gr) gr[j] = __float2bfloat16(g);
      }
      float pos = 0.f;
      if (live) {
        const float sg = 1.f / (1.f + __expf(-zk));
        const float arg = sg + a.log_eps;
        const float lg = logf(arg);
        const bool in = lg > -a.clamp && lg < a.clamp;
        a.zpos[sk] = in ? -(sg * (1.f - sg) / arg) * inv_n : 0.f;
        pos = fminf(fmaxf(lg, -a.clamp), a.clamp);
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        acc += __shfl_xor_sync(0xffffffffu, acc, o);
        pos += __shfl_xor_sync(0xffffffffu, pos, o);
      }
      if (lane == 0) local += -(pos + (float)n_row * acc);
    }
    if (gr)
      for (int j = a.N + lane; j < a.ldn; j += 32) gr[j] = __float2bfloat16(0.f);
  }
  sampled_mean(a, local, inv_n);
}

// backward, one warp per token: dH[t] (+)= dz_pos E[y] (+ sum_j dz_j E[neg_j] for per-token negatives);
// dE[y] += dz_pos h;  dE[neg_j] += dz_j h  (fp32 atomics).  MP: every masked-in slot's positive, summed in slot order
template <int D, bool MP>
__global__ void sampled_bwd_kernel(const SampledArgs a, __nv_bfloat16* __restrict__ d_hc, float* __restrict__ d_table,
                                   int add_to_dhc, const MultiPos mp) {
  const int n_valid = *a.n_valid;
  const int lane = threadIdx.x & 31, wpb = blockDim.x >> 5;
  for (int t = blockIdx.x * wpb + (threadIdx.x >> 5); t < n_valid; t += gridDim.x * wpb) {
    float h[D / 32], acc[D / 32];
#pragma unroll
    for (int k = 0; k < D / 64; ++k) {
      const float2 v = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(a.hc + (size_t)t * D + k * 64 + lane * 2));
      h[2 * k] = v.x;
      h[2 * k + 1] = v.y;
      float2 o = make_float2(0.f, 0.f);
      if (add_to_dhc) o = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(d_hc + (size_t)t * D + k * 64 + lane * 2));
      acc[2 * k] = o.x;
      acc[2 * k + 1] = o.y;
    }
    auto one = [&](int item, float g) {
      const __nv_bfloat16* er = a.table + (size_t)item * D;
      float* dr = d_table + (size_t)item * D;
#pragma unroll
      for (int k = 0; k < D / 64; ++k) {
        const float2 e = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(er + k * 64 + lane * 2));
        acc[2 * k] = fmaf(g, e.x, acc[2 * k]);
        acc[2 * k + 1] = fmaf(g, e.y, acc[2 * k + 1]);
        atomicAdd(dr + k * 64 + lane * 2, g * h[2 * k]);
        atomicAdd(dr + k * 64 + lane * 2 + 1, g * h[2 * k + 1]);
      }
    };
    if constexpr (MP) {
      for (int k = 0; k < mp.P; ++k) {
        const size_t s = (size_t)t * mp.P + k;
        if (mp.slot_mask[s]) one(a.labels[s], a.zpos[s]);
      }
    } else {
      one(a.labels[t], a.zpos[t]);
    }
    if (a.neg_mode != 0) {
      const int64_t* nr = a.negatives + neg_row(a, t) * a.N;
      const float* gz = a.zneg + (size_t)t * a.ldz;
      for (int j = 0; j < a.N; ++j) {
        const float g = gz[j];
        if (g != 0.f) one(clamp_item(nr[j], a.n_items), g);
      }
    }
#pragma unroll
    for (int k = 0; k < D / 64; ++k)
      *reinterpret_cast<uint32_t*>(d_hc + (size_t)t * D + k * 64 + lane * 2) = pack_bf16(acc[2 * k], acc[2 * k + 1]);
  }
}

// shared negatives: d_table[neg[j], :] += dE_neg[j, :]
__global__ void sampled_scatter_neg_kernel(const SampledArgs a, float* __restrict__ d_table) {
  const int lane = threadIdx.x & 31, wpb = blockDim.x >> 5;
  for (int j = blockIdx.x * wpb + (threadIdx.x >> 5); j < a.N; j += gridDim.x * wpb) {
    const int64_t id = a.negatives[j];
    if (id < 0 || id >= a.n_items) continue;
    for (int c = lane; c < a.d; c += 32) atomicAdd(d_table + (size_t)id * a.d + c, a.de_neg[(size_t)j * a.d + c]);
  }
}

// ------------------------------------------------------------------------------------------------------------------
// Full-catalog BCE over a positive SET per row (replay/nn/loss/bce.py:51-95, num_positives P > 1): the target of live row t
// is 1 at every distinct id in [0, n_items) among its P raw slots (scatter_(value=1); the slot mask is not read inside a
// live row).  rp_bce_head_* score labels[t] as the row's positive; the other ids of the set ("extra" positives) add
// -x_t,y / T_v to the loss and -1/T_v x E[y] to dH[t], -1/T_v x h_t to dE[y].
// ------------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ bool bce_extra(const int32_t* __restrict__ yr, int k, int y0, int n_items) {
  const int y = yr[k];
  if (y < 0 || y >= n_items || y == y0) return false;
  for (int j = 0; j < k; ++j)
    if (yr[j] == y) return false;
  return true;
}

// one warp per live row: row_sum[t] = sum of the extra positives' logits
template <int D>
__global__ void bce_extra_fwd_kernel(const __nv_bfloat16* __restrict__ hc, const __nv_bfloat16* __restrict__ table,
                                     const int32_t* __restrict__ labels, const int32_t* __restrict__ labels_p,
                                     const int32_t* __restrict__ n_valid_dev, int P, int n_items, float* __restrict__ row_sum) {
  const int n_valid = *n_valid_dev;
  const int lane = threadIdx.x & 31, wpb = blockDim.x >> 5;
  for (int t = blockIdx.x * wpb + (threadIdx.x >> 5); t < n_valid; t += gridDim.x * wpb) {
    float h[D / 32];
#pragma unroll
    for (int k = 0; k < D / 64; ++k) {
      const float2 v = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(hc + (size_t)t * D + k * 64 + lane * 2));
      h[2 * k] = v.x;
      h[2 * k + 1] = v.y;
    }
    const int32_t* yr = labels_p + (size_t)t * P;
    float s = 0.f;
    for (int k = 0; k < P; ++k)
      if (bce_extra(yr, k, labels[t], n_items)) s += warp_dot<D>(h, table + (size_t)yr[k] * D, lane);
    if (lane == 0) row_sum[t] = s;
  }
}

// one block: loss_out[0] -= (sum_t row_sum[t]) x loss_out[1], the rows summed in a fixed order
__global__ void __launch_bounds__(1024) bce_extra_loss_kernel(const float* __restrict__ row_sum,
                                                              const int32_t* __restrict__ n_valid_dev, float* loss_out) {
  __shared__ float red[32];
  const int n_valid = *n_valid_dev;
  float s = 0.f;
  for (int t = threadIdx.x; t < n_valid; t += blockDim.x) s += row_sum[t];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    float tot = 0.f;
    for (int w = 0; w < (int)(blockDim.x >> 5); ++w) tot += red[w];
    if (n_valid > 0) loss_out[0] -= tot * loss_out[1];
  }
}

// one warp per live row: dH[t] -= inv_n sum_extra E[y] (in registers, slot order), dE[y] -= inv_n h_t (fp32 atomics)
template <int D>
__global__ void bce_extra_bwd_kernel(const __nv_bfloat16* __restrict__ hc, const __nv_bfloat16* __restrict__ table,
                                     const int32_t* __restrict__ labels, const int32_t* __restrict__ labels_p,
                                     const int32_t* __restrict__ n_valid_dev, int P, int n_items,
                                     const float* __restrict__ loss_out, __nv_bfloat16* __restrict__ d_hc,
                                     float* __restrict__ d_table) {
  const int n_valid = *n_valid_dev;
  const float g = -loss_out[1];
  const int lane = threadIdx.x & 31, wpb = blockDim.x >> 5;
  for (int t = blockIdx.x * wpb + (threadIdx.x >> 5); t < n_valid; t += gridDim.x * wpb) {
    const int32_t* yr = labels_p + (size_t)t * P;
    float h[D / 32], acc[D / 32];
#pragma unroll
    for (int k = 0; k < D / 64; ++k) {
      const float2 v = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(hc + (size_t)t * D + k * 64 + lane * 2));
      h[2 * k] = v.x;
      h[2 * k + 1] = v.y;
      acc[2 * k] = 0.f;
      acc[2 * k + 1] = 0.f;
    }
    bool any = false;
    for (int kk = 0; kk < P; ++kk) {
      if (!bce_extra(yr, kk, labels[t], n_items)) continue;
      any = true;
      const __nv_bfloat16* er = table + (size_t)yr[kk] * D;
      float* dr = d_table + (size_t)yr[kk] * D;
#pragma unroll
      for (int k = 0; k < D / 64; ++k) {
        const float2 e = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(er + k * 64 + lane * 2));
        acc[2 * k] = fmaf(g, e.x, acc[2 * k]);
        acc[2 * k + 1] = fmaf(g, e.y, acc[2 * k + 1]);
        atomicAdd(dr + k * 64 + lane * 2, g * h[2 * k]);
        atomicAdd(dr + k * 64 + lane * 2 + 1, g * h[2 * k + 1]);
      }
    }
    if (!any) continue;
#pragma unroll
    for (int k = 0; k < D / 64; ++k) {
      uint32_t* p = reinterpret_cast<uint32_t*>(d_hc + (size_t)t * D + k * 64 + lane * 2);
      const float2 o = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(p));
      *p = pack_bf16(o.x + acc[2 * k], o.y + acc[2 * k + 1]);
    }
  }
}

}  // namespace rp

using namespace rp;

struct rp_sampled_desc {
  const void* hc; const void* table; const int32_t* labels; const int32_t* valid_idx; const int64_t* negatives;
  const int32_t* n_valid;
  int capacity, n_items, d, n_neg, neg_mode, seq_len, kind, ignore_index, vocab_size;
  float log_eps, clamp;
  float* loss_out;
  void* workspace; size_t workspace_bytes;
  const float* row_weight;
  int num_positives; const uint8_t* slot_mask; const int32_t* n_pairs;
};

static size_t ru(size_t x, size_t m) { return (x + m - 1) / m * m; }

static size_t sampled_layout(const rp_sampled_desc* s, SampledArgs* a) {
  const size_t cap128 = ru((size_t)s->capacity, 128);
  const int ldz = (int)ru((size_t)s->n_neg, 4), ldn = (int)ru((size_t)s->n_neg, 8);
  size_t off = 0;
  auto take = [&](size_t bytes) { const size_t o = off; off = ru(off + bytes, 256); return o; };
  const size_t P = s->num_positives > 1 ? (size_t)s->num_positives : 1;
  const size_t o_zpos = take(cap128 * P * 4), o_zneg = take(cap128 * ldz * 4);
  const size_t o_dz16 = s->neg_mode == 0 ? take(cap128 * ldn * 2) : 0;
  const size_t o_eneg = s->neg_mode == 0 ? take((size_t)s->n_neg * s->d * 2) : 0;
  const size_t o_deneg = s->neg_mode == 0 ? take((size_t)s->n_neg * s->d * 4) : 0;
  const size_t o_bs = take(1024 * 4), o_tk = take(64);
  if (a) {
    uint8_t* w = reinterpret_cast<uint8_t*>(s->workspace);
    a->zpos = reinterpret_cast<float*>(w + o_zpos);
    a->zneg = reinterpret_cast<float*>(w + o_zneg);
    a->dz16 = s->neg_mode == 0 ? reinterpret_cast<__nv_bfloat16*>(w + o_dz16) : nullptr;
    a->e_neg = s->neg_mode == 0 ? reinterpret_cast<__nv_bfloat16*>(w + o_eneg) : nullptr;
    a->de_neg = s->neg_mode == 0 ? reinterpret_cast<float*>(w + o_deneg) : nullptr;
    a->block_sums = reinterpret_cast<float*>(w + o_bs);
    a->ticket = reinterpret_cast<unsigned int*>(w + o_tk);
    a->ldz = ldz;
    a->ldn = ldn;
  }
  return off;
}

static int sampled_args(const rp_sampled_desc* s, SampledArgs* a, MultiPos* mp) {
  if (!s || !s->hc || !s->table || !s->labels || !s->negatives || !s->n_valid || !s->loss_out || !s->workspace) return RP_EINVAL;
  if (s->capacity <= 0 || s->n_items <= 0 || s->n_neg <= 0) return RP_ESHAPE;
  if (s->d != 64 && s->d != 128 && s->d != 256 && s->d != 512) return RP_ESHAPE;
  if (s->neg_mode < 0 || s->neg_mode > 2 || s->kind < 0 || s->kind > 5) return RP_EINVAL;
  if (s->kind == kCESampledWeighted && !s->row_weight) return RP_EINVAL;
  if (s->neg_mode != 0 && (!s->valid_idx || s->seq_len <= 0)) return RP_EINVAL;
  if (s->kind == kLegacyCE && s->vocab_size < 2) return RP_EINVAL;
  if (s->num_positives < 0 || s->num_positives > RP_MAX_POSITIVES) return RP_ESHAPE;
  if (s->num_positives > 1 && (!s->slot_mask || !s->n_pairs ||
                               (s->kind != kCESampled && s->kind != kBCESampled && s->kind != kCESampledWeighted)))
    return RP_EINVAL;
  if (s->workspace_bytes < sampled_layout(s, nullptr)) return RP_EWORKSPACE;
  a->hc = reinterpret_cast<const __nv_bfloat16*>(s->hc);
  a->table = reinterpret_cast<const __nv_bfloat16*>(s->table);
  a->labels = s->labels; a->valid_idx = s->valid_idx; a->negatives = s->negatives; a->n_valid = s->n_valid;
  a->row_weight = s->kind == kCESampledWeighted ? s->row_weight : nullptr;
  a->capacity = s->capacity; a->n_items = s->n_items; a->d = s->d; a->N = s->n_neg; a->neg_mode = s->neg_mode;
  a->L = s->seq_len; a->kind = s->kind; a->ignore_index = s->ignore_index; a->vocab_size = s->vocab_size;
  a->log_eps = s->log_eps; a->clamp = s->clamp; a->loss_out = s->loss_out;
  mp->P = s->num_positives > 1 ? s->num_positives : 1;
  mp->slot_mask = mp->P > 1 ? s->slot_mask : nullptr;
  mp->n_pairs = mp->P > 1 ? s->n_pairs : nullptr;
  sampled_layout(s, a);
  return RP_OK;
}

#define RP_DISPATCH_SD(d, CALL)          \
  switch (d) {                           \
    case 64: { constexpr int D = 64; CALL; } break;    \
    case 128: { constexpr int D = 128; CALL; } break;  \
    case 256: { constexpr int D = 256; CALL; } break;  \
    default: { constexpr int D = 512; CALL; } break;   \
  }

RP_API size_t rp_sampled_head_workspace_multi(int capacity, int d, int n_neg, int neg_mode, int num_positives) {
  rp_sampled_desc s;
  memset(&s, 0, sizeof(s));
  s.capacity = capacity; s.d = d; s.n_neg = n_neg; s.neg_mode = neg_mode; s.num_positives = num_positives;
  if (capacity <= 0 || d <= 0 || n_neg <= 0 || num_positives < 0 || num_positives > RP_MAX_POSITIVES) return 0;
  return sampled_layout(&s, nullptr);
}

RP_API size_t rp_sampled_head_workspace(int capacity, int d, int n_neg, int neg_mode) {
  return rp_sampled_head_workspace_multi(capacity, d, n_neg, neg_mode, 1);
}

// loss_out[0] = mean loss over the valid targets (the pairs with P > 1), loss_out[1] = 1 / their count; the workspace keeps d(loss)/d(logits) for the backward
RP_API int rp_sampled_head_fwd(const rp_sampled_desc* s, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  SampledArgs a;
  MultiPos mp;
  int rc = sampled_args(s, &a, &mp);
  if (rc != RP_OK) return rc;
  const int blocks = sm_count() * 4;
  RP_CUDA_CHECK(cudaMemsetAsync(a.ticket, 0, 64, stream));
  if (a.neg_mode == 0) {
    sampled_gather_neg_kernel<<<(a.N + 7) / 8, 256, 0, stream>>>(a);
    RP_LAUNCH_CHECK();
    rp_gemm_desc g = rp_gemm_default();
    g.A = a.hc; g.a_rows = a.capacity; g.a_cols = a.d; g.lda = a.d;
    g.B = a.e_neg; g.b_rows = a.N; g.b_cols = a.d; g.ldb = a.d;
    g.M = a.capacity; g.N = a.N; g.K = a.d;
    g.C = a.zneg; g.ldc = a.ldz; g.out_mode = 2;
    g.m_limit_dev = a.n_valid;
    if ((rc = rp_gemm(&g, stream_)) != RP_OK) return rc;
  }
  if (mp.P > 1) {
    RP_DISPATCH_SD(a.d, (sampled_logits_kernel<D, true><<<blocks, 256, 0, stream>>>(a, mp)));
    RP_LAUNCH_CHECK();
    sampled_loss_multi_kernel<<<blocks < 1024 ? blocks : 1024, 256, 0, stream>>>(a, mp);
  } else {
    RP_DISPATCH_SD(a.d, (sampled_logits_kernel<D, false><<<blocks, 256, 0, stream>>>(a, mp)));
    RP_LAUNCH_CHECK();
    sampled_loss_kernel<<<blocks < 1024 ? blocks : 1024, 256, 0, stream>>>(a);
  }
  RP_LAUNCH_CHECK();
  return RP_OK;
}

// d_hc bf16 [capacity, d] (rows < *n_valid written); d_table fp32 [>= n_items, d] ACCUMULATED (+=): zero it first
RP_API int rp_sampled_head_bwd(const rp_sampled_desc* s, void* d_hc, float* d_table, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  SampledArgs a;
  MultiPos mp;
  int rc = sampled_args(s, &a, &mp);
  if (rc != RP_OK) return rc;
  if (!d_hc || !d_table) return RP_EINVAL;
  const int blocks = sm_count() * 4;
  if (a.neg_mode == 0) {
    // dH = dz . E_neg
    rp_gemm_desc g = rp_gemm_default();
    g.A = a.dz16; g.a_rows = (a.capacity + 127) / 128 * 128; g.a_cols = a.N; g.lda = a.ldn;
    g.B = a.e_neg; g.b_rows = a.N; g.b_cols = a.d; g.ldb = a.d; g.b_mn = 1;
    g.M = a.capacity; g.N = a.d; g.K = a.N;
    g.C = d_hc; g.ldc = a.d; g.out_mode = 0;
    g.m_limit_dev = a.n_valid;
    if ((rc = rp_gemm(&g, stream_)) != RP_OK) return rc;
    // dE_neg = dz^T . hc
    g = rp_gemm_default();
    g.A = a.dz16; g.a_rows = (a.capacity + 127) / 128 * 128; g.a_cols = a.N; g.lda = a.ldn; g.a_mn = 1;
    g.B = a.hc; g.b_rows = a.capacity; g.b_cols = a.d; g.ldb = a.d; g.b_mn = 1;
    g.M = a.N; g.N = a.d; g.K = a.capacity;
    g.C = a.de_neg; g.ldc = a.d; g.out_mode = 2;
    g.k_limit_dev = a.n_valid;
    if ((rc = rp_gemm(&g, stream_)) != RP_OK) return rc;
    sampled_scatter_neg_kernel<<<(a.N + 7) / 8, 256, 0, stream>>>(a, d_table);
    RP_LAUNCH_CHECK();
  }
  __nv_bfloat16* dh = reinterpret_cast<__nv_bfloat16*>(d_hc);
  const int add = a.neg_mode == 0 ? 1 : 0;
  if (mp.P > 1) {
    RP_DISPATCH_SD(a.d, (sampled_bwd_kernel<D, true><<<blocks, 256, 0, stream>>>(a, dh, d_table, add, mp)));
  } else {
    RP_DISPATCH_SD(a.d, (sampled_bwd_kernel<D, false><<<blocks, 256, 0, stream>>>(a, dh, d_table, add, mp)));
  }
  RP_LAUNCH_CHECK();
  return RP_OK;
}

static int bce_multi_check(const void* hc, const void* table, const int32_t* labels, const int32_t* labels_p,
                           const int32_t* n_valid, int capacity, int num_positives, int n_items, int d) {
  if (!hc || !table || !labels || !labels_p || !n_valid) return RP_EINVAL;
  if (capacity <= 0 || n_items <= 0 || num_positives < 1 || num_positives > RP_MAX_POSITIVES) return RP_ESHAPE;
  if (d != 64 && d != 128 && d != 256 && d != 512) return RP_ESHAPE;
  return RP_OK;
}

RP_API int rp_bce_head_multi_fwd(const void* hc, const void* table, const int32_t* labels, const int32_t* labels_p,
                                 const int32_t* n_valid, int capacity, int num_positives, int n_items, int d, float* loss_out,
                                 float* row_sum, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  int rc = bce_multi_check(hc, table, labels, labels_p, n_valid, capacity, num_positives, n_items, d);
  if (rc != RP_OK) return rc;
  if (!loss_out || !row_sum) return RP_EINVAL;
  const __nv_bfloat16* h = reinterpret_cast<const __nv_bfloat16*>(hc);
  const __nv_bfloat16* e = reinterpret_cast<const __nv_bfloat16*>(table);
  RP_DISPATCH_SD(d, (bce_extra_fwd_kernel<D><<<sm_count() * 4, 256, 0, stream>>>(h, e, labels, labels_p, n_valid,
                                                                                 num_positives, n_items, row_sum)));
  RP_LAUNCH_CHECK();
  bce_extra_loss_kernel<<<1, 1024, 0, stream>>>(row_sum, n_valid, loss_out);
  RP_LAUNCH_CHECK();
  return RP_OK;
}

RP_API int rp_bce_head_multi_bwd(const void* hc, const void* table, const int32_t* labels, const int32_t* labels_p,
                                 const int32_t* n_valid, int capacity, int num_positives, int n_items, int d,
                                 const float* loss_out, void* d_hc, float* d_table, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  int rc = bce_multi_check(hc, table, labels, labels_p, n_valid, capacity, num_positives, n_items, d);
  if (rc != RP_OK) return rc;
  if (!loss_out || !d_hc || !d_table) return RP_EINVAL;
  const __nv_bfloat16* h = reinterpret_cast<const __nv_bfloat16*>(hc);
  const __nv_bfloat16* e = reinterpret_cast<const __nv_bfloat16*>(table);
  RP_DISPATCH_SD(d, (bce_extra_bwd_kernel<D><<<sm_count() * 4, 256, 0, stream>>>(
                        h, e, labels, labels_p, n_valid, num_positives, n_items, loss_out,
                        reinterpret_cast<__nv_bfloat16*>(d_hc), d_table)));
  RP_LAUNCH_CHECK();
  return RP_OK;
}
