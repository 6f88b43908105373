// rp_sampled_head.cu - sampled-softmax / sampled-BCE training heads (SURVEY.md §8 a9, f.2): logits only for the positive item
// and N sampled negatives per target token, loss and gradients.  Replaces
//   SampledLossBase.get_sampled_logits + mask_negative_logits      replay/nn/loss/base.py:40-154,157-196
//   CESampled.forward                                             replay/nn/loss/ce.py:199-249
//   BCESampled.forward                                            replay/nn/loss/bce.py:154-218
//   LogInCESampled.forward                                        replay/nn/loss/login_ce.py:240-375
//   CESampledWeighted.forward                                     replay/nn/loss/ce.py:252-330
//   legacy _compute_loss_ce_sampled / _compute_loss_bce_sampled    replay/models/nn/sequential/sasrec/lightning.py:310-376
// (single positive per position; the negatives are an INPUT, as in the reference's new path).
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

// one warp per valid token: z_pos = h . E[y]; (modes 1, 2) z_neg[j] = h . E[neg(t, j)]
template <int D>
__global__ void sampled_logits_kernel(const SampledArgs a) {
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
    const float zp = warp_dot<D>(h, a.table + (size_t)a.labels[t] * D, lane);
    if (lane == 0) a.zpos[t] = zp;
    if (a.neg_mode != 0) {
      const int64_t* nr = a.negatives + neg_row(a, t) * a.N;
      for (int j = 0; j < a.N; ++j) {
        const float z = warp_dot<D>(h, a.table + (size_t)clamp_item(nr[j], a.n_items) * D, lane);
        if (lane == 0) a.zneg[(size_t)t * a.ldz + j] = z;
      }
    }
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

// backward, one warp per token: dH[t] (+)= dz_pos E[y] (+ sum_j dz_j E[neg_j] for per-token negatives);
// dE[y] += dz_pos h;  dE[neg_j] += dz_j h  (fp32 atomics)
template <int D>
__global__ void sampled_bwd_kernel(const SampledArgs a, __nv_bfloat16* __restrict__ d_hc, float* __restrict__ d_table,
                                   int add_to_dhc) {
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
    one(a.labels[t], a.zpos[t]);
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
};

static size_t ru(size_t x, size_t m) { return (x + m - 1) / m * m; }

static size_t sampled_layout(const rp_sampled_desc* s, SampledArgs* a) {
  const size_t cap128 = ru((size_t)s->capacity, 128);
  const int ldz = (int)ru((size_t)s->n_neg, 4), ldn = (int)ru((size_t)s->n_neg, 8);
  size_t off = 0;
  auto take = [&](size_t bytes) { const size_t o = off; off = ru(off + bytes, 256); return o; };
  const size_t o_zpos = take(cap128 * 4), o_zneg = take(cap128 * ldz * 4);
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

static int sampled_args(const rp_sampled_desc* s, SampledArgs* a) {
  if (!s || !s->hc || !s->table || !s->labels || !s->negatives || !s->n_valid || !s->loss_out || !s->workspace) return RP_EINVAL;
  if (s->capacity <= 0 || s->n_items <= 0 || s->n_neg <= 0) return RP_ESHAPE;
  if (s->d != 64 && s->d != 128 && s->d != 256 && s->d != 512) return RP_ESHAPE;
  if (s->neg_mode < 0 || s->neg_mode > 2 || s->kind < 0 || s->kind > 5) return RP_EINVAL;
  if (s->kind == kCESampledWeighted && !s->row_weight) return RP_EINVAL;
  if (s->neg_mode != 0 && (!s->valid_idx || s->seq_len <= 0)) return RP_EINVAL;
  if (s->kind == kLegacyCE && s->vocab_size < 2) return RP_EINVAL;
  if (s->workspace_bytes < sampled_layout(s, nullptr)) return RP_EWORKSPACE;
  a->hc = reinterpret_cast<const __nv_bfloat16*>(s->hc);
  a->table = reinterpret_cast<const __nv_bfloat16*>(s->table);
  a->labels = s->labels; a->valid_idx = s->valid_idx; a->negatives = s->negatives; a->n_valid = s->n_valid;
  a->row_weight = s->kind == kCESampledWeighted ? s->row_weight : nullptr;
  a->capacity = s->capacity; a->n_items = s->n_items; a->d = s->d; a->N = s->n_neg; a->neg_mode = s->neg_mode;
  a->L = s->seq_len; a->kind = s->kind; a->ignore_index = s->ignore_index; a->vocab_size = s->vocab_size;
  a->log_eps = s->log_eps; a->clamp = s->clamp; a->loss_out = s->loss_out;
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

RP_API size_t rp_sampled_head_workspace(int capacity, int d, int n_neg, int neg_mode) {
  rp_sampled_desc s;
  memset(&s, 0, sizeof(s));
  s.capacity = capacity; s.d = d; s.n_neg = n_neg; s.neg_mode = neg_mode;
  if (capacity <= 0 || d <= 0 || n_neg <= 0) return 0;
  return sampled_layout(&s, nullptr);
}

// loss_out[0] = mean loss over the valid targets, loss_out[1] = 1/T_v; the workspace keeps d(loss)/d(logits) for the backward
RP_API int rp_sampled_head_fwd(const rp_sampled_desc* s, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  SampledArgs a;
  int rc = sampled_args(s, &a);
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
  RP_DISPATCH_SD(a.d, (sampled_logits_kernel<D><<<blocks, 256, 0, stream>>>(a)));
  RP_LAUNCH_CHECK();
  sampled_loss_kernel<<<blocks < 1024 ? blocks : 1024, 256, 0, stream>>>(a);
  RP_LAUNCH_CHECK();
  return RP_OK;
}

// d_hc bf16 [capacity, d] (rows < *n_valid written); d_table fp32 [>= n_items, d] ACCUMULATED (+=): zero it first
RP_API int rp_sampled_head_bwd(const rp_sampled_desc* s, void* d_hc, float* d_table, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  SampledArgs a;
  int rc = sampled_args(s, &a);
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
  RP_DISPATCH_SD(a.d, (sampled_bwd_kernel<D><<<blocks, 256, 0, stream>>>(a, reinterpret_cast<__nv_bfloat16*>(d_hc), d_table,
                                                                        a.neg_mode == 0 ? 1 : 0)));
  RP_LAUNCH_CHECK();
  return RP_OK;
}
