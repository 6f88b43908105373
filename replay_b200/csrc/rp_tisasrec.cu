// rp_tisasrec.cu - TiSASRec's time-interval attention (replay/models/nn/sequential/sasrec/model.py TiSasRecAttention,
// arXiv WSDM'20 "Time Interval Aware Self-Attention") without the reference's [B, L, L, d] time tensors.
//
// Per head, with r_ij = min(floor(|t_i - t_j|), time_span) computed here from the [B, L] timestamps:
//   S_ij = (q_i . k'_j + q_i . TKm_ij) * scale,   k' = k + dropout(pos_k),  TKm_ij = dropout(E_K[r_ij])
//   A = softmax(S) over the causal keys (pad query rows: A = 0, their block output is zeroed by the caller),
//   Ad = dropout(A),  o_i = sum_j Ad_ij (v'_j + TVm_ij),  v' = v + dropout(pos_v),  TVm_ij = dropout(E_V[r_ij])
// q . k'^T and Ad . v' are rp_gemm calls on the tensor cores; the kernels here add the time terms, which are per pair
// (and, with dropout, per element), so they cannot be a GEMM.  The time-term dropout masks are keyed by (token b*L + i,
// key j) and the padded column, and are regenerated in the backward from the same key (csrc/rp_philox.cuh stream).
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

#include "rp_b200.h"
#include "rp_host.h"
#include "rp_philox.cuh"
#include "rp_sm90.cuh"

namespace rp {
namespace ti {

constexpr int kSlot = 64;     // one 64-wide feature slot per head
constexpr int kMaxL = 256;
constexpr int kWarps = 8;
constexpr int kBwdCtas = 256;  // time-table gradient partials: at most kBwdCtas / H CTAs per head, each looping over sequences

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// r = min(floor(|a - b|), span) in the timestamps' own dtype (0 int64, 1 float32, 2 float64); raw 8-byte slots
__device__ __forceinline__ int interval(unsigned long long a, unsigned long long b, int dtype, int span) {
  if (dtype == 0) {
    long long d = (long long)a - (long long)b;
    d = d < 0 ? -d : d;
    return d > span ? span : (int)d;
  }
  if (dtype == 1) {
    const float d = floorf(fabsf(__uint_as_float((uint32_t)a) - __uint_as_float((uint32_t)b)));
    return d > (float)span ? span : (int)d;
  }
  const double d = floor(fabs(__longlong_as_double((long long)a) - __longlong_as_double((long long)b)));
  return d > (double)span ? span : (int)d;
}

__device__ __forceinline__ unsigned long long load_time(const void* times, int dtype, long long t) {
  if (dtype == 1) return (unsigned long long)__float_as_uint(reinterpret_cast<const float*>(times)[t]);
  return reinterpret_cast<const unsigned long long*>(times)[t];
}

// --------------------------------------------------------------------------------------------------------------------
// Forward rows: one CTA per (sequence, head), one warp per query row.  In: S = q . k'^T (fp32 [B*H, Lp, Lp]).  Out: the
// probabilities A (bf16, saved for the backward), Ad (bf16, the A operand of the o GEMM; may alias A when drop_p == 0)
// and hpre = q_in + sum_j Ad_ij TVm_ij (bf16, the residual of the o GEMM).
// --------------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kWarps * 32) ti_fwd_kernel(rp_ti_attn_desc p, const float* __restrict__ S,
                                                             const __nv_bfloat16* __restrict__ q_in, __nv_bfloat16* a_save,
                                                             __nv_bfloat16* ad, __nv_bfloat16* __restrict__ hpre) {
  extern __shared__ __align__(16) unsigned char smem[];
  const int n_r = p.time_span + 1;
  __nv_bfloat16* tk = reinterpret_cast<__nv_bfloat16*>(smem);            // [n_r][64]
  __nv_bfloat16* tv = tk + (size_t)n_r * kSlot;                             // [n_r][64]
  unsigned long long* ts = reinterpret_cast<unsigned long long*>(tv + (size_t)n_r * kSlot);  // [L]
  uint32_t* ck = reinterpret_cast<uint32_t*>(ts + kMaxL);                   // [64] column keys of the head's slot
  float* wsm = reinterpret_cast<float*>(ck + kSlot);                        // per warp: q[64], ad[256], r[256], rkv[256]
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float* qs = wsm + warp * (kSlot + 3 * kMaxL);
  float* adw = qs + kSlot;
  int* rw = reinterpret_cast<int*>(adw + kMaxL);
  uint32_t* rkv = reinterpret_cast<uint32_t*>(rw + kMaxL);

  const int bz = blockIdx.x, b = bz / p.H, h = bz % p.H, L = p.L, Lp = (L + 63) & ~63;
  const bool drop = p.drop_p > 0.f;
  const unsigned long long seed = p.seed + (drop && p.seed_ptr ? *p.seed_ptr : 0ull);
  const uint32_t thr = drop ? (uint32_t)(p.drop_p * 4294967296.0) : 0u;
  const float ks = drop ? 1.f / (1.f - p.drop_p) : 1.f;
  for (int e = threadIdx.x; e < n_r * (kSlot / 8); e += blockDim.x) {
    const int r = e / (kSlot / 8), c = (e % (kSlot / 8)) * 8;
    const size_t src = (size_t)r * p.ld_t + h * kSlot + c;
    *reinterpret_cast<uint4*>(tk + r * kSlot + c) = *reinterpret_cast<const uint4*>(
        reinterpret_cast<const __nv_bfloat16*>(p.time_k) + src);
    *reinterpret_cast<uint4*>(tv + r * kSlot + c) = *reinterpret_cast<const uint4*>(
        reinterpret_cast<const __nv_bfloat16*>(p.time_v) + src);
  }
  for (int j = threadIdx.x; j < L; j += blockDim.x) ts[j] = load_time(p.times, p.times_dtype, (long long)b * L + j);
  for (int c = threadIdx.x; c < kSlot; c += blockDim.x) ck[c] = drop_col_key((uint32_t)(h * kSlot + c));
  __syncthreads();

  const int c0 = 2 * lane;
  for (int i = warp; i < L; i += kWarps) {
    const long long t = (long long)b * L + i;
    const size_t row = ((size_t)bz * Lp + i) * Lp;
    const size_t col = (size_t)t * p.ldq + h * kSlot + c0;
    const uint32_t qin = *reinterpret_cast<const uint32_t*>(q_in + col);
    if (!p.pad_mask[t]) {  // dead query row: no attention, hpre = q_in
      for (int j = lane; j < Lp; j += 32) {
        a_save[row + j] = __float2bfloat16(0.f);
        ad[row + j] = __float2bfloat16(0.f);
      }
      *reinterpret_cast<uint32_t*>(hpre + col) = qin;
      continue;
    }
    {
      const float2 qf = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(
          reinterpret_cast<const __nv_bfloat16*>(p.q) + col));
      qs[c0] = qf.x;
      qs[c0 + 1] = qf.y;
    }
    __syncwarp();
    // phase 1: one lane per key j <= i
    float sv[kMaxL / 32];
    float m = -INFINITY;
    const unsigned long long ti_ = ts[i];
#pragma unroll
    for (int k = 0; k < kMaxL / 32; ++k) {
      const int j = lane + 32 * k;
      sv[k] = -INFINITY;
      if (j <= i) {
        const int r = interval(ti_, ts[j], p.times_dtype, p.time_span);
        rw[j] = r;
        const __nv_bfloat16* e = tk + r * kSlot;
        float dot = 0.f;
        if (drop) {
          const uint32_t rk = drop_row_key(seed, p.tk_off, (unsigned long long)t * L + j);
          rkv[j] = drop_row_key(seed, p.tv_off, (unsigned long long)t * L + j);
#pragma unroll 8
          for (int c = 0; c < kSlot; c += 2) {
            const float2 ev = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(e + c));
            if (drop_mix(rk, ck[c]) >= thr) dot += qs[c] * ev.x;
            if (drop_mix(rk, ck[c + 1]) >= thr) dot += qs[c + 1] * ev.y;
          }
          dot *= ks;
        } else {
#pragma unroll 8
          for (int c = 0; c < kSlot; c += 2) {
            const float2 ev = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(e + c));
            dot += qs[c] * ev.x + qs[c + 1] * ev.y;
          }
        }
        sv[k] = (S[row + j] + dot) * p.scale;
        m = fmaxf(m, sv[k]);
      }
    }
    m = warp_max(m);
    float sum = 0.f;
#pragma unroll
    for (int k = 0; k < kMaxL / 32; ++k) {
      sv[k] = (lane + 32 * k <= i) ? __expf(sv[k] - m) : 0.f;
      sum += sv[k];
    }
    const float inv = 1.f / warp_sum(sum);
    const uint32_t rka = drop ? drop_row_key(seed, p.att_off, (unsigned long long)bz * Lp + i) : 0u;
#pragma unroll
    for (int k = 0; k < kMaxL / 32; ++k) {
      const int j = lane + 32 * k;
      if (j >= Lp) break;
      const float a = sv[k] * inv;
      float d = a;
      if (drop) d = drop_mix(rka, drop_col_key((uint32_t)j)) >= thr ? a * ks : 0.f;
      a_save[row + j] = __float2bfloat16(a);
      if (ad != a_save) ad[row + j] = __float2bfloat16(d);
      if (j <= i) adw[j] = __bfloat162float(__float2bfloat16(d));   // the value the o GEMM multiplies v' by
    }
    __syncwarp();
    // phase 2: lane owns columns c0, c0 + 1;  sum_j Ad_ij TVm_ij
    float o0 = 0.f, o1 = 0.f;
    const uint32_t ck0 = ck[c0], ck1 = ck[c0 + 1];
    for (int j = 0; j <= i; ++j) {
      const float w = adw[j];
      if (w == 0.f) continue;
      const float2 ev = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(tv + rw[j] * kSlot + c0));
      if (drop) {
        const uint32_t rk = rkv[j];
        o0 += drop_mix(rk, ck0) >= thr ? w * ev.x : 0.f;
        o1 += drop_mix(rk, ck1) >= thr ? w * ev.y : 0.f;
      } else {
        o0 += w * ev.x;
        o1 += w * ev.y;
      }
    }
    const float2 qi = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&qin));
    *reinterpret_cast<uint32_t*>(hpre + col) = pack_bf16(qi.x + o0 * ks, qi.y + o1 * ks);
    __syncwarp();
  }
}

// --------------------------------------------------------------------------------------------------------------------
// Backward rows: CTA (g, h) takes sequences b = g, g + G, ... of head h, one warp per query row.  In: A (forward save),
// dpd = dO . v'^T (bf16 [B*H, Lp, Lp], overwritten with dS), dO.  Out: dS (the A operand of dQ = dS k' and dK' = dS^T q,
// scale included), Ad (the A operand of dV' = Ad^T dO; not written when it aliases A), dq_t = sum_j dS_ij TKm_ij (the
// residual of the dQ GEMM) and the CTA's partial time-table gradients in shared memory, stored to ws[g][h][table].
// The shared-memory sums use fp32 atomics, so their order - and the last bits of the time-table gradients - vary from run
// to run; the partials are reduced across CTAs in a fixed order (ti_table_reduce_kernel).
// --------------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kWarps * 32) ti_bwd_kernel(rp_ti_attn_desc p, const __nv_bfloat16* __restrict__ a_save,
                                                             __nv_bfloat16* __restrict__ dpd, __nv_bfloat16* ad,
                                                             const __nv_bfloat16* __restrict__ d_o,
                                                             __nv_bfloat16* __restrict__ dq_t, float* __restrict__ ws) {
  extern __shared__ __align__(16) unsigned char smem[];
  const int n_r = p.time_span + 1;
  float* acc_k = reinterpret_cast<float*>(smem);                   // [n_r][64]
  float* acc_v = acc_k + (size_t)n_r * kSlot;                      // [n_r][64]
  unsigned long long* ts = reinterpret_cast<unsigned long long*>(acc_v + (size_t)n_r * kSlot);
  uint32_t* ck = reinterpret_cast<uint32_t*>(ts + kMaxL);
  float* wsm = reinterpret_cast<float*>(ck + kSlot);               // per warp: q[64], dO[64], ds[256], ad[256], r, rkk, rkv
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float* qs = wsm + warp * (2 * kSlot + 5 * kMaxL);
  float* dos = qs + kSlot;
  float* dsw = dos + kSlot;
  float* adw = dsw + kMaxL;
  int* rw = reinterpret_cast<int*>(adw + kMaxL);
  uint32_t* rkk = reinterpret_cast<uint32_t*>(rw + kMaxL);
  uint32_t* rkv = rkk + kMaxL;

  const int h = blockIdx.y, L = p.L, Lp = (L + 63) & ~63;
  const bool drop = p.drop_p > 0.f;
  const unsigned long long seed = p.seed + (drop && p.seed_ptr ? *p.seed_ptr : 0ull);
  const uint32_t thr = drop ? (uint32_t)(p.drop_p * 4294967296.0) : 0u;
  const float ks = drop ? 1.f / (1.f - p.drop_p) : 1.f;
  const __nv_bfloat16* TK = reinterpret_cast<const __nv_bfloat16*>(p.time_k) + h * kSlot;
  const __nv_bfloat16* TV = reinterpret_cast<const __nv_bfloat16*>(p.time_v) + h * kSlot;
  for (int e = threadIdx.x; e < 2 * n_r * kSlot; e += blockDim.x) acc_k[e] = 0.f;
  for (int c = threadIdx.x; c < kSlot; c += blockDim.x) ck[c] = drop_col_key((uint32_t)(h * kSlot + c));
  const int c0 = 2 * lane;

  for (int b = blockIdx.x; b < p.B; b += gridDim.x) {
    const int bz = b * p.H + h;
    __syncthreads();   // ts of the previous sequence is no longer read
    for (int j = threadIdx.x; j < L; j += blockDim.x) ts[j] = load_time(p.times, p.times_dtype, (long long)b * L + j);
    __syncthreads();
    for (int i = warp; i < L; i += kWarps) {
      const long long t = (long long)b * L + i;
      const size_t row = ((size_t)bz * Lp + i) * Lp;
      const size_t col = (size_t)t * p.ldq + h * kSlot + c0;
      if (!p.pad_mask[t]) {
        for (int j = lane; j < L; j += 32) {
          dpd[row + j] = __float2bfloat16(0.f);
          if (ad != a_save) ad[row + j] = __float2bfloat16(0.f);
        }
        *reinterpret_cast<uint32_t*>(dq_t + col) = 0u;
        continue;
      }
      {
        const float2 qf = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(
            reinterpret_cast<const __nv_bfloat16*>(p.q) + col));
        const float2 gf = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(d_o + col));
        qs[c0] = qf.x; qs[c0 + 1] = qf.y;
        dos[c0] = gf.x; dos[c0 + 1] = gf.y;
      }
      __syncwarp();
      // phase 1: one lane per key j <= i:  dAd_ij = dpd_ij + dO_i . TVm_ij, dA = dAd * keep, rowsum of A dA
      float av[kMaxL / 32], dav[kMaxL / 32];
      float dot = 0.f;
      const unsigned long long ti_ = ts[i];
      const uint32_t rka = drop ? drop_row_key(seed, p.att_off, (unsigned long long)bz * Lp + i) : 0u;
#pragma unroll
      for (int k = 0; k < kMaxL / 32; ++k) {
        const int j = lane + 32 * k;
        av[k] = 0.f;
        dav[k] = 0.f;
        if (j <= i) {
          const int r = interval(ti_, ts[j], p.times_dtype, p.time_span);
          rw[j] = r;
          const __nv_bfloat16* e = TV + (size_t)r * p.ld_t;
          float tvd = 0.f;
          if (drop) {
            const uint32_t rk = drop_row_key(seed, p.tv_off, (unsigned long long)t * L + j);
            rkv[j] = rk;
            rkk[j] = drop_row_key(seed, p.tk_off, (unsigned long long)t * L + j);
#pragma unroll 8
            for (int c = 0; c < kSlot; c += 2) {
              const float2 ev = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(e + c));
              if (drop_mix(rk, ck[c]) >= thr) tvd += dos[c] * ev.x;
              if (drop_mix(rk, ck[c + 1]) >= thr) tvd += dos[c + 1] * ev.y;
            }
            tvd *= ks;
          } else {
#pragma unroll 8
            for (int c = 0; c < kSlot; c += 2) {
              const float2 ev = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(e + c));
              tvd += dos[c] * ev.x + dos[c + 1] * ev.y;
            }
          }
          const float keep = drop ? (drop_mix(rka, drop_col_key((uint32_t)j)) >= thr ? ks : 0.f) : 1.f;
          av[k] = __bfloat162float(a_save[row + j]);
          dav[k] = (__bfloat162float(dpd[row + j]) + tvd) * keep;
          adw[j] = av[k] * keep;
          dot += av[k] * dav[k];
        }
      }
      dot = warp_sum(dot);
#pragma unroll
      for (int k = 0; k < kMaxL / 32; ++k) {
        const int j = lane + 32 * k;
        if (j >= L) break;
        const float ds = j <= i ? av[k] * (dav[k] - dot) * p.scale : 0.f;
        dpd[row + j] = __float2bfloat16(ds);
        if (ad != a_save) ad[row + j] = __float2bfloat16(j <= i ? adw[j] : 0.f);
        if (j <= i) dsw[j] = ds;
      }
      __syncwarp();
      // phase 2: lane owns columns c0, c0 + 1:  dq_t, and the time-table gradients of the row's pairs
      float g0 = 0.f, g1 = 0.f;
      const float q0 = qs[c0] * ks, q1 = qs[c0 + 1] * ks, o0 = dos[c0] * ks, o1 = dos[c0 + 1] * ks;
      const uint32_t ck0 = ck[c0], ck1 = ck[c0 + 1];
      for (int j = 0; j <= i; ++j) {
        const int r = rw[j];
        const float ds = dsw[j], w = adw[j];
        bool kk0 = true, kk1 = true, kv0 = true, kv1 = true;
        if (drop) {
          kk0 = drop_mix(rkk[j], ck0) >= thr; kk1 = drop_mix(rkk[j], ck1) >= thr;
          kv0 = drop_mix(rkv[j], ck0) >= thr; kv1 = drop_mix(rkv[j], ck1) >= thr;
        }
        if (ds != 0.f) {
          const float2 ev = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(TK + (size_t)r * p.ld_t + c0));
          if (kk0) { g0 += ds * ev.x; atomicAdd(acc_k + r * kSlot + c0, ds * q0); }
          if (kk1) { g1 += ds * ev.y; atomicAdd(acc_k + r * kSlot + c0 + 1, ds * q1); }
        }
        if (w != 0.f) {
          if (kv0) atomicAdd(acc_v + r * kSlot + c0, w * o0);
          if (kv1) atomicAdd(acc_v + r * kSlot + c0 + 1, w * o1);
        }
      }
      *reinterpret_cast<uint32_t*>(dq_t + col) = pack_bf16(g0 * ks, g1 * ks);
      __syncwarp();
    }
  }
  __syncthreads();
  float* dst = ws + ((size_t)blockIdx.x * p.H + h) * 2 * n_r * kSlot;
  for (int e = threadIdx.x; e < 2 * n_r * kSlot; e += blockDim.x) dst[e] = acc_k[e];
}

// d_table[t][r][h*64 + c] += sum over g = 0 .. G-1 (in order) of ws[g][h][t][r][c], for the true columns c < head_dim
__global__ void ti_table_reduce_kernel(const float* __restrict__ ws, int G, int H, int n_r, int head_dim, long long ld_t,
                                       float* __restrict__ d_tk, float* __restrict__ d_tv) {
  const long long n = (long long)H * 2 * n_r * kSlot;
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < n; e += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(e % kSlot), r = (int)((e / kSlot) % n_r), tbl = (int)((e / ((long long)kSlot * n_r)) % 2);
    const int h = (int)(e / (2LL * kSlot * n_r));
    if (c >= head_dim) continue;
    float s = 0.f;
    for (int g = 0; g < G; ++g) s += ws[(((size_t)g * H + h) * 2 + tbl) * n_r * kSlot + (size_t)r * kSlot + c];
    float* d = tbl == 0 ? d_tk : d_tv;
    d[(size_t)r * ld_t + h * kSlot + c] += s;
  }
}

// kv[t][c] += dropout(pos_k[t % L][c]) (c < d), kv[t][d + c] += dropout(pos_v[t % L][c]); token row keys
__global__ void ti_pos_add_kernel(__nv_bfloat16* __restrict__ kv, long long ld, const float* __restrict__ pos_k,
                                  const float* __restrict__ pos_v, long long T, int L, int d, float drop_p,
                                  unsigned long long seed, const unsigned long long* __restrict__ seed_ptr,
                                  unsigned long long off_k, unsigned long long off_v) {
  if (drop_p > 0.f && seed_ptr) seed += *seed_ptr;
  const uint32_t thr = drop_p > 0.f ? (uint32_t)(drop_p * 4294967296.0) : 0u;
  const float ks = drop_p > 0.f ? 1.f / (1.f - drop_p) : 1.f;
  const long long n = T * 2 * d;
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < n; e += (long long)gridDim.x * blockDim.x) {
    const long long t = e / (2 * d);
    const int cc = (int)(e % (2 * d)), half = cc >= d, c = cc - half * d;
    float v = (half ? pos_v : pos_k)[(size_t)(t % L) * d + c];
    if (drop_p > 0.f) v = drop_mix(drop_row_key(seed, half ? off_v : off_k, (unsigned long long)t), drop_col_key((uint32_t)c)) >= thr ? v * ks : 0.f;
    __nv_bfloat16* o = kv + (size_t)t * ld + cc;
    *o = __float2bfloat16(__bfloat162float(*o) + v);
  }
}

// d_pos_{k,v}[l][c] += sum over b (in order) of dropout'(dkv[b*L + l][c | d + c]), true columns only
__global__ void ti_pos_bwd_kernel(const __nv_bfloat16* __restrict__ dkv, long long ld, int B, int L, int d, int head_dim,
                                  float drop_p, unsigned long long seed, const unsigned long long* __restrict__ seed_ptr,
                                  unsigned long long off_k, unsigned long long off_v, float* __restrict__ d_pos_k,
                                  float* __restrict__ d_pos_v) {
  if (drop_p > 0.f && seed_ptr) seed += *seed_ptr;
  const uint32_t thr = drop_p > 0.f ? (uint32_t)(drop_p * 4294967296.0) : 0u;
  const float ks = drop_p > 0.f ? 1.f / (1.f - drop_p) : 1.f;
  const long long n = (long long)L * 2 * d;
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < n; e += (long long)gridDim.x * blockDim.x) {
    const int l = (int)(e / (2 * d)), cc = (int)(e % (2 * d)), half = cc >= d, c = cc - half * d;
    if (c % kSlot >= head_dim) continue;
    const uint32_t ckey = drop_col_key((uint32_t)c);
    float s = 0.f;
    for (int b = 0; b < B; ++b) {
      const long long t = (long long)b * L + l;
      const float g = __bfloat162float(dkv[(size_t)t * ld + cc]);
      if (drop_p > 0.f) s += drop_mix(drop_row_key(seed, half ? off_v : off_k, (unsigned long long)t), ckey) >= thr ? g * ks : 0.f;
      else s += g;
    }
    (half ? d_pos_v : d_pos_k)[(size_t)l * d + c] += s;
  }
}

inline size_t fwd_smem(int n_r) {
  return (size_t)2 * n_r * kSlot * sizeof(__nv_bfloat16) + kMaxL * 8 + kSlot * 4 + (size_t)kWarps * (kSlot + 3 * kMaxL) * 4;
}
inline size_t bwd_smem(int n_r) {
  return (size_t)2 * n_r * kSlot * sizeof(float) + kMaxL * 8 + kSlot * 4 + (size_t)kWarps * (2 * kSlot + 5 * kMaxL) * 4;
}
inline int bwd_ctas(int B, int H) {
  const int g = kBwdCtas / H;
  return g < 1 ? 1 : (g < B ? g : B);
}

int check_desc(const rp_ti_attn_desc* p) {
  if (!p || !p->q || !p->pad_mask || !p->times || !p->time_k || !p->time_v) return RP_EINVAL;
  if (p->times_dtype < 0 || p->times_dtype > 2 || p->drop_p < 0.f || p->drop_p >= 1.f) return RP_EINVAL;
  if (p->B <= 0 || p->H <= 0 || p->L <= 0 || p->L > kMaxL || p->H * kSlot > RP_TI_MAX_COLS || p->ldq < p->H * kSlot ||
      p->ld_t < p->H * kSlot || p->time_span < 1 || p->time_span > RP_TI_MAX_SPAN || p->head_dim < 1 || p->head_dim > kSlot)
    return RP_ESHAPE;
  if (p->ldq % 2 || p->ld_t % 8) return RP_EALIGN;
  return RP_OK;
}

}  // namespace ti
}  // namespace rp

using namespace rp::ti;

RP_API int rp_ti_attn_fwd(const rp_ti_attn_desc* p, const float* s, const void* q_in, void* a_save, void* ad, void* hpre,
                          void* stream_) {
  const int rc = check_desc(p);
  if (rc != RP_OK) return rc;
  if (!s || !q_in || !a_save || !ad || !hpre || (ad == a_save && p->drop_p > 0.f)) return RP_EINVAL;
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  const size_t smem = fwd_smem(p->time_span + 1);
  RP_CUDA_CHECK(cudaFuncSetAttribute(ti_fwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  ti_fwd_kernel<<<p->B * p->H, kWarps * 32, smem, stream>>>(*p, s, reinterpret_cast<const __nv_bfloat16*>(q_in),
                                                              reinterpret_cast<__nv_bfloat16*>(a_save),
                                                              reinterpret_cast<__nv_bfloat16*>(ad),
                                                              reinterpret_cast<__nv_bfloat16*>(hpre));
  RP_LAUNCH_CHECK();
  return RP_OK;
}

RP_API size_t rp_ti_attn_bwd_workspace(int B, int H, int time_span) {
  if (B <= 0 || H <= 0 || time_span < 1 || time_span > RP_TI_MAX_SPAN) return 0;
  return (size_t)bwd_ctas(B, H) * H * 2 * (time_span + 1) * kSlot * sizeof(float);
}

RP_API int rp_ti_attn_bwd(const rp_ti_attn_desc* p, const void* a_save, void* dpd, void* ad, const void* d_o, void* dq_t,
                          void* ws, size_t ws_bytes, float* d_time_k, float* d_time_v, void* stream_) {
  const int rc = check_desc(p);
  if (rc != RP_OK) return rc;
  if (!a_save || !dpd || !ad || !d_o || !dq_t || !ws || !d_time_k || !d_time_v || (ad == a_save && p->drop_p > 0.f))
    return RP_EINVAL;
  if (ws_bytes < rp_ti_attn_bwd_workspace(p->B, p->H, p->time_span)) return RP_EWORKSPACE;
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  const int n_r = p->time_span + 1, G = bwd_ctas(p->B, p->H);
  const size_t smem = bwd_smem(n_r);
  RP_CUDA_CHECK(cudaFuncSetAttribute(ti_bwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  ti_bwd_kernel<<<dim3(G, p->H), kWarps * 32, smem, stream>>>(
      *p, reinterpret_cast<const __nv_bfloat16*>(a_save), reinterpret_cast<__nv_bfloat16*>(dpd),
      reinterpret_cast<__nv_bfloat16*>(ad), reinterpret_cast<const __nv_bfloat16*>(d_o), reinterpret_cast<__nv_bfloat16*>(dq_t),
      reinterpret_cast<float*>(ws));
  RP_LAUNCH_CHECK();
  const long long n = (long long)p->H * 2 * n_r * kSlot;
  ti_table_reduce_kernel<<<(int)((n + 255) / 256), 256, 0, stream>>>(reinterpret_cast<const float*>(ws), G, p->H, n_r,
                                                                      p->head_dim, p->ld_t, d_time_k, d_time_v);
  RP_LAUNCH_CHECK();
  return RP_OK;
}

RP_API int rp_ti_pos_add(void* kv, long long ld_kv, const float* pos_k, const float* pos_v, int T, int L, int d, float drop_p,
                         unsigned long long seed, const unsigned long long* seed_ptr, unsigned long long off_k,
                         unsigned long long off_v, void* stream_) {
  if (!kv || !pos_k || !pos_v || drop_p < 0.f || drop_p >= 1.f) return RP_EINVAL;
  if (T <= 0 || L <= 0 || T % L || d <= 0 || ld_kv < 2 * d) return RP_ESHAPE;
  const long long n = (long long)T * 2 * d;
  const int grid = (int)((n + 255) / 256 < 8192 ? (n + 255) / 256 : 8192);
  ti_pos_add_kernel<<<grid, 256, 0, reinterpret_cast<cudaStream_t>(stream_)>>>(
      reinterpret_cast<__nv_bfloat16*>(kv), ld_kv, pos_k, pos_v, T, L, d, drop_p, seed, seed_ptr, off_k, off_v);
  RP_LAUNCH_CHECK();
  return RP_OK;
}

RP_API int rp_ti_pos_bwd(const void* dkv, long long ld_kv, int B, int L, int d, int head_dim, float drop_p,
                         unsigned long long seed, const unsigned long long* seed_ptr, unsigned long long off_k,
                         unsigned long long off_v, float* d_pos_k, float* d_pos_v, void* stream_) {
  if (!dkv || !d_pos_k || !d_pos_v || drop_p < 0.f || drop_p >= 1.f) return RP_EINVAL;
  if (B <= 0 || L <= 0 || d <= 0 || ld_kv < 2 * d || head_dim < 1 || head_dim > kSlot) return RP_ESHAPE;
  const long long n = (long long)L * 2 * d;
  ti_pos_bwd_kernel<<<(int)((n + 255) / 256), 256, 0, reinterpret_cast<cudaStream_t>(stream_)>>>(
      reinterpret_cast<const __nv_bfloat16*>(dkv), ld_kv, B, L, d, head_dim, drop_p, seed, seed_ptr, off_k, off_v, d_pos_k,
      d_pos_v);
  RP_LAUNCH_CHECK();
  return RP_OK;
}
