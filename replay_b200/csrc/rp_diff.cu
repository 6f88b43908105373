// rp_diff.cu - DiffTransformer encoder kernels (replay/nn/sequential/sasrec/diff_transformer.py, arXiv 2410.05258):
// fused differential attention forward, its row-wise softmax backward and the lambda gradient chain, RMSNorm forward /
// backward with a configurable group width, and the SwiGLU gate.  Every reduction runs in a fixed order (no float
// atomics), so two runs are bitwise identical.
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

#include "rp_b200.h"
#include "rp_host.h"

namespace rp {
namespace diff {

constexpr int kQkSlot = 64;        // per-head q1 / q2 / k1 / k2 slot width
constexpr int kMaxL = 256;
constexpr int kKStride = kQkSlot + 2;  // bf16 pitch of a resident key row: 33 words, conflict-free across key rows
constexpr int kFwdWarps = 16;
constexpr int kFwdRows = 64;       // query rows per CTA
constexpr int kRmsParts = 1024;    // per-warp weight-gradient partials of rp_rmsnorm_bwd

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

// lambda_h = exp(sum lq1*lk1) - exp(sum lq2*lk2) + lambda_init, summed in index order (one thread)
__device__ float head_lambda(const rp_diff_lambda& lp, int h, float* e1_out = nullptr, float* e2_out = nullptr) {
  float s1 = 0.f, s2 = 0.f;
  for (int j = 0; j < lp.head_dim; ++j) {
    s1 += lp.q1[h * lp.head_dim + j] * lp.k1[h * lp.head_dim + j];
    s2 += lp.q2[h * lp.head_dim + j] * lp.k2[h * lp.head_dim + j];
  }
  const float e1 = expf(s1), e2 = expf(s2);
  if (e1_out) *e1_out = e1;
  if (e2_out) *e2_out = e2;
  return e1 - e2 + lp.lambda_init;
}

// One CTA per (64 query rows, sequence * head); one warp per query row at a time.  K1, K2 and V of the keys the tile can
// see stay resident in shared memory (bf16).  Pass 1 forms both score rows and their max / sum; pass 2 forms
// A = e1 * inv1 - lambda * e2 * inv2 in shared memory and O = A . V; the epilogue applies the per-head RMSNorm.
template <int VS>
__global__ void __launch_bounds__(kFwdWarps * 32) diff_attn_fwd_kernel(rp_diff_attn_desc a) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  __nv_bfloat16* sk1 = reinterpret_cast<__nv_bfloat16*>(smem_raw);
  __nv_bfloat16* sk2 = sk1 + kMaxL * kKStride;
  __nv_bfloat16* sv = sk2 + kMaxL * kKStride;
  float* sq = reinterpret_cast<float*>(sv + kMaxL * VS);  // per warp: q1 [64] | q2 [64]
  float* sp = sq + kFwdWarps * 2 * kQkSlot;                // per warp: p1 [256] | p2 [256]
  __shared__ float s_lambda;

  const int bh = blockIdx.y, b = bh / a.H, h = bh % a.H;
  const int L = a.L, Lp = (L + 63) & ~63, hd = a.head_dim;
  const int q0 = blockIdx.x * kFwdRows;
  const int nk = min(L, q0 + kFwdRows);  // causal: keys beyond the tile's last row are never visible
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const __nv_bfloat16* qk = reinterpret_cast<const __nv_bfloat16*>(a.qk);
  const __nv_bfloat16* vv = reinterpret_cast<const __nv_bfloat16*>(a.v);
  const long long row0 = (long long)b * L;

  if (threadIdx.x == 0) s_lambda = head_lambda(a.lam, h);
  // keys: 32-bit copies of bf16 pairs
  for (int idx = threadIdx.x; idx < nk * (kQkSlot / 2); idx += blockDim.x) {
    const int j = idx / (kQkSlot / 2), c = (idx % (kQkSlot / 2)) * 2;
    const __nv_bfloat16* src = qk + (row0 + j) * a.ld_qk + a.k_c0 + h * 2 * kQkSlot + c;
    *reinterpret_cast<uint32_t*>(sk1 + j * kKStride + c) = *reinterpret_cast<const uint32_t*>(src);
    *reinterpret_cast<uint32_t*>(sk2 + j * kKStride + c) = *reinterpret_cast<const uint32_t*>(src + kQkSlot);
  }
  for (int idx = threadIdx.x; idx < nk * (VS / 8); idx += blockDim.x) {
    const int j = idx / (VS / 8), c = (idx % (VS / 8)) * 8;
    *reinterpret_cast<uint4*>(sv + j * VS + c) =
        *reinterpret_cast<const uint4*>(vv + (row0 + j) * a.ldv + a.v_c0 + h * VS + c);
  }
  __syncthreads();
  const float lambda = s_lambda;
  const float scale = a.scale;
  const float out_scale = 1.f - a.lam.lambda_init;
  float* q1 = sq + warp * 2 * kQkSlot;
  float* q2 = q1 + kQkSlot;
  float* p1 = sp + warp * 2 * kMaxL;
  float* p2 = p1 + kMaxL;
  __nv_bfloat16* e1s = reinterpret_cast<__nv_bfloat16*>(a.e1_save);
  __nv_bfloat16* e2s = reinterpret_cast<__nv_bfloat16*>(a.e2_save);

  for (int i = q0 + warp; i < min(L, q0 + kFwdRows); i += kFwdWarps) {
    const long long tok = row0 + i;
    const __nv_bfloat16* qrow = qk + tok * a.ld_qk + a.q_c0 + h * 2 * kQkSlot;
    for (int c = lane; c < kQkSlot; c += 32) {
      q1[c] = __bfloat162float(qrow[c]);
      q2[c] = __bfloat162float(qrow[kQkSlot + c]);
    }
    __syncwarp();
    // pass 1: scores of both maps over the visible keys (j <= i and (pad[j] or j == i)), running max
    float m1 = -INFINITY, m2 = -INFINITY;
    for (int j = lane; j <= i; j += 32) {
      const bool vis = (j == i) || a.pad_mask[row0 + j];
      float s1 = -INFINITY, s2 = -INFINITY;
      if (vis) {
        float acc1 = 0.f, acc2 = 0.f;
        const __nv_bfloat162* k1 = reinterpret_cast<const __nv_bfloat162*>(sk1 + j * kKStride);
        const __nv_bfloat162* k2 = reinterpret_cast<const __nv_bfloat162*>(sk2 + j * kKStride);
        for (int c = 0; c < hd; c += 2) {
          const float2 x1 = __bfloat1622float2(k1[c >> 1]);
          const float2 x2 = __bfloat1622float2(k2[c >> 1]);
          acc1 = fmaf(q1[c], x1.x, fmaf(q1[c + 1], x1.y, acc1));
          acc2 = fmaf(q2[c], x2.x, fmaf(q2[c + 1], x2.y, acc2));
        }
        s1 = acc1 * scale;
        s2 = acc2 * scale;
      }
      p1[j] = s1;
      p2[j] = s2;
      m1 = fmaxf(m1, s1);
      m2 = fmaxf(m2, s2);
    }
    m1 = warp_max(m1);
    m2 = warp_max(m2);
    float z1 = 0.f, z2 = 0.f;
    for (int j = lane; j <= i; j += 32) {
      const float e1 = p1[j] == -INFINITY ? 0.f : __expf(p1[j] - m1);
      const float e2 = p2[j] == -INFINITY ? 0.f : __expf(p2[j] - m2);
      p1[j] = e1;
      p2[j] = e2;
      z1 += e1;
      z2 += e2;
    }
    const float inv1 = 1.f / warp_sum(z1), inv2 = 1.f / warp_sum(z2);
    if (e1s) {
      const long long r = ((long long)bh * Lp + i) * Lp;
      for (int j = lane; j < Lp; j += 32) {
        e1s[r + j] = __float2bfloat16(j <= i ? p1[j] : 0.f);
        e2s[r + j] = __float2bfloat16(j <= i ? p2[j] : 0.f);
      }
      if (lane == 0) {
        a.inv1[(long long)bh * Lp + i] = inv1;
        a.inv2[(long long)bh * Lp + i] = inv2;
      }
    }
    // pass 2: A = A1 - lambda * A2, O = A . V
    for (int j = lane; j <= i; j += 32) p1[j] = p1[j] * inv1 - lambda * (p2[j] * inv2);
    __syncwarp();
    float o[VS / 32], o2[VS / 32];
#pragma unroll
    for (int t = 0; t < VS / 32; ++t) o[t] = o2[t] = 0.f;
    for (int j = 0; j <= i; ++j) {
      const float aj = p1[j], a2j = p2[j] * inv2;
#pragma unroll
      for (int t = 0; t < VS / 32; ++t) {
        const float vj = __bfloat162float(sv[j * VS + lane + 32 * t]);
        o[t] = fmaf(aj, vj, o[t]);
        o2[t] = fmaf(a2j, vj, o2[t]);
      }
    }
    // per-head RMSNorm over the 2h true value columns (padded columns are zero)
    float ss = 0.f;
#pragma unroll
    for (int t = 0; t < VS / 32; ++t) ss += o[t] * o[t];
    const float rstd = rsqrtf(warp_sum(ss) / (float)(2 * hd) + a.eps);
    __nv_bfloat16* orow = reinterpret_cast<__nv_bfloat16*>(a.out) + tok * a.ldo + h * VS;
    // e1_save switches every save (as rp_diff_attn_fwd validates them): a set o_pre alone must not be written
    __nv_bfloat16* prow = e1s ? reinterpret_cast<__nv_bfloat16*>(a.o_pre) + tok * a.ldo + h * VS : nullptr;
#pragma unroll
    for (int t = 0; t < VS / 32; ++t) {
      const int c = lane + 32 * t;
      orow[c] = __float2bfloat16(o[t] * rstd * a.rms_scale[c] * out_scale);
      if (prow) {
        prow[c] = __float2bfloat16(o[t]);
        a.o32_save[tok * a.ldo + h * VS + c] = o[t];
        a.o2_save[tok * a.ldo + h * VS + c] = o2[t];
      }
    }
    __syncwarp();
  }
}

// One warp per row (sequence * head, query i): A1 = e1 * inv1, A2 = e2 * inv2, r1 = sum A1 dA, r2 = sum A2 dA;
// dS1 = A1 (dA - r1) s, dS2 = -lambda A2 (dA - r2) s, A = A1 - lambda A2, dlambda partial = -r2.
__global__ void __launch_bounds__(256) diff_softmax_bwd_kernel(const __nv_bfloat16* __restrict__ e1, const __nv_bfloat16* __restrict__ e2,
                                                               const float* __restrict__ inv1, const float* __restrict__ inv2,
                                                               const __nv_bfloat16* dA, __nv_bfloat16* dS1, __nv_bfloat16* dS2,
                                                               __nv_bfloat16* A, float* __restrict__ dlam_part, int BH, int H, int L,
                                                               float scale, rp_diff_lambda lam, const __nv_bfloat16* __restrict__ d_on,
                                                               const float* __restrict__ o32, const float* __restrict__ o2,
                                                               const float* __restrict__ rms_scale, float eps, long long ld_o,
                                                               int v_slot) {
  __shared__ float s_lambda[8];
  const int Lp = (L + 63) & ~63;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long long rows = (long long)BH * L;
  for (long long row = (long long)blockIdx.x * 8 + warp; row < rows; row += (long long)gridDim.x * 8) {
    const int bh = (int)(row / L), i = (int)(row % L);
    if (lane == 0) s_lambda[warp] = head_lambda(lam, bh % H);
    __syncwarp();
    const float lambda = s_lambda[warp];
    const long long base = ((long long)bh * Lp + i) * Lp;
    const float i1 = inv1[(long long)bh * Lp + i], i2 = inv2[(long long)bh * Lp + i];
    // r1 = sum_j A1 dA from the saved exponentials.  r2 = sum_j A2 dA = dO_pre . (A2 V), with dO_pre recomputed in fp32 from
    // the normalised output's gradient and the fp32 O_pre: the per-head RMSNorm makes dO_pre orthogonal to O_pre, so the
    // bf16-rounded dO_pre would lose r2 - and the lambda gradient, its sum over every row - to cancellation.
    float r1 = 0.f;
    for (int j = lane; j <= i; j += 32)
      r1 += __bfloat162float(e1[base + j]) * i1 * __bfloat162float(dA[base + j]);
    const long long off = ((long long)(bh / H) * L + i) * ld_o + (bh % H) * v_slot;
    const float alpha = 1.f - lam.lambda_init;
    float ss = 0.f, gx = 0.f, g2 = 0.f, x2 = 0.f;
    for (int c = lane; c < v_slot; c += 32) {
      const float x = o32[off + c], gw = __bfloat162float(d_on[off + c]) * rms_scale[c] * alpha;
      ss += x * x;
      gx += gw * x;
      g2 += gw * o2[off + c];
      x2 += x * o2[off + c];
    }
    ss = warp_sum(ss);
    gx = warp_sum(gx);
    g2 = warp_sum(g2);
    x2 = warp_sum(x2);
    r1 = warp_sum(r1);
    const float n = (float)(2 * lam.head_dim), rstd = rsqrtf(ss / n + eps);
    const float r2 = rstd * g2 - rstd * rstd * rstd * gx / n * x2;
    for (int j = lane; j < L; j += 32) {
      const float g = __bfloat162float(dA[base + j]);
      const float a1 = __bfloat162float(e1[base + j]) * i1, a2 = __bfloat162float(e2[base + j]) * i2;
      dS1[base + j] = __float2bfloat16(a1 * (g - r1) * scale);
      dS2[base + j] = __float2bfloat16(-lambda * a2 * (g - r2) * scale);
      A[base + j] = __float2bfloat16(a1 - lambda * a2);
    }
    if (lane == 0) dlam_part[(long long)bh * Lp + i] = -r2;
    __syncwarp();
  }
}

// One CTA per head: dlambda = sum over sequences and rows of the partials (fixed order), then the chain into lambda_*.
__global__ void __launch_bounds__(256) diff_lambda_bwd_kernel(const float* __restrict__ dlam_part, int B, int H, int L,
                                                              rp_diff_lambda lam, float* gq1, float* gk1, float* gq2, float* gk2) {
  __shared__ float red[256];
  __shared__ float s_e[2];
  const int h = blockIdx.x, Lp = (L + 63) & ~63;
  float acc = 0.f;
  for (long long n = threadIdx.x; n < (long long)B * L; n += blockDim.x) {
    const int b = (int)(n / L), i = (int)(n % L);
    acc += dlam_part[((long long)b * H + h) * Lp + i];
  }
  red[threadIdx.x] = acc;
  __syncthreads();
  for (int s = 128; s > 0; s >>= 1) {
    if (threadIdx.x < s) red[threadIdx.x] += red[threadIdx.x + s];
    __syncthreads();
  }
  if (threadIdx.x == 0) head_lambda(lam, h, &s_e[0], &s_e[1]);
  __syncthreads();
  const float dl = red[0];
  for (int j = threadIdx.x; j < lam.head_dim; j += blockDim.x) {
    const int k = h * lam.head_dim + j;
    gq1[k] += dl * s_e[0] * lam.k1[k];
    gk1[k] += dl * s_e[0] * lam.q1[k];
    gq2[k] -= dl * s_e[1] * lam.k2[k];
    gk2[k] -= dl * s_e[1] * lam.q2[k];
  }
}

// y = x * rstd * w[c % G] * alpha, rstd over the group's n_true features; one warp per (row, group)
template <int G>
__global__ void __launch_bounds__(256) rmsnorm_fwd_kernel(const __nv_bfloat16* __restrict__ x, const float* __restrict__ w, float eps,
                                                          float alpha, int n_rows, int d, int n_true, const int32_t* n_rows_dev,
                                                          const int32_t* gather, __nv_bfloat16* __restrict__ y) {
  constexpr int PER = (G + 31) / 32;
  const int groups = d / G;
  const int rows = n_rows_dev ? min(n_rows, *n_rows_dev) : n_rows;
  const long long items = (long long)rows * groups;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (long long it = (long long)blockIdx.x * 8 + warp; it < items; it += (long long)gridDim.x * 8) {
    const int r = (int)(it / groups), g = (int)(it % groups);
    const long long src = gather ? gather[r] : r;
    const __nv_bfloat16* xr = x + src * d + g * G;
    float v[PER];
    float ss = 0.f;
#pragma unroll
    for (int t = 0; t < PER; ++t) {
      const int c = lane + 32 * t;
      v[t] = c < G ? __bfloat162float(xr[c]) : 0.f;
      ss += v[t] * v[t];
    }
    const float rstd = rsqrtf(warp_sum(ss) / (float)n_true + eps);
    __nv_bfloat16* yr = y + (long long)r * d + g * G;
#pragma unroll
    for (int t = 0; t < PER; ++t) {
      const int c = lane + 32 * t;
      if (c < G) yr[c] = __float2bfloat16(v[t] * rstd * w[c] * alpha);
    }
  }
}

// dx = rstd (g w alpha) - x rstd^3 / n_true * sum(g w alpha x); dw partials per warp (fixed item assignment), reduced by
// rp_reduce_splits in a fixed order.
template <int G>
__global__ void __launch_bounds__(256) rmsnorm_bwd_kernel(const __nv_bfloat16* __restrict__ dy, const __nv_bfloat16* __restrict__ x,
                                                          const float* __restrict__ w, float eps, float alpha, int n_rows, int d,
                                                          int n_true, const int32_t* n_rows_dev, const int32_t* gather,
                                                          __nv_bfloat16* __restrict__ dx, float* __restrict__ dw_part) {
  constexpr int PER = (G + 31) / 32;
  const int groups = d / G;
  const int rows = n_rows_dev ? min(n_rows, *n_rows_dev) : n_rows;
  const long long items = (long long)rows * groups;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int gw = blockIdx.x * 8 + warp;
  float dwp[PER];
#pragma unroll
  for (int t = 0; t < PER; ++t) dwp[t] = 0.f;
  for (long long it = gw; it < items; it += (long long)gridDim.x * 8) {
    const int r = (int)(it / groups), g = (int)(it % groups);
    const long long src = gather ? gather[r] : r;
    const __nv_bfloat16* xr = x + src * d + g * G;
    const __nv_bfloat16* gr = dy + (long long)r * d + g * G;
    float xv[PER], gv[PER];
    float ss = 0.f, dot = 0.f;
#pragma unroll
    for (int t = 0; t < PER; ++t) {
      const int c = lane + 32 * t;
      xv[t] = c < G ? __bfloat162float(xr[c]) : 0.f;
      gv[t] = c < G ? __bfloat162float(gr[c]) * w[c] * alpha : 0.f;
      ss += xv[t] * xv[t];
      dot += gv[t] * xv[t];
    }
    const float rstd = rsqrtf(warp_sum(ss) / (float)n_true + eps);
    dot = warp_sum(dot);
    const float k = rstd * rstd * rstd * dot / (float)n_true;
    __nv_bfloat16* dxr = dx + src * d + g * G;
#pragma unroll
    for (int t = 0; t < PER; ++t) {
      const int c = lane + 32 * t;
      if (c < G) {
        dxr[c] = __float2bfloat16(rstd * gv[t] - xv[t] * k);
        dwp[t] += __bfloat162float(gr[c]) * xv[t] * rstd * alpha;
      }
    }
  }
#pragma unroll
  for (int t = 0; t < PER; ++t) {
    const int c = lane + 32 * t;
    if (c < G) dw_part[(long long)gw * G + c] = dwp[t];
  }
}

__device__ __forceinline__ float silu(float g) { return g / (1.f + __expf(-g)); }

__global__ void swiglu_fwd_kernel(const __nv_bfloat16* __restrict__ gl, long long n, int F, __nv_bfloat16* __restrict__ u) {
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < n; e += (long long)gridDim.x * blockDim.x) {
    const long long r = e / F;
    const int c = (int)(e % F);
    const float g = __bfloat162float(gl[r * 2 * F + c]), l = __bfloat162float(gl[r * 2 * F + F + c]);
    u[e] = __float2bfloat16(silu(g) * l);
  }
}

__global__ void swiglu_bwd_kernel(const __nv_bfloat16* __restrict__ du, const __nv_bfloat16* __restrict__ gl, long long n, int F,
                                  __nv_bfloat16* __restrict__ dgl) {
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < n; e += (long long)gridDim.x * blockDim.x) {
    const long long r = e / F;
    const int c = (int)(e % F);
    const float g = __bfloat162float(gl[r * 2 * F + c]), l = __bfloat162float(gl[r * 2 * F + F + c]);
    const float d = __bfloat162float(du[e]);
    const float sg = 1.f / (1.f + __expf(-g));
    dgl[r * 2 * F + c] = __float2bfloat16(d * l * sg * (1.f + g * (1.f - sg)));
    dgl[r * 2 * F + F + c] = __float2bfloat16(d * g * sg);
  }
}

static int grid_for(long long work, int per_block) {
  long long g = (work + per_block - 1) / per_block;
  const long long cap = (long long)sm_count() * 16;
  if (g > cap) g = cap;
  return g < 1 ? 1 : (int)g;
}

static bool lambda_ok(const rp_diff_lambda& l) {
  return l.q1 && l.k1 && l.q2 && l.k2 && l.head_dim >= 1 && l.head_dim <= kQkSlot;
}

}  // namespace diff
}  // namespace rp

using namespace rp::diff;

RP_API int rp_diff_attn_fwd(const rp_diff_attn_desc* a, void* stream_) {
  if (!a || !a->qk || !a->v || !a->pad_mask || !a->out || !a->rms_scale || !lambda_ok(a->lam)) return RP_EINVAL;
  if (a->B <= 0 || a->H <= 0 || a->L <= 0 || a->L > kMaxL || a->head_dim != a->lam.head_dim) return RP_ESHAPE;
  if (a->v_slot != 64 && a->v_slot != 128) return RP_ESHAPE;
  if (2 * a->head_dim > a->v_slot) return RP_ESHAPE;
  const bool save = a->e1_save != nullptr;
  if (save && (!a->e2_save || !a->inv1 || !a->inv2 || !a->o_pre || !a->o32_save || !a->o2_save)) return RP_EINVAL;
  if ((a->ld_qk | a->ldv | a->q_c0 | a->k_c0 | a->v_c0) & 7 || (a->ldo & 7)) return RP_EALIGN;
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  const dim3 grid((a->L + kFwdRows - 1) / kFwdRows, a->B * a->H);
  const size_t base = (size_t)2 * kMaxL * kKStride * 2 + (size_t)kFwdWarps * (2 * kQkSlot + 2 * kMaxL) * 4;
  if (a->v_slot == 64) {
    const size_t smem = base + (size_t)kMaxL * 64 * 2;
    RP_CUDA_CHECK(cudaFuncSetAttribute(diff_attn_fwd_kernel<64>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    diff_attn_fwd_kernel<64><<<grid, kFwdWarps * 32, smem, stream>>>(*a);
  } else {
    const size_t smem = base + (size_t)kMaxL * 128 * 2;
    RP_CUDA_CHECK(cudaFuncSetAttribute(diff_attn_fwd_kernel<128>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    diff_attn_fwd_kernel<128><<<grid, kFwdWarps * 32, smem, stream>>>(*a);
  }
  RP_LAUNCH_CHECK();
  return RP_OK;
}

RP_API int rp_diff_attn_softmax_bwd(const void* e1, const void* e2, const float* inv1, const float* inv2, const void* dA,
                                    void* dS1, void* dS2, void* A, float* dlam_part, int BH, int H, int L, float scale,
                                    const rp_diff_lambda* lam, const void* d_on, const float* o32, const float* o2,
                                    const float* rms_scale, float eps, long long ld_o, int v_slot, void* stream_) {
  if (!e1 || !e2 || !inv1 || !inv2 || !dA || !dS1 || !dS2 || !A || !dlam_part || !lam || !lambda_ok(*lam) || !d_on || !o32 || !o2 ||
      !rms_scale)
    return RP_EINVAL;
  if (BH <= 0 || H <= 0 || BH % H || L <= 0 || L > kMaxL || (v_slot != 64 && v_slot != 128) || ld_o < (long long)H * v_slot)
    return RP_ESHAPE;
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  diff_softmax_bwd_kernel<<<grid_for((long long)BH * L, 8), 256, 0, stream>>>(
      reinterpret_cast<const __nv_bfloat16*>(e1), reinterpret_cast<const __nv_bfloat16*>(e2), inv1, inv2,
      reinterpret_cast<const __nv_bfloat16*>(dA), reinterpret_cast<__nv_bfloat16*>(dS1), reinterpret_cast<__nv_bfloat16*>(dS2),
      reinterpret_cast<__nv_bfloat16*>(A), dlam_part, BH, H, L, scale, *lam, reinterpret_cast<const __nv_bfloat16*>(d_on), o32, o2,
      rms_scale, eps, ld_o, v_slot);
  RP_LAUNCH_CHECK();
  return RP_OK;
}

RP_API int rp_diff_lambda_bwd(const float* dlam_part, int B, int H, int L, const rp_diff_lambda* lam, float* gq1, float* gk1,
                              float* gq2, float* gk2, void* stream_) {
  if (!dlam_part || !lam || !lambda_ok(*lam) || !gq1 || !gk1 || !gq2 || !gk2) return RP_EINVAL;
  if (B <= 0 || H <= 0 || L <= 0 || L > kMaxL) return RP_ESHAPE;
  diff_lambda_bwd_kernel<<<H, 256, 0, reinterpret_cast<cudaStream_t>(stream_)>>>(dlam_part, B, H, L, *lam, gq1, gk1, gq2, gk2);
  RP_LAUNCH_CHECK();
  return RP_OK;
}

static bool rms_shape_ok(int group, int d, int n_true, int n_rows) {
  return (group == 64 || group == 128 || group == 256 || group == 512) && d > 0 && d <= 512 && d % group == 0 && n_true >= 1 &&
         n_true <= group && n_rows >= 0;
}

RP_API int rp_rmsnorm_fwd(const void* x, const float* w, float eps, float alpha, int n_rows, int d, int group, int n_true,
                          const int32_t* n_rows_dev, const int32_t* gather, void* y, void* stream_) {
  if (!x || !w || !y) return RP_EINVAL;
  if (!rms_shape_ok(group, d, n_true, n_rows)) return RP_ESHAPE;
  if (n_rows == 0) return RP_OK;
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  const int grid = grid_for((long long)n_rows * (d / group), 8);
  auto xp = reinterpret_cast<const __nv_bfloat16*>(x);
  auto yp = reinterpret_cast<__nv_bfloat16*>(y);
  if (group == 64) rmsnorm_fwd_kernel<64><<<grid, 256, 0, stream>>>(xp, w, eps, alpha, n_rows, d, n_true, n_rows_dev, gather, yp);
  else if (group == 128) rmsnorm_fwd_kernel<128><<<grid, 256, 0, stream>>>(xp, w, eps, alpha, n_rows, d, n_true, n_rows_dev, gather, yp);
  else if (group == 256) rmsnorm_fwd_kernel<256><<<grid, 256, 0, stream>>>(xp, w, eps, alpha, n_rows, d, n_true, n_rows_dev, gather, yp);
  else rmsnorm_fwd_kernel<512><<<grid, 256, 0, stream>>>(xp, w, eps, alpha, n_rows, d, n_true, n_rows_dev, gather, yp);
  RP_LAUNCH_CHECK();
  return RP_OK;
}

RP_API size_t rp_rmsnorm_bwd_workspace(int group) {
  return (group == 64 || group == 128 || group == 256 || group == 512) ? (size_t)kRmsParts * group * sizeof(float) : 0;
}

RP_API int rp_rmsnorm_bwd(const void* dy, const void* x, const float* w, float eps, float alpha, int n_rows, int d, int group,
                          int n_true, const int32_t* n_rows_dev, const int32_t* gather, void* dx, float* dw, void* workspace,
                          size_t workspace_bytes, void* stream_) {
  if (!dy || !x || !w || !dx || !dw || !workspace) return RP_EINVAL;
  if (!rms_shape_ok(group, d, n_true, n_rows)) return RP_ESHAPE;
  if (workspace_bytes < rp_rmsnorm_bwd_workspace(group)) return RP_EWORKSPACE;
  if (n_rows == 0) return RP_OK;
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  const int grid = kRmsParts / 8;
  auto dyp = reinterpret_cast<const __nv_bfloat16*>(dy);
  auto xp = reinterpret_cast<const __nv_bfloat16*>(x);
  auto dxp = reinterpret_cast<__nv_bfloat16*>(dx);
  float* part = reinterpret_cast<float*>(workspace);
  if (group == 64) rmsnorm_bwd_kernel<64><<<grid, 256, 0, stream>>>(dyp, xp, w, eps, alpha, n_rows, d, n_true, n_rows_dev, gather, dxp, part);
  else if (group == 128) rmsnorm_bwd_kernel<128><<<grid, 256, 0, stream>>>(dyp, xp, w, eps, alpha, n_rows, d, n_true, n_rows_dev, gather, dxp, part);
  else if (group == 256) rmsnorm_bwd_kernel<256><<<grid, 256, 0, stream>>>(dyp, xp, w, eps, alpha, n_rows, d, n_true, n_rows_dev, gather, dxp, part);
  else rmsnorm_bwd_kernel<512><<<grid, 256, 0, stream>>>(dyp, xp, w, eps, alpha, n_rows, d, n_true, n_rows_dev, gather, dxp, part);
  RP_LAUNCH_CHECK();
  return rp_reduce_splits(part, kRmsParts, group, group, dw, 1, stream_);
}

RP_API int rp_swiglu_fwd(const void* gl, long long n_rows, int F, void* u, void* stream_) {
  if (!gl || !u) return RP_EINVAL;
  if (n_rows < 0 || F <= 0) return RP_ESHAPE;
  const long long n = n_rows * F;
  if (n == 0) return RP_OK;
  swiglu_fwd_kernel<<<grid_for(n, 256), 256, 0, reinterpret_cast<cudaStream_t>(stream_)>>>(
      reinterpret_cast<const __nv_bfloat16*>(gl), n, F, reinterpret_cast<__nv_bfloat16*>(u));
  RP_LAUNCH_CHECK();
  return RP_OK;
}

RP_API int rp_swiglu_bwd(const void* du, const void* gl, long long n_rows, int F, void* dgl, void* stream_) {
  if (!du || !gl || !dgl) return RP_EINVAL;
  if (n_rows < 0 || F <= 0) return RP_ESHAPE;
  const long long n = n_rows * F;
  if (n == 0) return RP_OK;
  swiglu_bwd_kernel<<<grid_for(n, 256), 256, 0, reinterpret_cast<cudaStream_t>(stream_)>>>(
      reinterpret_cast<const __nv_bfloat16*>(du), reinterpret_cast<const __nv_bfloat16*>(gl), n, F,
      reinterpret_cast<__nv_bfloat16*>(dgl));
  RP_LAUNCH_CHECK();
  return RP_OK;
}
