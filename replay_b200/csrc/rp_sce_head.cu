// rp_sce_head.cu - scalable cross-entropy (SCE, arXiv 2409.18721) training head of the legacy SASRec.  Replaces
//   ScalableCrossEntropyLoss.__call__                  replay/models/nn/loss/sce.py:43-124
//   SasRec._compute_loss_scalable_ce                   replay/models/nn/sequential/sasrec/lightning.py:383-392
// and autograd's backward of it.  The item table is a detached copy in the reference (sasrec/model.py:374-381), so the
// head produces d_hc only.
//
// Forward, for every position t of the batch (hc row t = b * L + l, pad rows included):
//   draw      buckets [n_b, d] = randn(n_b, d_true) / d_true^0.25, or (mix_x) omega^T . hc with omega = randn(T, n_b) / d_true^0.25
//             (Philox normals keyed by seed + *rng_counter, or a caller-given draw), rounded to bf16;
//   select    top_x = top-k(buckets . hc^T + {0 | -inf for pad rows}, bs_x), top_y = top-k(buckets . table^T, bs_y), both with
//             rp_score_topk (exact, ties by ascending column);
//   bucket CE per bucket b and selected row t: logits x_t . table[Y_b] with label collisions at -inf plus the correct logit
//             c_t = x_t . table[y_t]; CE_bt = lse - c_t (fp32).  S = X_b . Y_b^T runs through batched rp_gemm in chunks of
//             buckets so the fp32 S stays inside a bounded workspace;
//   reduce    l_t = max over the buckets that selected t; loss = mean of l_t over the rows with l_t != 0 (NaN when none).
// Backward: only the winning slot(s) of a row carry gradient (ties split evenly, as torch's scatter_reduce amax backward);
// G = softmax * weight in bf16 in place of S, dX_b = G . Y_b (batched rp_gemm), then every row gathers its winners' dX rows
// plus (p_c - 1) * weight * table[y_t] in bucket order: no float atomics, bitwise reproducible.
#include <algorithm>
#include <cstdlib>

#include "rp_host.h"
#include "rp_gemm_desc.h"
#include "rp_philox.cuh"
#include "rp_sm90.cuh"

// stages of rp_sce_head_fwd (include/rp_b200.h)
#define RP_SCE_DRAW 1
#define RP_SCE_SELECT_X 2
#define RP_SCE_SELECT_Y 4
#define RP_SCE_BUCKET_CE 8
#define RP_SCE_ALL 15

extern "C" size_t rp_score_topk_workspace(int n_users, int n_items, int d, int K);
extern "C" int rp_score_topk(const void* hq, const void* table, const float* bias, const int32_t* seen_sorted, int S,
                             int n_users, int n_items, int d, int K, const int64_t* candidates, int64_t* out_ids,
                             float* out_scores, void* workspace, size_t workspace_bytes, void* stream);

namespace rp {

constexpr unsigned long long kSceSite = 0x5CEull << 40;   // Philox counter offset of the bucket draw
constexpr size_t kSceChunkBytes = 256ull << 20;            // fp32 S + dX of one chunk of buckets (RP_SCE_CHUNK_BYTES overrides)

struct SceArgs {
  const __nv_bfloat16* hc;
  const __nv_bfloat16* table;
  const int64_t* labels;
  const uint8_t* pad;
  const int32_t* n_rows;
  int cap, n_items, d, d_true, hd_valid, nb, bsx, bsy, mix;
  int bsxp, bsyp, nbp, chunk;
  unsigned long long seed;
  const unsigned long long* rng_counter;
  float* draw;
  int64_t* top_x;
  float* score_x;
  int64_t* top_y;
  float* loss_out;
  // workspace
  __nv_bfloat16* buckets;   // [nb, d]
  __nv_bfloat16* omega;     // [cap64, nbp] (mix_x)
  float* rowbias;           // [cap128]
  float* score_y;           // [nb, bsy]
  __nv_bfloat16* xb;        // [nb * bsxp, d]
  __nv_bfloat16* yb;        // [nb * bsyp, d]
  float* S;                 // [chunk * bsxp, bsyp]  (backward: bf16 G in place, pitch 2 * bsyp)
  float* dX;                // [chunk * bsxp, d]
  float* ce;                // [nb * bsx]  -1 = slot carries nothing
  float* lse;               // [nb * bsx]
  float* cc;                // [nb * bsx]  correct logit
  float* gc;                // [nb * bsx]  (p_c - 1) * weight
  int32_t* lab;             // [cap] label of a row that can carry loss, else -1
  uint32_t* maxkey;         // [cap] bits(max CE) + 1, 0 = not selected
  uint32_t* cnt;            // [cap] number of slots at the maximum
  int32_t* win;             // [cap] lowest slot at the maximum
  float* dacc;              // [cap, d]
  float* block_sums;        // [1024]
  float* inv_n;             // [1]
  unsigned int* ticket;
  void* topk_ws;
  size_t topk_ws_bytes;
};

__device__ __forceinline__ int pad_col(int j, int hd_valid) {
  if (hd_valid == 0) return j;
  const int slot = hd_valid <= 64 ? 64 : 128;
  return (j / hd_valid) * slot + j % hd_valid;
}

// rows that may carry loss: inside the batch, a real input position, label inside the catalog
__global__ void sce_prep_kernel(const SceArgs a) {
  const int n = *a.n_rows;
  const int cap128 = (a.cap + 127) / 128 * 128;
  for (int t = blockIdx.x * blockDim.x + threadIdx.x; t < cap128; t += gridDim.x * blockDim.x) {
    int y = -1;
    if (t < a.cap && t < n && a.pad[t]) {
      const int64_t l = a.labels[t];
      if (l >= 0 && l < a.n_items) y = (int)l;
    }
    a.rowbias[t] = y >= 0 ? 0.f : -INFINITY;
    if (t < a.cap) a.lab[t] = y;
  }
}

__global__ void sce_reset_kernel(const SceArgs a) {
  for (int t = blockIdx.x * blockDim.x + threadIdx.x; t < a.cap; t += gridDim.x * blockDim.x) {
    a.maxkey[t] = 0u;
    a.cnt[t] = 0u;
    a.win[t] = 0x7fffffff;
  }
}

// standard normals, two per Philox call (Box-Muller), keyed by (seed + *counter, site + pair index)
__global__ void sce_draw_kernel(const SceArgs a, long long n_elems) {
  const unsigned long long seed = a.seed + *a.rng_counter;
  for (long long p = blockIdx.x * (long long)blockDim.x + threadIdx.x; 2 * p < n_elems; p += (long long)gridDim.x * blockDim.x) {
    const uint4 r = philox4x32(seed, kSceSite + (unsigned long long)p);
    const float u1 = ((float)r.x + 1.f) * 2.3283064365386963e-10f;   // (0, 1]
    const float u2 = (float)r.y * 2.3283064365386963e-10f;
    const float rad = sqrtf(-2.f * logf(u1));
    float s, c;
    sincospif(2.f * u2, &s, &c);
    a.draw[2 * p] = rad * c;
    if (2 * p + 1 < n_elems) a.draw[2 * p + 1] = rad * s;
  }
}

// draw -> bf16 bucket matrix (true columns scattered into the feature slots) or bf16 omega (rows beyond the batch zero)
__global__ void sce_bucket_kernel(const SceArgs a, float scale) {
  if (!a.mix) {
    const long long total = (long long)a.nb * a.d;
    for (long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x; e < total; e += (long long)gridDim.x * blockDim.x)
      a.buckets[e] = __float2bfloat16(0.f);
    __syncthreads();   // one block (launched with a single CTA in this mode)
    for (long long e = threadIdx.x; e < (long long)a.nb * a.d_true; e += blockDim.x) {
      const int b = (int)(e / a.d_true), j = (int)(e % a.d_true);
      a.buckets[(size_t)b * a.d + pad_col(j, a.hd_valid)] = __float2bfloat16(a.draw[e] * scale);
    }
    return;
  }
  const int n = *a.n_rows;
  const int cap64 = (a.cap + 63) / 64 * 64;
  const long long total = (long long)cap64 * a.nbp;
  for (long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x; e < total; e += (long long)gridDim.x * blockDim.x) {
    const int t = (int)(e / a.nbp), b = (int)(e % a.nbp);
    const float v = (t < n && b < a.nb) ? a.draw[(size_t)t * a.nb + b] * scale : 0.f;
    a.omega[e] = __float2bfloat16(v);
  }
}

__global__ void sce_gather_kernel(const SceArgs a) {
  const int lane = threadIdx.x & 31, wpb = blockDim.x >> 5;
  const long long rows_x = (long long)a.nb * a.bsxp, rows = rows_x + (long long)a.nb * a.bsyp;
  const int nvec = a.d / 8;
  for (long long r = blockIdx.x * (long long)wpb + (threadIdx.x >> 5); r < rows; r += (long long)gridDim.x * wpb) {
    const uint4* src = nullptr;
    uint4* dst;
    if (r < rows_x) {
      const int b = (int)(r / a.bsxp), i = (int)(r % a.bsxp);
      dst = reinterpret_cast<uint4*>(a.xb + r * a.d);
      if (i < a.bsx) {
        const size_t s = (size_t)b * a.bsx + i;
        const long long t = a.top_x[s];
        if (a.score_x[s] > -INFINITY && t >= 0 && t < a.cap) src = reinterpret_cast<const uint4*>(a.hc + t * a.d);
      }
    } else {
      const long long q = r - rows_x;
      const int b = (int)(q / a.bsyp), j = (int)(q % a.bsyp);
      dst = reinterpret_cast<uint4*>(a.yb + q * a.d);
      if (j < a.bsy) src = reinterpret_cast<const uint4*>(a.table + a.top_y[(size_t)b * a.bsy + j] * a.d);
    }
    for (int c = lane; c < nvec; c += 32) dst[c] = src ? src[c] : make_uint4(0u, 0u, 0u, 0u);
  }
}

template <int D>
__device__ __forceinline__ float sce_dot(const __nv_bfloat16* __restrict__ x, const __nv_bfloat16* __restrict__ w, int lane) {
  float acc = 0.f;
#pragma unroll
  for (int k = 0; k < D / 64; ++k) {
    const float2 u = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(x + k * 64 + lane * 2));
    const float2 v = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(w + k * 64 + lane * 2));
    acc = fmaf(u.x, v.x, fmaf(u.y, v.y, acc));
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  return acc;
}

__device__ __forceinline__ int slot_row(const SceArgs& a, int b, int i) {
  const long long t = a.top_x[(size_t)b * a.bsx + i];
  if (!(a.score_x[(size_t)b * a.bsx + i] > -INFINITY) || t < 0 || t >= a.cap) return -1;
  return a.lab[t] >= 0 ? (int)t : -1;
}

// one warp per slot of buckets [b0, b0 + nc): correct logit, collision mask, lse, CE
template <int D>
__global__ void sce_row_fwd_kernel(const SceArgs a, int b0, int nc) {
  const int lane = threadIdx.x & 31, wpb = blockDim.x >> 5;
  const long long n_slots = (long long)nc * a.bsx;
  for (long long r = blockIdx.x * (long long)wpb + (threadIdx.x >> 5); r < n_slots; r += (long long)gridDim.x * wpb) {
    const int bl = (int)(r / a.bsx), i = (int)(r % a.bsx), b = b0 + bl;
    const size_t slot = (size_t)b * a.bsx + i;
    const int t = slot_row(a, b, i);
    if (t < 0) {
      if (lane == 0) a.ce[slot] = -1.f;
      continue;
    }
    const int y = a.lab[t];
    const float c = sce_dot<D>(a.hc + (size_t)t * D, a.table + (size_t)y * D, lane);
    const float* srow = a.S + ((size_t)bl * a.bsxp + i) * a.bsyp;
    const int64_t* ty = a.top_y + (size_t)b * a.bsy;
    float m = c;
    for (int j = lane; j < a.bsy; j += 32)
      if (ty[j] != (int64_t)y) m = fmaxf(m, srow[j]);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    float s = 0.f;
    for (int j = lane; j < a.bsy; j += 32)
      if (ty[j] != (int64_t)y) s += __expf(srow[j] - m);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (lane == 0) {
      s += __expf(c - m);
      const float lse = m + logf(s);
      a.ce[slot] = fmaxf(lse - c, 0.f);
      a.lse[slot] = lse;
      a.cc[slot] = c;
    }
  }
}

// per row: the largest CE over the slots that selected it (integer max of the bits: CE >= 0), then the slots at it
__global__ void sce_amax_kernel(const SceArgs a, int pass) {
  const long long n_slots = (long long)a.nb * a.bsx;
  for (long long s = blockIdx.x * (long long)blockDim.x + threadIdx.x; s < n_slots; s += (long long)gridDim.x * blockDim.x) {
    const float ce = a.ce[s];
    if (ce < 0.f) continue;
    const int t = (int)a.top_x[s];
    const uint32_t key = __float_as_uint(ce) + 1u;
    if (pass == 0) {
      atomicMax(a.maxkey + t, key);
    } else if (a.maxkey[t] == key) {
      atomicAdd(a.cnt + t, 1u);
      atomicMin(a.win + t, (int)s);
    }
  }
}

// loss = mean of the per-row maxima that are != 0; fixed-order reduction (block partials, the last block adds them)
__global__ void sce_loss_kernel(const SceArgs a) {
  float sum = 0.f;
  int n = 0;
  for (int t = blockIdx.x * blockDim.x + threadIdx.x; t < a.cap; t += gridDim.x * blockDim.x) {
    const uint32_t k = a.maxkey[t];
    if (k > 1u) {
      sum += __uint_as_float(k - 1u);
      ++n;
    }
  }
  __shared__ float red[32];
  __shared__ int redn[32];
  __shared__ bool last;
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    sum += __shfl_xor_sync(0xffffffffu, sum, o);
    n += __shfl_xor_sync(0xffffffffu, n, o);
  }
  if (lane == 0) {
    red[w] = sum;
    redn[w] = n;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    float s2 = 0.f;
    int n2 = 0;
    for (int i = 0; i < (int)(blockDim.x >> 5); ++i) {
      s2 += red[i];
      n2 += redn[i];
    }
    a.block_sums[blockIdx.x] = s2;
    reinterpret_cast<int*>(a.block_sums)[512 + blockIdx.x] = n2;
    __threadfence();
    last = (atomicAdd(a.ticket, 1u) == gridDim.x - 1);
  }
  __syncthreads();
  if (last && threadIdx.x == 0) {
    __threadfence();
    float s3 = 0.f;
    int n3 = 0;
    for (int i = 0; i < (int)gridDim.x; ++i) {
      s3 += reinterpret_cast<volatile float*>(a.block_sums)[i];
      n3 += reinterpret_cast<volatile int*>(a.block_sums)[512 + i];
    }
    const float inv = n3 > 0 ? __frcp_rn((float)n3) : 0.f;   // 1 / count rounded once (fast-math 1.f / x is approximate)
    a.loss_out[0] = n3 > 0 ? s3 * inv : __int_as_float(0x7fc00000);   // mean of nothing: NaN, as torch.mean
    a.loss_out[1] = inv;
    a.inv_n[0] = inv;
    *a.ticket = 0u;
  }
}

// backward row pass, one warp per slot: G = softmax * weight (bf16, in place of the slot's S row), gc = (p_c - 1) * weight
__global__ void sce_row_bwd_kernel(const SceArgs a, int b0, int nc) {
  const int lane = threadIdx.x & 31, wpb = blockDim.x >> 5;
  const long long n_slots = (long long)nc * a.bsx;
  for (long long r = blockIdx.x * (long long)wpb + (threadIdx.x >> 5); r < n_slots; r += (long long)gridDim.x * wpb) {
    const int bl = (int)(r / a.bsx), i = (int)(r % a.bsx), b = b0 + bl;
    const size_t slot = (size_t)b * a.bsx + i;
    const int t = slot_row(a, b, i);
    float wgt = 0.f;
    if (t >= 0) {
      const uint32_t k = a.maxkey[t];
      if (k > 1u && __float_as_uint(a.ce[slot]) + 1u == k) wgt = a.inv_n[0] / (float)a.cnt[t];
    }
    float* srow = a.S + ((size_t)bl * a.bsxp + i) * a.bsyp;
    __nv_bfloat16* grow = reinterpret_cast<__nv_bfloat16*>(srow);
    if (wgt == 0.f) {
      for (int j = lane; j < a.bsyp; j += 32) grow[j] = __float2bfloat16(0.f);
      if (lane == 0) a.gc[slot] = 0.f;
      continue;
    }
    const int y = a.lab[t];
    const float lse = a.lse[slot];
    const int64_t* ty = a.top_y + (size_t)b * a.bsy;
    float v[32];   // bs_y <= 1024: the whole fp32 row is read before its bf16 image overwrites it
#pragma unroll
    for (int q = 0; q < 32; ++q) {
      const int j = lane + 32 * q;
      v[q] = (j < a.bsy && ty[j] != (int64_t)y) ? __expf(srow[j] - lse) * wgt : 0.f;
    }
    __syncwarp();
#pragma unroll
    for (int q = 0; q < 32; ++q) {
      const int j = lane + 32 * q;
      if (j < a.bsyp) grow[j] = __float2bfloat16(v[q]);
    }
    if (lane == 0) a.gc[slot] = (__expf(a.cc[slot] - lse) - 1.f) * wgt;
  }
}

// one warp per row: dacc[t] += dX[winner slot] + gc * table[y_t] for the winners inside buckets [b0, b0 + nc), in bucket order
template <int D>
__global__ void sce_collect_kernel(const SceArgs a, int b0, int nc) {
  const int lane = threadIdx.x & 31, wpb = blockDim.x >> 5;
  for (int t = blockIdx.x * wpb + (threadIdx.x >> 5); t < a.cap; t += gridDim.x * wpb) {
    const uint32_t key = a.maxkey[t];
    if (key <= 1u) continue;
    const int n_win = (int)a.cnt[t];
    if (n_win == 1) {
      const int b = a.win[t] / a.bsx;
      if (b < b0 || b >= b0 + nc) continue;
    }
    float acc[D / 32];
    float* dr = a.dacc + (size_t)t * D;
#pragma unroll
    for (int k = 0; k < D / 64; ++k) {
      const float2 o = *reinterpret_cast<const float2*>(dr + k * 64 + lane * 2);
      acc[2 * k] = o.x;
      acc[2 * k + 1] = o.y;
    }
    const __nv_bfloat16* wy = a.table + (size_t)a.lab[t] * D;
    auto add = [&](int b, int i) {
      const float* xr = a.dX + ((size_t)(b - b0) * a.bsxp + i) * D;
      const float g = a.gc[(size_t)b * a.bsx + i];
#pragma unroll
      for (int k = 0; k < D / 64; ++k) {
        const float2 x = *reinterpret_cast<const float2*>(xr + k * 64 + lane * 2);
        const float2 w = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(wy + k * 64 + lane * 2));
        acc[2 * k] += fmaf(g, w.x, x.x);
        acc[2 * k + 1] += fmaf(g, w.y, x.y);
      }
    };
    if (n_win == 1) {
      const int s = a.win[t];
      add(s / a.bsx, s % a.bsx);
    } else {
      // tied maxima (bit-equal CE in several buckets): scan each bucket of the chunk for the row, in bucket order
      for (int b = b0; b < b0 + nc; ++b) {
        for (int i0 = 0; i0 < a.bsx; i0 += 32) {
          const int i = i0 + lane;
          const size_t s = (size_t)b * a.bsx + i;
          const bool hit = i < a.bsx && a.top_x[s] == (int64_t)t && a.ce[s] >= 0.f && __float_as_uint(a.ce[s]) + 1u == key;
          const unsigned m = __ballot_sync(0xffffffffu, hit);
          if (m) {
            add(b, i0 + __ffs(m) - 1);
            break;   // a bucket selects a row at most once
          }
        }
      }
    }
#pragma unroll
    for (int k = 0; k < D / 64; ++k) *reinterpret_cast<float2*>(dr + k * 64 + lane * 2) = make_float2(acc[2 * k], acc[2 * k + 1]);
  }
}

__global__ void sce_to_bf16_kernel(const float* __restrict__ src, __nv_bfloat16* __restrict__ dst, long long n) {
  for (long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x; 2 * e < n; e += (long long)gridDim.x * blockDim.x) {
    const float2 v = *reinterpret_cast<const float2*>(src + 2 * e);
    *reinterpret_cast<uint32_t*>(dst + 2 * e) = pack_bf16(v.x, v.y);
  }
}

}  // namespace rp

using namespace rp;

struct rp_sce_desc {
  const void* hc; const void* table; const int64_t* labels; const uint8_t* pad_mask; const int32_t* n_rows;
  int capacity, n_items, d, d_true, hd_valid;
  int n_buckets, bucket_size_x, bucket_size_y, mix_x;
  unsigned long long seed; const unsigned long long* rng_counter; int draw_given;
  float* draw; int64_t* top_x; float* score_x; int64_t* top_y;
  float* loss_out;
  void* workspace; size_t workspace_bytes;
};

static size_t ru(size_t x, size_t m) { return (x + m - 1) / m * m; }

static size_t sce_layout(const rp_sce_desc* s, SceArgs* a) {
  const size_t cap = (size_t)s->capacity, nb = (size_t)s->n_buckets, d = (size_t)s->d;
  const size_t bsx = (size_t)s->bucket_size_x, bsy = (size_t)s->bucket_size_y;
  const size_t bsxp = ru(bsx, 64), bsyp = ru(bsy, 64), nbp = ru(nb, 64);
  const size_t per_bucket = bsxp * bsyp * 4 + bsxp * d * 4;
  const char* env = getenv("RP_SCE_CHUNK_BYTES");   // read per call: the workspace query and the launches must agree
  const size_t budget = env ? (size_t)atoll(env) : kSceChunkBytes;
  size_t chunk = budget / per_bucket;
  chunk = chunk < 1 ? 1 : (chunk > nb ? nb : chunk);
  const size_t topk_ws = std::max(rp_score_topk_workspace((int)nb, (int)cap, (int)d, (int)bsx),
                                  rp_score_topk_workspace((int)nb, s->n_items, (int)d, (int)bsy));
  size_t off = 0;
  auto take = [&](size_t bytes) { const size_t o = off; off = ru(off + bytes, 256); return o; };
  const size_t o_buck = take(nb * d * 2);
  const size_t o_omega = s->mix_x ? take(ru(cap, 64) * nbp * 2) : 0;
  const size_t o_rb = take(ru(cap, 128) * 4), o_sy = take(nb * bsy * 4);
  const size_t o_xb = take(nb * bsxp * d * 2), o_yb = take(nb * bsyp * d * 2);
  const size_t o_S = take(chunk * bsxp * bsyp * 4), o_dX = take(chunk * bsxp * d * 4);
  const size_t o_ce = take(nb * bsx * 4), o_lse = take(nb * bsx * 4), o_cc = take(nb * bsx * 4), o_gc = take(nb * bsx * 4);
  const size_t o_lab = take(cap * 4), o_mk = take(cap * 4), o_cnt = take(cap * 4), o_win = take(cap * 4);
  const size_t o_dacc = take(cap * d * 4);
  const size_t o_bs = take(1024 * 4), o_inv = take(64), o_tk = take(64);
  const size_t o_tws = take(topk_ws);
  if (a) {
    uint8_t* w = reinterpret_cast<uint8_t*>(s->workspace);
    a->buckets = reinterpret_cast<__nv_bfloat16*>(w + o_buck);
    a->omega = s->mix_x ? reinterpret_cast<__nv_bfloat16*>(w + o_omega) : nullptr;
    a->rowbias = reinterpret_cast<float*>(w + o_rb);
    a->score_y = reinterpret_cast<float*>(w + o_sy);
    a->xb = reinterpret_cast<__nv_bfloat16*>(w + o_xb);
    a->yb = reinterpret_cast<__nv_bfloat16*>(w + o_yb);
    a->S = reinterpret_cast<float*>(w + o_S);
    a->dX = reinterpret_cast<float*>(w + o_dX);
    a->ce = reinterpret_cast<float*>(w + o_ce);
    a->lse = reinterpret_cast<float*>(w + o_lse);
    a->cc = reinterpret_cast<float*>(w + o_cc);
    a->gc = reinterpret_cast<float*>(w + o_gc);
    a->lab = reinterpret_cast<int32_t*>(w + o_lab);
    a->maxkey = reinterpret_cast<uint32_t*>(w + o_mk);
    a->cnt = reinterpret_cast<uint32_t*>(w + o_cnt);
    a->win = reinterpret_cast<int32_t*>(w + o_win);
    a->dacc = reinterpret_cast<float*>(w + o_dacc);
    a->block_sums = reinterpret_cast<float*>(w + o_bs);
    a->inv_n = reinterpret_cast<float*>(w + o_inv);
    a->ticket = reinterpret_cast<unsigned int*>(w + o_tk);
    a->topk_ws = w + o_tws;
    a->topk_ws_bytes = topk_ws;
    a->bsxp = (int)bsxp;
    a->bsyp = (int)bsyp;
    a->nbp = (int)nbp;
    a->chunk = (int)chunk;
  }
  return off;
}

static bool sce_shape_ok(const rp_sce_desc* s) {
  if (s->capacity <= 0 || s->n_items <= 0 || s->n_buckets <= 0) return false;
  if (s->d != 64 && s->d != 128 && s->d != 256 && s->d != 512) return false;
  if (s->hd_valid < 0 || s->hd_valid > 128 || (s->hd_valid > 0 && s->d % (s->hd_valid <= 64 ? 64 : 128))) return false;
  if (s->d_true != feat_count(s->d, s->hd_valid)) return false;   // pad_col scatters exactly d_true columns into the slots
  if (s->bucket_size_x < 1 || s->bucket_size_x > 1024 || s->bucket_size_x > s->capacity) return false;
  if (s->bucket_size_y < 1 || s->bucket_size_y > 1024 || s->bucket_size_y > s->n_items) return false;
  return true;
}

static int sce_args(const rp_sce_desc* s, SceArgs* a) {
  if (!s || !s->hc || !s->table || !s->labels || !s->pad_mask || !s->n_rows || !s->rng_counter || !s->draw || !s->top_x ||
      !s->score_x || !s->top_y || !s->loss_out || !s->workspace)
    return RP_EINVAL;
  if (!sce_shape_ok(s)) return RP_ESHAPE;
  if (s->workspace_bytes < sce_layout(s, nullptr)) return RP_EWORKSPACE;
  a->hc = reinterpret_cast<const __nv_bfloat16*>(s->hc);
  a->table = reinterpret_cast<const __nv_bfloat16*>(s->table);
  a->labels = s->labels; a->pad = s->pad_mask; a->n_rows = s->n_rows;
  a->cap = s->capacity; a->n_items = s->n_items; a->d = s->d; a->d_true = s->d_true; a->hd_valid = s->hd_valid;
  a->nb = s->n_buckets; a->bsx = s->bucket_size_x; a->bsy = s->bucket_size_y; a->mix = s->mix_x ? 1 : 0;
  a->seed = s->seed; a->rng_counter = s->rng_counter;
  a->draw = s->draw; a->top_x = s->top_x; a->score_x = s->score_x; a->top_y = s->top_y; a->loss_out = s->loss_out;
  sce_layout(s, a);
  return RP_OK;
}

#define RP_DISPATCH_SCE(d, CALL)                       \
  switch (d) {                                         \
    case 64: { constexpr int D = 64; CALL; } break;    \
    case 128: { constexpr int D = 128; CALL; } break;  \
    case 256: { constexpr int D = 256; CALL; } break;  \
    default: { constexpr int D = 512; CALL; } break;   \
  }

// S[b] = X_b . Y_b^T for the buckets [b0, b0 + nc) of a chunk (fp32, pitch bsyp)
static int sce_scores(const SceArgs& a, int b0, int nc, void* stream) {
  rp_gemm_desc g = rp_gemm_default();
  g.A = a.xb; g.a_rows = (long long)a.nb * a.bsxp; g.a_cols = a.d; g.lda = a.d;
  g.B = a.yb; g.b_rows = (long long)a.nb * a.bsyp; g.b_cols = a.d; g.ldb = a.d;
  g.M = a.bsx; g.N = a.bsy; g.K = a.d; g.batch = nc;
  g.a_r0 = b0 * a.bsxp; g.a_ro = a.bsxp;
  g.b_r0 = b0 * a.bsyp; g.b_ro = a.bsyp;
  g.C = a.S; g.ldc = a.bsyp; g.c_oo = (long long)a.bsxp * a.bsyp; g.out_mode = 2;
  return rp_gemm(&g, stream);
}

RP_API size_t rp_sce_head_workspace(int capacity, int n_items, int d, int n_buckets, int bucket_size_x, int bucket_size_y,
                                    int mix_x) {
  rp_sce_desc s;
  memset(&s, 0, sizeof(s));
  s.capacity = capacity; s.n_items = n_items; s.d = d; s.d_true = d; s.n_buckets = n_buckets;
  s.bucket_size_x = bucket_size_x; s.bucket_size_y = bucket_size_y; s.mix_x = mix_x;
  if (!sce_shape_ok(&s)) return 0;
  return sce_layout(&s, nullptr);
}

RP_API int rp_sce_head_fwd(const rp_sce_desc* s, int stages, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  SceArgs a;
  int rc = sce_args(s, &a);
  if (rc != RP_OK) return rc;
  if (stages & ~RP_SCE_ALL) return RP_EINVAL;
  const int blocks = sm_count() * 4;
  if (stages & RP_SCE_DRAW) {
    sce_prep_kernel<<<(a.cap + 128 + 255) / 256, 256, 0, stream>>>(a);
    RP_LAUNCH_CHECK();
    const long long n_draw = a.mix ? (long long)a.cap * a.nb : (long long)a.nb * a.d_true;
    if (!s->draw_given) {
      sce_draw_kernel<<<(unsigned)std::min<long long>((n_draw / 2 + 255) / 256 + 1, blocks), 256, 0, stream>>>(a, n_draw);
      RP_LAUNCH_CHECK();
    }
    const float scale = 1.f / sqrtf(sqrtf((float)a.d_true));
    sce_bucket_kernel<<<a.mix ? blocks : 1, 256, 0, stream>>>(a, scale);
    RP_LAUNCH_CHECK();
    if (a.mix) {   // buckets = omega^T . hc over the rows of the batch (k_limit: *n_rows, omega is zero beyond)
      rp_gemm_desc g = rp_gemm_default();
      g.A = a.omega; g.a_rows = (a.cap + 63) / 64 * 64; g.a_cols = a.nbp; g.lda = a.nbp; g.a_mn = 1;
      g.B = a.hc; g.b_rows = a.cap; g.b_cols = a.d; g.ldb = a.d; g.b_mn = 1;
      g.M = a.nb; g.N = a.d; g.K = a.cap;
      g.C = a.buckets; g.ldc = a.d; g.out_mode = 0;
      g.k_limit_dev = a.n_rows;
      if ((rc = rp_gemm(&g, stream_)) != RP_OK) return rc;
    }
  }
  if (stages & RP_SCE_SELECT_X) {
    rc = rp_score_topk(a.buckets, a.hc, a.rowbias, nullptr, 0, a.nb, a.cap, a.d, a.bsx, nullptr, a.top_x, a.score_x,
                       a.topk_ws, a.topk_ws_bytes, stream_);
    if (rc != RP_OK) return rc;
  }
  if (stages & RP_SCE_SELECT_Y) {
    rc = rp_score_topk(a.buckets, a.table, nullptr, nullptr, 0, a.nb, a.n_items, a.d, a.bsy, nullptr, a.top_y, a.score_y,
                       a.topk_ws, a.topk_ws_bytes, stream_);
    if (rc != RP_OK) return rc;
  }
  if (stages & RP_SCE_BUCKET_CE) {
    const long long rows = (long long)a.nb * (a.bsxp + a.bsyp);
    sce_gather_kernel<<<(unsigned)std::min<long long>((rows + 7) / 8, blocks), 256, 0, stream>>>(a);
    RP_LAUNCH_CHECK();
    sce_reset_kernel<<<(a.cap + 255) / 256, 256, 0, stream>>>(a);
    RP_LAUNCH_CHECK();
    for (int b0 = 0; b0 < a.nb; b0 += a.chunk) {
      const int nc = std::min(a.chunk, a.nb - b0);
      if ((rc = sce_scores(a, b0, nc, stream_)) != RP_OK) return rc;
      RP_DISPATCH_SCE(a.d, (sce_row_fwd_kernel<D><<<blocks, 256, 0, stream>>>(a, b0, nc)));
      RP_LAUNCH_CHECK();
    }
    sce_amax_kernel<<<blocks, 256, 0, stream>>>(a, 0);
    RP_LAUNCH_CHECK();
    sce_amax_kernel<<<blocks, 256, 0, stream>>>(a, 1);
    RP_LAUNCH_CHECK();
    RP_CUDA_CHECK(cudaMemsetAsync(a.ticket, 0, 64, stream));
    sce_loss_kernel<<<std::min(blocks, 512), 256, 0, stream>>>(a);
    RP_LAUNCH_CHECK();
  }
  return RP_OK;
}

RP_API int rp_sce_head_bwd(const rp_sce_desc* s, void* d_hc, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  SceArgs a;
  int rc = sce_args(s, &a);
  if (rc != RP_OK) return rc;
  if (!d_hc) return RP_EINVAL;
  const int blocks = sm_count() * 4;
  RP_CUDA_CHECK(cudaMemsetAsync(a.dacc, 0, (size_t)a.cap * a.d * 4, stream));
  for (int b0 = 0; b0 < a.nb; b0 += a.chunk) {
    const int nc = std::min(a.chunk, a.nb - b0);
    if ((rc = sce_scores(a, b0, nc, stream_)) != RP_OK) return rc;
    sce_row_bwd_kernel<<<blocks, 256, 0, stream>>>(a, b0, nc);
    RP_LAUNCH_CHECK();
    // dX_b = G_b . Y_b  (G bf16 in place of S: pitch 2 * bsyp elements; Y_b read MN-major)
    rp_gemm_desc g = rp_gemm_default();
    g.A = a.S; g.a_rows = (long long)a.chunk * a.bsxp; g.a_cols = a.bsyp; g.lda = 2ll * a.bsyp;
    g.B = a.yb; g.b_rows = (long long)a.nb * a.bsyp; g.b_cols = a.d; g.ldb = a.d; g.b_mn = 1;
    g.M = a.bsx; g.N = a.d; g.K = a.bsyp; g.batch = nc;
    g.a_ro = a.bsxp;
    g.b_r0 = b0 * a.bsyp; g.b_ro = a.bsyp;
    g.C = a.dX; g.ldc = a.d; g.c_oo = (long long)a.bsxp * a.d; g.out_mode = 2;
    if ((rc = rp_gemm(&g, stream_)) != RP_OK) return rc;
    RP_DISPATCH_SCE(a.d, (sce_collect_kernel<D><<<blocks, 256, 0, stream>>>(a, b0, nc)));
    RP_LAUNCH_CHECK();
  }
  const long long n = (long long)a.cap * a.d;
  sce_to_bf16_kernel<<<(unsigned)std::min<long long>((n / 2 + 255) / 256, blocks), 256, 0, stream>>>(
      a.dacc, reinterpret_cast<__nv_bfloat16*>(d_hc), n);
  RP_LAUNCH_CHECK();
  return RP_OK;
}
