// rp_block_fused.cu - the fused one-pass kernels of a SASRec transformer block on wgmma (training and inference).
// They share one pattern: the d x d weights stay resident in shared memory, a persistent CTA walks 128-token tiles (TMA),
// each of the two warpgroups owns 64 rows of the tile, every GEMM result stays in registers (accumulator layout) where the
// LayerNorm / ReLU / dropout work runs, and its bf16 result is the register A operand of the next wgmma (rp_sm90.cuh,
// "row fragments").  d in {64, 128}.
#include "rp_host.h"
#include "rp_philox.cuh"
#include "rp_sm90.cuh"

// ==================================================================================================================
// Before the attention (training and inference):
//
//   rp_ln_qkv_fused      q_in = LayerNorm1(x) ;  Q = q_in Wq^T + bq ;  [K | V] = x Wkv^T + bkv            (one pass, x read once)
//   rp_pre_attn_bwd      dq_in = dQ Wq + dh ;  t = LayerNorm1-backward(dq_in) ;  dx = [dK | dV] Wkv + t     (one pass)
//
// Replaces  attention_layernorms[i] + the packed in-projection of torch.nn.MultiheadAttention(query = LN(x), key = value = x)
//   replay/nn/sequential/sasrec/transformer.py:99-106 ; replay/models/nn/sequential/sasrec/model.py:434-435
// and autograd's backward of both; every activation tile is read once and written once.  LayerNorm row statistics come from
// the four threads of a quad.

namespace rp {

static constexpr int kBlockThreads = 256;   // two warpgroups: rows [0, 64) / [64, 128) of the token tile

// dropout row key of row r: its token (packed rows) or the row itself
__device__ __forceinline__ unsigned long long row_token(const int32_t* row_tok, int r, int n_rows) {
  return (unsigned long long)(row_tok && r < n_rows ? row_tok[r] : r);
}

struct LnQkvParams {
  const float* ln_w;
  const float* ln_b;
  const float* b_in;          // [3d] packed in_proj_bias (q | k | v)
  float eps;
  int T;
  int hd_valid;               // > 0: padded feature slots (rp_sm90.cuh feat_valid): statistics over the real features only
  __nv_bfloat16* q_in;        // [T, d]   LayerNorm output (residual of the block, saved for the backward)
  __nv_bfloat16* Q;           // [T, d]
  __nv_bfloat16* KV;          // [T, 2d]
  float* mean_out;            // [T] or null
  float* rstd_out;
  int kv_only;                // predict, final block: only [K | V] = x Wkv^T + bkv (no LayerNorm, no Q: those run on the B last rows)
  const int32_t* n_rows_dev;  // packed rows: the row count lives on the device (<= T, which sizes the grid and the maps), or null
};

// acc + bias (columns c0 + fragment column) -> packed bf16
template <int R>
__device__ __forceinline__ void frag_bias_pack(const float (&acc)[R], const float* bias, uint32_t (&pk)[R / 2]) {
  const int fc = frag_col(threadIdx.x & 127);
#pragma unroll
  for (int j = 0; j < R / 4; ++j) {
    const float b0 = bias[8 * j + fc], b1 = bias[8 * j + fc + 1];
    pk[2 * j] = pack_bf16(acc[4 * j] + b0, acc[4 * j + 1] + b1);
    pk[2 * j + 1] = pack_bf16(acc[4 * j + 2] + b0, acc[4 * j + 3] + b1);
  }
}

template <int KCH>
__global__ void __launch_bounds__(kBlockThreads, 1)
ln_qkv_fused_kernel(const __grid_constant__ CUtensorMap tmX, const __grid_constant__ CUtensorMap tmWq,
                    const __grid_constant__ CUtensorMap tmWkv, const LnQkvParams p) {
  constexpr int D = KCH * 64, R = D / 2;
  constexpr int WQ_BYTES = KCH * D * 128;        // [D x D] as KCH chunks of [D rows x 64]
  constexpr int WKV_BYTES = KCH * 2 * D * 128;   // [2D x D]
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sWq = smem;
  uint8_t* sWkv = smem + WQ_BYTES;
  uint8_t* sX = smem + WQ_BYTES + WKV_BYTES;     // [128 x D]: KCH chunks of 16 KB
  __shared__ uint64_t bar_w, bar_x;
  __shared__ __align__(16) float s_lnw[D], s_lnb[D], s_bias[3 * D];

  const int T = p.n_rows_dev ? *p.n_rows_dev : p.T;   // rows [T, p.T) of a packed batch are stale: never stored nor summed
  const int n_tiles = (T + 127) / 128;
  const int my_tiles = n_tiles > (int)blockIdx.x ? (n_tiles - 1 - (int)blockIdx.x) / (int)gridDim.x + 1 : 0;
  auto load_x = [&](int it) {
    const int t = (int)blockIdx.x + it * (int)gridDim.x;
    mbar_arrive_expect_tx(&bar_x, KCH * 16384);
    for (int kc = 0; kc < KCH; ++kc) tma_load_2d(sX + kc * 16384, &tmX, &bar_x, kc * 64, t * 128);
  };
  if (threadIdx.x == 0) {
    mbar_init(&bar_w, 1);
    mbar_init(&bar_x, 1);
    fence_barrier_init();
    mbar_arrive_expect_tx(&bar_w, WQ_BYTES + WKV_BYTES);
    for (int kc = 0; kc < KCH; ++kc) {
      tma_load_2d(sWq + kc * (D * 128), &tmWq, &bar_w, kc * 64, 0);
      tma_load_2d(sWkv + kc * (2 * D * 128), &tmWkv, &bar_w, kc * 64, 0);
    }
    if (my_tiles > 0) load_x(0);
  }
  for (int i = threadIdx.x; i < 3 * D; i += kBlockThreads) {
    if (i < D && !p.kv_only) {
      s_lnw[i] = p.ln_w[i];
      s_lnb[i] = p.ln_b[i];
    }
    s_bias[i] = p.b_in[i];
  }
  __syncthreads();
  const int wg = threadIdx.x >> 7, t = threadIdx.x & 127;
  const int fr = frag_row(t), fc = frag_col(t);
  const uint32_t aX = smem_u32(sX) + wg * 8192;
  const float inv_d = 1.f / (float)feat_count(D, p.hd_valid);   // padded columns are zero: sums need no mask
  mbar_wait(&bar_w, 0);
  for (int it = 0; it < my_tiles; ++it) {
    const int tile = (int)blockIdx.x + it * (int)gridDim.x;
    const int ra = tile * 128 + 64 * wg + fr;   // global rows ra, ra + 8 of this thread
    mbar_wait(&bar_x, it & 1);
    // ---- [K | V] = x . Wkv^T + bkv, one d-wide half at a time
#pragma unroll 1
    for (int hv = 0; hv < 2; ++hv) {
      float acc[R];
      uint32_t pk[R / 2];
      wg_gemm_ss_wt<D, KCH>(acc, aX, smem_u32(sWkv) + hv * D * 128, 2 * D * 128);
      frag_bias_pack(acc, s_bias + D + hv * D, pk);
      frag_store_bf16(pk, p.KV + hv * D, 2 * D, ra, T);
    }
    float xv[R];
    if (!p.kv_only) frag_load_tile(sX, 64 * wg + fr, xv);
    named_bar_sync(1, kBlockThreads);   // the x tile has been read
    if (threadIdx.x == 0 && it + 1 < my_tiles) load_x(it + 1);
    if (p.kv_only) continue;
    // ---- q_in = LayerNorm(x), rows ra (h = 0) and ra + 8 (h = 1)
    float mean[2], rstd[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      float sum = 0.f, sq = 0.f;
#pragma unroll
      for (int j = 0; j < R / 4; ++j)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const float x = xv[4 * j + 2 * h + e];
          sum += x;
          sq = fmaf(x, x, sq);
        }
      sum = quad_sum(sum);
      sq = quad_sum(sq);
      mean[h] = sum * inv_d;
      const float var = fmaxf(sq * inv_d - mean[h] * mean[h], 0.f);
      rstd[h] = rsqrtf(var + p.eps);
    }
    uint32_t pq[R / 2];
#pragma unroll
    for (int j = 0; j < R / 4; ++j)
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int c = 8 * j + fc;
        pq[2 * j + h] = pack_bf16((xv[4 * j + 2 * h] - mean[h]) * rstd[h] * s_lnw[c] + s_lnb[c],
                                  (xv[4 * j + 2 * h + 1] - mean[h]) * rstd[h] * s_lnw[c + 1] + s_lnb[c + 1]);
      }
    frag_store_bf16(pq, p.q_in, D, ra, T);
    if (fc == 0 && p.mean_out) {
#pragma unroll
      for (int h = 0; h < 2; ++h)
        if (ra + 8 * h < T) {
          p.mean_out[ra + 8 * h] = mean[h];
          p.rstd_out[ra + 8 * h] = rstd[h];
        }
    }
    // ---- Q = q_in . Wq^T + bq  (the bf16 q_in as the register A operand)
    float acc[R];
    uint32_t pk[R / 2];
    wg_gemm_rs_wt<D, KCH>(acc, pq, smem_u32(sWq));
    frag_bias_pack(acc, s_bias, pk);
    frag_store_bf16(pk, p.Q, D, ra, T);
  }
}

template <int KCH>
static int launch_ln_qkv(const CUtensorMap& tmX, const CUtensorMap& tmWq, const CUtensorMap& tmWkv, const LnQkvParams& p,
                         cudaStream_t st) {
  constexpr int D = KCH * 64;
  const int smem = 3 * KCH * D * 128 + KCH * 128 * 128 + 1024;
  auto kern = ln_qkv_fused_kernel<KCH>;
  RP_CUDA_CHECK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  const int n_tiles = (p.T + 127) / 128;
  const int grid = n_tiles < sm_count() ? n_tiles : sm_count();
  kern<<<grid, kBlockThreads, smem, st>>>(tmX, tmWq, tmWkv, p);
  RP_LAUNCH_CHECK();
  return RP_OK;
}

}  // namespace rp

using namespace rp;

// x bf16 [T, d]; w_in bf16 [3d, d] (packed in_proj_weight: rows [0,d) = Wq, [d,3d) = Wk | Wv), b_in fp32 [3d]; ln_w / ln_b fp32 [d].
// Outputs: q_in bf16 [T, d] = LayerNorm(x), Q bf16 [T, d] = q_in Wq^T + bq, KV bf16 [T, 2d] = x [Wk | Wv]^T + [bk | bv],
// mean / rstd fp32 [T] (optional, both or none).  No output may alias x.  d in {64, 128}.
static int ln_qkv(const void* x, const float* ln_w, const float* ln_b, float eps, const void* w_in, const float* b_in, int T,
                  int d, void* q_in, void* Q, void* KV, float* mean_out, float* rstd_out, int hd_valid, const int32_t* n_rows_dev,
                  void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  const bool kv_only = q_in == nullptr && Q == nullptr;   // [K | V] projection alone (LayerNorm parameters not read)
  if (!x || !w_in || !b_in || !KV || T <= 0) return RP_EINVAL;
  if (!kv_only && (!ln_w || !ln_b || !q_in || !Q)) return RP_EINVAL;
  if ((mean_out == nullptr) != (rstd_out == nullptr)) return RP_EINVAL;
  if (kv_only) mean_out = rstd_out = nullptr;
  if (d != 64 && d != 128) return RP_ESHAPE;
  if (hd_valid < 0 || hd_valid > 128 || (hd_valid > 0 && d % (hd_valid <= 64 ? 64 : 128))) return RP_ESHAPE;
  if ((!kv_only && (q_in == x || Q == x)) || KV == x) return RP_EINVAL;
  CUtensorMap tmX, tmWq, tmWkv;
  int rc;
  if ((rc = make_tmap_bf16(&tmX, x, T, d, d, 128)) != RP_OK) return rc;
  if ((rc = make_tmap_bf16(&tmWq, w_in, d, d, d, d)) != RP_OK) return rc;
  if ((rc = make_tmap_bf16(&tmWkv, reinterpret_cast<const __nv_bfloat16*>(w_in) + (size_t)d * d, 2 * d, d, d, 2 * d)) != RP_OK)
    return rc;
  LnQkvParams p;
  p.ln_w = ln_w; p.ln_b = ln_b; p.b_in = b_in; p.eps = eps; p.T = T; p.hd_valid = hd_valid;
  p.q_in = reinterpret_cast<__nv_bfloat16*>(q_in); p.Q = reinterpret_cast<__nv_bfloat16*>(Q);
  p.KV = reinterpret_cast<__nv_bfloat16*>(KV); p.mean_out = mean_out; p.rstd_out = rstd_out;
  p.kv_only = kv_only ? 1 : 0;
  p.n_rows_dev = n_rows_dev;
  return d == 64 ? launch_ln_qkv<1>(tmX, tmWq, tmWkv, p, stream) : launch_ln_qkv<2>(tmX, tmWq, tmWkv, p, stream);
}

RP_API int rp_ln_qkv_fused(const void* x, const float* ln_w, const float* ln_b, float eps, const void* w_in, const float* b_in,
                           int T, int d, void* q_in, void* Q, void* KV, float* mean_out, float* rstd_out, int hd_valid,
                           void* stream_) {
  return ln_qkv(x, ln_w, ln_b, eps, w_in, b_in, T, d, q_in, Q, KV, mean_out, rstd_out, hd_valid, nullptr, stream_);
}

// Packed rows: the same over the first *n_rows_dev rows of the [T, *] arrays (T, the capacity, sizes the grid and the maps).
RP_API int rp_ln_qkv_fused_rows(const void* x, const float* ln_w, const float* ln_b, float eps, const void* w_in,
                                const float* b_in, int T, int d, void* q_in, void* Q, void* KV, float* mean_out, float* rstd_out,
                                int hd_valid, const int32_t* n_rows_dev, void* stream_) {
  if (!n_rows_dev) return RP_EINVAL;
  return ln_qkv(x, ln_w, ln_b, eps, w_in, b_in, T, d, q_in, Q, KV, mean_out, rstd_out, hd_valid, n_rows_dev, stream_);
}

// ------------------------------------------------------------------------------------------------------------------
// Backward of the pre-attention part:   dq_in = dQ Wq + dh ;  t = LN1-backward(dq_in ; x, mean, rstd, w) ;  dx = dKV Wkv + t
// (q_in = LN1(x) feeds the Q projection AND is the residual of the block: `x = q + attention(q, x, x)`,
//  replay/nn/sequential/sasrec/transformer.py:99-107, so dh - the gradient of h = q_in + attn - adds to dq_in directly;
//  K and V are projected from the un-normalised x, so their gradient by-passes the LayerNorm.)
// Per 128-token tile two GEMMs (contraction over the projection outputs: the weights are read MN-major in place) from the
// staged dQ | dKV tile; the LayerNorm parameter gradients (column sums over the tokens of dq and dq * xhat) are accumulated in
// registers over the CTA's tiles and added to the gradient buffers once per CTA.
// ------------------------------------------------------------------------------------------------------------------
namespace rp {

struct PreAttnBwdParams {
  const __nv_bfloat16* dh;    // [T, d] gradient of h = q_in + attn wrt h (residual branch into q_in)
  const __nv_bfloat16* x;     // [T, d] input of LayerNorm1
  const float* mean;
  const float* rstd;
  const float* ln_w;
  __nv_bfloat16* dx;          // [T, d]
  float* dln_w;               // [d] +=
  float* dln_b;               // [d] +=
  int T;
  int hd_valid;               // > 0: padded feature slots - statistics over the real features, no gradient into padded inputs
  const int32_t* n_rows_dev;  // as in LnQkvParams
};

template <int KCH>
__global__ void __launch_bounds__(kBlockThreads, 1)
pre_attn_bwd_kernel(const __grid_constant__ CUtensorMap tmDQ, const __grid_constant__ CUtensorMap tmDKV,
                    const __grid_constant__ CUtensorMap tmWq, const __grid_constant__ CUtensorMap tmWkv, const PreAttnBwdParams p) {
  constexpr int D = KCH * 64, R = D / 2;
  constexpr int NCH = 3 * KCH;                  // A chunks ([128 x 64]) per tile: KCH of dQ, then 2 KCH of [dK | dV]
  constexpr int WQ_BYTES = KCH * KCH * 8192;    // MN-major B: K chunks (64 output features) x N chunks (64 input features)
  constexpr int WKV_BYTES = 2 * KCH * KCH * 8192;
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sWq = smem;
  uint8_t* sWkv = smem + WQ_BYTES;
  uint8_t* sA = smem + WQ_BYTES + WKV_BYTES;    // NCH chunks of 16 KB
  __shared__ uint64_t bar_w, bar_a;
  __shared__ __align__(16) float s_lnw[D];
  __shared__ float s_red[2 * 8 * D];

  const int T = p.n_rows_dev ? *p.n_rows_dev : p.T;   // rows [T, p.T) of a packed batch are stale: never stored nor summed
  const int n_tiles = (T + 127) / 128;
  const int my_tiles = n_tiles > (int)blockIdx.x ? (n_tiles - 1 - (int)blockIdx.x) / (int)gridDim.x + 1 : 0;
  auto load_a = [&](int it) {
    const int t = (int)blockIdx.x + it * (int)gridDim.x;
    mbar_arrive_expect_tx(&bar_a, NCH * 16384);
    for (int c = 0; c < NCH; ++c) {
      if (c < KCH) tma_load_2d(sA + c * 16384, &tmDQ, &bar_a, c * 64, t * 128);
      else tma_load_2d(sA + c * 16384, &tmDKV, &bar_a, (c - KCH) * 64, t * 128);
    }
  };
  if (threadIdx.x == 0) {
    mbar_init(&bar_w, 1);
    mbar_init(&bar_a, 1);
    fence_barrier_init();
    mbar_arrive_expect_tx(&bar_w, WQ_BYTES + WKV_BYTES);
    for (int kc = 0; kc < KCH; ++kc)
      for (int nc = 0; nc < KCH; ++nc) tma_load_2d(sWq + (kc * KCH + nc) * 8192, &tmWq, &bar_w, nc * 64, kc * 64);
    for (int kc = 0; kc < 2 * KCH; ++kc)
      for (int nc = 0; nc < KCH; ++nc) tma_load_2d(sWkv + (kc * KCH + nc) * 8192, &tmWkv, &bar_w, nc * 64, kc * 64);
    if (my_tiles > 0) load_a(0);
  }
  for (int i = threadIdx.x; i < D; i += kBlockThreads) s_lnw[i] = p.ln_w[i];
  __syncthreads();
  const int wg = threadIdx.x >> 7, t = threadIdx.x & 127;
  const int fr = frag_row(t), fc = frag_col(t);
  const uint32_t aA = smem_u32(sA) + wg * 8192;
  const float inv_d = 1.f / (float)feat_count(D, p.hd_valid);
  float cw[R / 2], cb[R / 2];   // LayerNorm parameter gradients of this thread's columns, summed over its rows and tiles
  acc_zero(cw);
  acc_zero(cb);
  mbar_wait(&bar_w, 0);
  for (int it = 0; it < my_tiles; ++it) {
    const int tile = (int)blockIdx.x + it * (int)gridDim.x;
    const int ra = tile * 128 + 64 * wg + fr;
    float dq[R];
    mbar_wait(&bar_a, it & 1);
    wg_gemm_ss_w<D, KCH>(dq, aA, smem_u32(sWq));   // dQ . Wq
    {
      float hv[R];
      frag_load_bf16(p.dh, D, ra, T, hv);
#pragma unroll
      for (int i = 0; i < R; ++i) dq[i] += hv[i];
    }
    {
      // LayerNorm backward, in place: dq -> t (the LayerNorm input gradient)
      float xv[R];
      frag_load_bf16(p.x, D, ra, T, xv);
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int r = ra + 8 * h;
        const bool ok = r < T;
        const float rs = ok ? p.rstd[r] : 0.f, nmr = ok ? -p.mean[r] * rs : 0.f;   // xhat = x * rstd - mean * rstd (0 beyond T)
        float s1 = 0.f, s2 = 0.f;
#pragma unroll
        for (int j = 0; j < R / 4; ++j)
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int i = 4 * j + 2 * h + e;
            const float g = dq[i] * s_lnw[8 * j + fc + e], xh = fmaf(xv[i], rs, nmr);
            s1 += g;
            s2 = fmaf(g, xh, s2);
            if (ok) {
              cw[2 * j + e] = fmaf(dq[i], xh, cw[2 * j + e]);
              cb[2 * j + e] += dq[i];
            }
          }
        const float m1 = quad_sum(s1) * inv_d, m2 = quad_sum(s2) * inv_d;
#pragma unroll
        for (int j = 0; j < R / 4; ++j)
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int i = 4 * j + 2 * h + e, c = 8 * j + fc + e;
            const float tt = rs * (dq[i] * s_lnw[c] - m1 - fmaf(xv[i], rs, nmr) * m2);
            dq[i] = feat_valid(c, p.hd_valid) ? tt : 0.f;   // padded inputs of the LayerNorm do not exist: no gradient
          }
      }
    }
    float acc2[R];
    wg_gemm_ss_w<D, 2 * KCH>(acc2, aA + KCH * 16384, smem_u32(sWkv));  // [dK | dV] . Wkv
    named_bar_sync(1, kBlockThreads);   // the staged tile has been read
    if (threadIdx.x == 0 && it + 1 < my_tiles) load_a(it + 1);
#pragma unroll
    for (int i = 0; i < R; ++i) acc2[i] += dq[i];
    uint32_t pk[R / 2];
    frag_pack(acc2, pk);
    frag_store_bf16(pk, p.dx, D, ra, T);
  }
  frag_colsum_commit<R>(cw, cb, s_red, p.dln_w, p.dln_b, kBlockThreads);
}

template <int KCH>
static int launch_pre_attn_bwd(const CUtensorMap& tmDQ, const CUtensorMap& tmDKV, const CUtensorMap& tmWq,
                               const CUtensorMap& tmWkv, const PreAttnBwdParams& p, cudaStream_t st) {
  const int smem = 3 * KCH * KCH * 8192 + 3 * KCH * 128 * 128 + 1024;
  auto kern = pre_attn_bwd_kernel<KCH>;
  RP_CUDA_CHECK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  const int n_tiles = (p.T + 127) / 128;
  const int grid = n_tiles < sm_count() ? n_tiles : sm_count();
  kern<<<grid, kBlockThreads, smem, st>>>(tmDQ, tmDKV, tmWq, tmWkv, p);
  RP_LAUNCH_CHECK();
  return RP_OK;
}

}  // namespace rp

// dQ bf16 [T, d]; dKV bf16 [T, 2d]; dh, x bf16 [T, d]; mean, rstd fp32 [T] (LayerNorm1 statistics of x); ln_w fp32 [d];
// w_in bf16 [3d, d] (packed in_proj_weight).  Outputs: dx bf16 [T, d] (no aliasing with the inputs); dln_w / dln_b fp32 [d] are
// ACCUMULATED (+=, fp32 atomics: one per column and CTA).  d in {64, 128}.
static int pre_attn_bwd(const void* dQ, const void* dKV, const void* dh, const void* x, const float* mean, const float* rstd,
                        const float* ln_w, const void* w_in, int T, int d, void* dx, float* dln_w, float* dln_b, int hd_valid,
                        const int32_t* n_rows_dev, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (!dQ || !dKV || !dh || !x || !mean || !rstd || !ln_w || !w_in || !dx || !dln_w || !dln_b || T <= 0) return RP_EINVAL;
  if (d != 64 && d != 128) return RP_ESHAPE;
  if (hd_valid < 0 || hd_valid > 128 || (hd_valid > 0 && d % (hd_valid <= 64 ? 64 : 128))) return RP_ESHAPE;
  if (dx == dQ || dx == dKV || dx == dh || dx == x) return RP_EINVAL;
  CUtensorMap tmDQ, tmDKV, tmWq, tmWkv;
  int rc;
  if ((rc = make_tmap_bf16(&tmDQ, dQ, T, d, d, 128)) != RP_OK) return rc;
  if ((rc = make_tmap_bf16(&tmDKV, dKV, T, 2 * d, 2 * d, 128)) != RP_OK) return rc;
  if ((rc = make_tmap_bf16(&tmWq, w_in, d, d, d, 64)) != RP_OK) return rc;
  if ((rc = make_tmap_bf16(&tmWkv, reinterpret_cast<const __nv_bfloat16*>(w_in) + (size_t)d * d, 2 * d, d, d, 64)) != RP_OK)
    return rc;
  PreAttnBwdParams p;
  p.dh = reinterpret_cast<const __nv_bfloat16*>(dh); p.x = reinterpret_cast<const __nv_bfloat16*>(x);
  p.mean = mean; p.rstd = rstd; p.ln_w = ln_w; p.dx = reinterpret_cast<__nv_bfloat16*>(dx);
  p.dln_w = dln_w; p.dln_b = dln_b; p.T = T; p.hd_valid = hd_valid; p.n_rows_dev = n_rows_dev;
  return d == 64 ? launch_pre_attn_bwd<1>(tmDQ, tmDKV, tmWq, tmWkv, p, stream)
                 : launch_pre_attn_bwd<2>(tmDQ, tmDKV, tmWq, tmWkv, p, stream);
}

RP_API int rp_pre_attn_bwd(const void* dQ, const void* dKV, const void* dh, const void* x, const float* mean, const float* rstd,
                           const float* ln_w, const void* w_in, int T, int d, void* dx, float* dln_w, float* dln_b,
                           int hd_valid, void* stream_) {
  return pre_attn_bwd(dQ, dKV, dh, x, mean, rstd, ln_w, w_in, T, d, dx, dln_w, dln_b, hd_valid, nullptr, stream_);
}

// Packed rows: the first *n_rows_dev rows only (the LayerNorm parameter gradients sum exactly those rows).
RP_API int rp_pre_attn_bwd_rows(const void* dQ, const void* dKV, const void* dh, const void* x, const float* mean,
                                const float* rstd, const float* ln_w, const void* w_in, int T, int d, void* dx, float* dln_w,
                                float* dln_b, int hd_valid, const int32_t* n_rows_dev, void* stream_) {
  if (!n_rows_dev) return RP_EINVAL;
  return pre_attn_bwd(dQ, dKV, dh, x, mean, rstd, ln_w, w_in, T, d, dx, dln_w, dln_b, hd_valid, n_rows_dev, stream_);
}


// ==================================================================================================================
// Post-attention block (out-projection + LayerNorm + point-wise feed-forward) for inference and training.

namespace rp {

// ------------------------------------------------------------------------------------------------------------------
// Everything after the attention of one SASRec block in ONE pass over the tokens:
//   h = O Wo^T + bo + q_in ;  y = LayerNorm(h) ;  out = relu(y W1^T + b1) W2^T + b2 + y
// (replaces out-projection GEMM + LayerNorm + two FFN GEMMs: h and y never reach HBM in inference).  Per 128-token tile three
// chained wgmma GEMMs; y and u stay in registers as the bf16 A operands of the next one, the LayerNorm statistics of a row
// come from the four threads of a quad.
// ------------------------------------------------------------------------------------------------------------------
struct PostAttnParams {
  const float* bo;
  const float* ln_w;
  const float* ln_b;
  const float* b1;
  const float* b2;
  const __nv_bfloat16* q_in;   // residual of the out-projection, [T, d]
  const uint8_t* rowmask;
  __nv_bfloat16* out;
  float eps;
  int T;
  // TRAIN: activations saved for the backward (bf16 [T, d]; u is stored AFTER its dropout, as the un-fused path does) and
  // the two dropouts of the FFN (replay/nn/ffn.py:49-55), regenerated in the backward from (seed, site offset, element index)
  __nv_bfloat16* h_save;
  __nv_bfloat16* y_save;
  __nv_bfloat16* u_save;
  float* mean_out;
  float* rstd_out;
  float drop_p;
  unsigned long long seed, off1, off2;
  const unsigned long long* seed_ptr;
  int hd_valid;                // > 0: padded feature slots (rp_sm90.cuh): LayerNorm statistics over the real features only
  const int32_t* n_rows_dev;   // packed rows (as in LnQkvParams), or null
  const int32_t* row_tok;      // packed rows: token of every row, the dropout row key (null: the row itself)
};

template <int KCH, bool TRAIN>
__global__ void __launch_bounds__(kBlockThreads, 1)
post_attn_fused_kernel(const __grid_constant__ CUtensorMap tmO, const __grid_constant__ CUtensorMap tmWo,
                       const __grid_constant__ CUtensorMap tmW1, const __grid_constant__ CUtensorMap tmW2, const PostAttnParams p) {
  constexpr int D = KCH * 64, R = D / 2;
  constexpr int W_BYTES = KCH * D * 128;
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sWo = smem;
  uint8_t* sW1 = smem + W_BYTES;
  uint8_t* sW2 = smem + 2 * W_BYTES;
  uint8_t* sO = smem + 3 * W_BYTES;            // [128 x D]
  __shared__ uint64_t bar_w, bar_o;
  __shared__ __align__(16) float s_vec[5][D];     // bo, ln_w, ln_b, b1, b2
  __shared__ __align__(16) uint32_t s_ck[D];      // dropout column keys

  const int T = p.n_rows_dev ? *p.n_rows_dev : p.T;   // rows [T, p.T) of a packed batch are stale: never stored nor summed
  const int n_tiles = (T + 127) / 128;
  const int my_tiles = n_tiles > (int)blockIdx.x ? (n_tiles - 1 - (int)blockIdx.x) / (int)gridDim.x + 1 : 0;
  auto load_o = [&](int it) {
    const int t = (int)blockIdx.x + it * (int)gridDim.x;
    mbar_arrive_expect_tx(&bar_o, KCH * 16384);
    for (int kc = 0; kc < KCH; ++kc) tma_load_2d(sO + kc * 16384, &tmO, &bar_o, kc * 64, t * 128);
  };
  if (threadIdx.x == 0) {
    mbar_init(&bar_w, 1);
    mbar_init(&bar_o, 1);
    fence_barrier_init();
    mbar_arrive_expect_tx(&bar_w, 3 * W_BYTES);
    for (int kc = 0; kc < KCH; ++kc) {
      tma_load_2d(sWo + kc * (D * 128), &tmWo, &bar_w, kc * 64, 0);
      tma_load_2d(sW1 + kc * (D * 128), &tmW1, &bar_w, kc * 64, 0);
      tma_load_2d(sW2 + kc * (D * 128), &tmW2, &bar_w, kc * 64, 0);
    }
    if (my_tiles > 0) load_o(0);
  }
  for (int i = threadIdx.x; i < D; i += kBlockThreads) {
    s_vec[0][i] = p.bo[i];
    s_vec[1][i] = p.ln_w[i];
    s_vec[2][i] = p.ln_b[i];
    s_vec[3][i] = p.b1[i];
    s_vec[4][i] = p.b2[i];
    s_ck[i] = drop_col_key((uint32_t)i);
  }
  __syncthreads();
  const int wg = threadIdx.x >> 7, t = threadIdx.x & 127;
  const int fr = frag_row(t), fc = frag_col(t);
  const bool drop = TRAIN && p.drop_p > 0.f;
  const float keep_scale = drop ? 1.f / (1.f - p.drop_p) : 1.f;
  const uint32_t drop_thr = drop ? (uint32_t)(p.drop_p * 4294967296.0) : 0u;
  const unsigned long long seed_eff = TRAIN ? p.seed + ((p.drop_p > 0.f && p.seed_ptr) ? *p.seed_ptr : 0ull) : 0ull;
  const float inv_d = 1.f / (float)feat_count(D, p.hd_valid);   // padded columns are zero: sums need no mask
  mbar_wait(&bar_w, 0);
  for (int it = 0; it < my_tiles; ++it) {
    const int tile = (int)blockIdx.x + it * (int)gridDim.x;
    const int ra = tile * 128 + 64 * wg + fr;
    mbar_wait(&bar_o, it & 1);
    // ---- h = O Wo^T + bo + q_in
    float hv[R];
    wg_gemm_ss_wt<D, KCH>(hv, smem_u32(sO) + wg * 8192, smem_u32(sWo));
    named_bar_sync(1, kBlockThreads);   // the O tile has been read
    if (threadIdx.x == 0 && it + 1 < my_tiles) load_o(it + 1);
    {
      float qv[R];
      frag_load_bf16(p.q_in, D, ra, T, qv);
#pragma unroll
      for (int i = 0; i < R; ++i) {
        hv[i] += s_vec[0][8 * (i >> 2) + fc + (i & 1)] + qv[i];
        if (TRAIN) hv[i] = __bfloat162float(__float2bfloat16(hv[i]));   // the statistics describe exactly the bf16 h the backward reads
      }
    }
    if (TRAIN) {
      uint32_t ph[R / 2];
      frag_pack(hv, ph);
      frag_store_bf16(ph, p.h_save, D, ra, T);
    }
    // ---- y = LayerNorm(h) (bf16: the A operand of the next GEMM and the residual of the block)
    uint32_t py[R / 2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      float sum = 0.f, sq = 0.f;
#pragma unroll
      for (int j = 0; j < R / 4; ++j)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const float x = hv[4 * j + 2 * h + e];
          sum += x;
          sq = fmaf(x, x, sq);
        }
      const float mean = quad_sum(sum) * inv_d;
      const float var = fmaxf(quad_sum(sq) * inv_d - mean * mean, 0.f);
      const float rstd = rsqrtf(var + p.eps);
      if (TRAIN && fc == 0 && ra + 8 * h < T) {
        p.mean_out[ra + 8 * h] = mean;
        p.rstd_out[ra + 8 * h] = rstd;
      }
#pragma unroll
      for (int j = 0; j < R / 4; ++j) {
        const int i = 4 * j + 2 * h, c = 8 * j + fc;
        py[2 * j + h] = pack_bf16((hv[i] - mean) * rstd * s_vec[1][c] + s_vec[2][c], (hv[i + 1] - mean) * rstd * s_vec[1][c + 1] + s_vec[2][c + 1]);
      }
    }
    if (TRAIN) frag_store_bf16(py, p.y_save, D, ra, T);
    // ---- u = dropout1(relu(y W1^T + b1))
    float acc[R];
    wg_gemm_rs_wt<D, KCH>(acc, py, smem_u32(sW1));
    uint32_t pu[R / 2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const uint32_t rk1 = drop ? drop_row_key(seed_eff, p.off1, row_token(p.row_tok, ra + 8 * h, T)) : 0u;
#pragma unroll
      for (int j = 0; j < R / 4; ++j) {
        const int i = 4 * j + 2 * h, c = 8 * j + fc;
        float a0 = fmaxf(acc[i] + s_vec[3][c], 0.f), a1 = fmaxf(acc[i + 1] + s_vec[3][c + 1], 0.f);
        if (drop) {
          a0 = drop_mix(rk1, s_ck[c]) >= drop_thr ? a0 * keep_scale : 0.f;
          a1 = drop_mix(rk1, s_ck[c + 1]) >= drop_thr ? a1 * keep_scale : 0.f;
        }
        pu[2 * j + h] = pack_bf16(a0, a1);
      }
    }
    if (TRAIN) frag_store_bf16(pu, p.u_save, D, ra, T);
    // ---- out = (y + dropout2(u W2^T + b2)) [* rowmask]
    wg_gemm_rs_wt<D, KCH>(acc, pu, smem_u32(sW2));
    uint32_t po[R / 2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int r = ra + 8 * h;
      const float keep = (p.rowmask == nullptr || (r < T && p.rowmask[r])) ? 1.f : 0.f;
      const uint32_t rk2 = drop ? drop_row_key(seed_eff, p.off2, row_token(p.row_tok, r, T)) : 0u;
#pragma unroll
      for (int j = 0; j < R / 4; ++j) {
        const int i = 4 * j + 2 * h, c = 8 * j + fc;
        float f0 = acc[i] + s_vec[4][c], f1 = acc[i + 1] + s_vec[4][c + 1];
        if (drop) {
          f0 = drop_mix(rk2, s_ck[c]) >= drop_thr ? f0 * keep_scale : 0.f;
          f1 = drop_mix(rk2, s_ck[c + 1]) >= drop_thr ? f1 * keep_scale : 0.f;
        }
        const float2 yf = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&py[2 * j + h]));
        po[2 * j + h] = pack_bf16((f0 + yf.x) * keep, (f1 + yf.y) * keep);
      }
    }
    frag_store_bf16(po, p.out, D, ra, T);
  }
}

template <int KCH, bool TRAIN>
static int launch_post_attn(const CUtensorMap& tmO, const CUtensorMap& tmWo, const CUtensorMap& tmW1, const CUtensorMap& tmW2,
                            const PostAttnParams& p, cudaStream_t st) {
  constexpr int D = KCH * 64;
  const int smem = 3 * KCH * D * 128 + KCH * 128 * 128 + 1024;
  auto kern = post_attn_fused_kernel<KCH, TRAIN>;
  RP_CUDA_CHECK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  const int n_tiles = (p.T + 127) / 128;
  const int grid = n_tiles < sm_count() ? n_tiles : sm_count();
  kern<<<grid, kBlockThreads, smem, st>>>(tmO, tmWo, tmW1, tmW2, p);
  RP_LAUNCH_CHECK();
  return RP_OK;
}

}  // namespace rp

using namespace rp;

// Inference: out-projection + residual + LayerNorm + FFN of one SASRec block in one pass (see post_attn_fused_kernel).
//   o, q_in, out bf16 [T, d] (out may not alias o / q_in); wo, w1, w2 bf16 [d, d]; bo, ln_w, ln_b, b1, b2 fp32 [d]; d in {64,128}.
//   replaces (eval)  out_proj + "x = q + a" + LayerNorm + FFN   replay/nn/sequential/sasrec/transformer.py:99-110 ;
//                                                              replay/models/nn/sequential/sasrec/model.py:435-441
RP_API int rp_post_attn_fused(const void* o, const void* q_in, const void* wo, const float* bo, const float* ln_w,
                              const float* ln_b, float eps, const void* w1, const float* b1, const void* w2, const float* b2,
                              const uint8_t* rowmask, int T, int d, void* out, int hd_valid, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (!o || !q_in || !wo || !bo || !ln_w || !ln_b || !w1 || !b1 || !w2 || !b2 || !out || T <= 0) return RP_EINVAL;
  if (d != 64 && d != 128) return RP_ESHAPE;
  if (hd_valid < 0 || hd_valid > 128 || (hd_valid > 0 && d % (hd_valid <= 64 ? 64 : 128))) return RP_ESHAPE;
  if (out == o || out == q_in) return RP_EINVAL;
  CUtensorMap tmO, tmWo, tmW1, tmW2;
  int rc;
  if ((rc = make_tmap_bf16(&tmO, o, T, d, d, 128)) != RP_OK) return rc;
  if ((rc = make_tmap_bf16(&tmWo, wo, d, d, d, d)) != RP_OK) return rc;
  if ((rc = make_tmap_bf16(&tmW1, w1, d, d, d, d)) != RP_OK) return rc;
  if ((rc = make_tmap_bf16(&tmW2, w2, d, d, d, d)) != RP_OK) return rc;
  PostAttnParams p;
  p.bo = bo; p.ln_w = ln_w; p.ln_b = ln_b; p.b1 = b1; p.b2 = b2;
  p.q_in = reinterpret_cast<const __nv_bfloat16*>(q_in); p.rowmask = rowmask;
  p.out = reinterpret_cast<__nv_bfloat16*>(out); p.eps = eps; p.T = T;
  p.h_save = p.y_save = p.u_save = nullptr; p.mean_out = p.rstd_out = nullptr;
  p.drop_p = 0.f; p.seed = p.off1 = p.off2 = 0ull; p.seed_ptr = nullptr; p.hd_valid = hd_valid;
  p.n_rows_dev = nullptr; p.row_tok = nullptr;
  return d == 64 ? launch_post_attn<1, false>(tmO, tmWo, tmW1, tmW2, p, stream)
                 : launch_post_attn<2, false>(tmO, tmWo, tmW1, tmW2, p, stream);
}

// Training forward of everything after the attention of one SASRec block, one pass over the tokens:
//   h = O Wo^T + bo + q_in ; y = LayerNorm(h) ; u = dropout1(relu(y W1^T + b1)) ; out = (y + dropout2(u W2^T + b2)) [* rowmask]
// and the activations the backward needs are written on the way: h, y, u (bf16 [T, d]) and the LayerNorm statistics
// (fp32 [T]) - 2 tensors read, 4 written, against 14 [T, d] passes of the four separate launches
// (out-projection GEMM, LayerNorm, two FFN GEMMs).  Dropout element e of site s uses word (e & 3) of
// drop_mix(drop_row_key(seed + *seed_ptr, off_s, row), drop_col_key(column)): the same stream rp_gemm's epilogue and rp_dropout_bwd use.
//   replaces (train)  replay/nn/sequential/sasrec/transformer.py:99-110 ; replay/nn/ffn.py:43-57 ;
//                     replay/models/nn/sequential/sasrec/model.py:435-441,496-506
static int post_attn_train(const void* o, const void* q_in, const void* wo, const float* bo, const float* ln_w,
                           const float* ln_b, float eps, const void* w1, const float* b1, const void* w2, const float* b2,
                           const uint8_t* rowmask, int T, int d, float drop_p, unsigned long long seed,
                           unsigned long long drop_off1, unsigned long long drop_off2, const unsigned long long* seed_ptr,
                           void* h_save, void* y_save, void* u_save, float* mean_out, float* rstd_out, void* out, int hd_valid,
                           const int32_t* n_rows_dev, const int32_t* row_tok, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (!o || !q_in || !wo || !bo || !ln_w || !ln_b || !w1 || !b1 || !w2 || !b2 || !out || T <= 0) return RP_EINVAL;
  if (!h_save || !y_save || !u_save || !mean_out || !rstd_out) return RP_EINVAL;
  if (d != 64 && d != 128) return RP_ESHAPE;
  if (drop_p < 0.f || drop_p >= 1.f || (drop_off1 & 3) || (drop_off2 & 3)) return RP_EINVAL;
  if (hd_valid < 0 || hd_valid > 128 || (hd_valid > 0 && d % (hd_valid <= 64 ? 64 : 128))) return RP_ESHAPE;
  if (out == o || out == q_in) return RP_EINVAL;
  CUtensorMap tmO, tmWo, tmW1, tmW2;
  int rc;
  if ((rc = make_tmap_bf16(&tmO, o, T, d, d, 128)) != RP_OK) return rc;
  if ((rc = make_tmap_bf16(&tmWo, wo, d, d, d, d)) != RP_OK) return rc;
  if ((rc = make_tmap_bf16(&tmW1, w1, d, d, d, d)) != RP_OK) return rc;
  if ((rc = make_tmap_bf16(&tmW2, w2, d, d, d, d)) != RP_OK) return rc;
  PostAttnParams p;
  p.bo = bo; p.ln_w = ln_w; p.ln_b = ln_b; p.b1 = b1; p.b2 = b2;
  p.q_in = reinterpret_cast<const __nv_bfloat16*>(q_in); p.rowmask = rowmask;
  p.out = reinterpret_cast<__nv_bfloat16*>(out); p.eps = eps; p.T = T;
  p.h_save = reinterpret_cast<__nv_bfloat16*>(h_save); p.y_save = reinterpret_cast<__nv_bfloat16*>(y_save);
  p.u_save = reinterpret_cast<__nv_bfloat16*>(u_save); p.mean_out = mean_out; p.rstd_out = rstd_out;
  p.drop_p = drop_p; p.seed = seed; p.off1 = drop_off1; p.off2 = drop_off2; p.seed_ptr = seed_ptr; p.hd_valid = hd_valid;
  p.n_rows_dev = n_rows_dev; p.row_tok = row_tok;
  return d == 64 ? launch_post_attn<1, true>(tmO, tmWo, tmW1, tmW2, p, stream)
                 : launch_post_attn<2, true>(tmO, tmWo, tmW1, tmW2, p, stream);
}

RP_API int rp_post_attn_train(const void* o, const void* q_in, const void* wo, const float* bo, const float* ln_w,
                              const float* ln_b, float eps, const void* w1, const float* b1, const void* w2, const float* b2,
                              const uint8_t* rowmask, int T, int d, float drop_p, unsigned long long seed,
                              unsigned long long drop_off1, unsigned long long drop_off2, const unsigned long long* seed_ptr,
                              void* h_save, void* y_save, void* u_save, float* mean_out, float* rstd_out, void* out,
                              int hd_valid, void* stream_) {
  return post_attn_train(o, q_in, wo, bo, ln_w, ln_b, eps, w1, b1, w2, b2, rowmask, T, d, drop_p, seed, drop_off1, drop_off2,
                         seed_ptr, h_save, y_save, u_save, mean_out, rstd_out, out, hd_valid, nullptr, nullptr, stream_);
}

// Packed rows: the first *n_rows_dev rows only; row r draws its dropout with the key of token row_tok[r], so the kept
// elements are those of the padded run.
RP_API int rp_post_attn_train_rows(const void* o, const void* q_in, const void* wo, const float* bo, const float* ln_w,
                                   const float* ln_b, float eps, const void* w1, const float* b1, const void* w2, const float* b2,
                                   int T, int d, float drop_p, unsigned long long seed, unsigned long long drop_off1,
                                   unsigned long long drop_off2, const unsigned long long* seed_ptr, void* h_save, void* y_save,
                                   void* u_save, float* mean_out, float* rstd_out, void* out, int hd_valid,
                                   const int32_t* n_rows_dev, const int32_t* row_tok, void* stream_) {
  if (!n_rows_dev || !row_tok) return RP_EINVAL;
  return post_attn_train(o, q_in, wo, bo, ln_w, ln_b, eps, w1, b1, w2, b2, nullptr, T, d, drop_p, seed, drop_off1, drop_off2,
                         seed_ptr, h_save, y_save, u_save, mean_out, rstd_out, out, hd_valid, n_rows_dev, row_tok, stream_);
}


// ==================================================================================================================
// Backward of everything AFTER the attention of one SASRec block, one pass over the tokens:
//
//   forward (rp_post_attn_train):  h = O Wo^T + bo + q_in ; y = LN2(h) ; u = drop1(relu(y W1^T + b1)) ; x' = (y + drop2(u W2^T + b2)) [* pad]
//   here, given dz = d loss / d x':
//     dzm = dz [* pad] ;  d_t = drop2'(dzm) ;  du = (d_t W2) * relu'/drop1'(u) ;  dy = du W1 + dzm ;
//     dh  = LN2-backward(dy ; h, mean, rstd, w) ;  d_o = dh Wo          (+ dLN2.weight, dLN2.bias)
//
// Replaces autograd's backward of  replay/nn/sequential/sasrec/transformer.py:107-110 + replay/nn/ffn.py:43-57
// (legacy: replay/models/nn/sequential/sasrec/model.py:436-441,496-506).  dz, u and h are read once; d_t, du, dh (operands of
// the grouped weight-gradient launch, dh also the residual gradient into the pre-attention part) and d_o are written once.
// Three chained wgmma GEMMs per 128-token tile whose A operands (d_t, du, dh) never leave the registers; the weights are read
// MN-major in place (contraction over their output features) and stay resident in shared memory.

namespace rp {

struct PostAttnBwdParams {
  const __nv_bfloat16* u;      // [T, d] saved FFN hidden activation AFTER its dropout (zero = ReLU-clipped or dropped)
  const __nv_bfloat16* h;      // [T, d] saved LayerNorm2 input
  const float* mean;
  const float* rstd;
  const float* ln_w;
  const uint8_t* rowmask;      // legacy: the block output was multiplied by the pad mask (or null)
  __nv_bfloat16* d_t;          // [T, d] or null (then d_t == dz: no dropout, no row mask)
  __nv_bfloat16* du;
  __nv_bfloat16* dh;
  __nv_bfloat16* d_o;
  float* dln_w;
  float* dln_b;
  float drop_p;
  unsigned long long seed, off2;
  const unsigned long long* seed_ptr;
  int T;
  int hd_valid;                // > 0: padded feature slots - LN statistics over the real features, no gradient into padded inputs
  const int32_t* n_rows_dev;   // as in PostAttnParams
  const int32_t* row_tok;
};

template <int KCH>
__global__ void __launch_bounds__(kBlockThreads, 1)
post_attn_bwd_kernel(const __grid_constant__ CUtensorMap tmDZ, const __grid_constant__ CUtensorMap tmW2,
                     const __grid_constant__ CUtensorMap tmW1, const __grid_constant__ CUtensorMap tmWo, const PostAttnBwdParams p) {
  constexpr int D = KCH * 64, R = D / 2;
  constexpr int W_BYTES = KCH * KCH * 8192;   // MN-major B: K chunks (64 output features) x N chunks (64 input features)
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sW2 = smem;
  uint8_t* sW1 = smem + W_BYTES;
  uint8_t* sWo = smem + 2 * W_BYTES;
  uint8_t* sZ = smem + 3 * W_BYTES;            // [128 x D]
  __shared__ uint64_t bar_w, bar_z;
  __shared__ __align__(16) float s_lnw[D];
  __shared__ __align__(16) uint32_t s_ck[D];      // dropout column keys (rp_philox.cuh)
  __shared__ float s_red[2 * 8 * D];

  const int T = p.n_rows_dev ? *p.n_rows_dev : p.T;   // rows [T, p.T) of a packed batch are stale: never stored nor summed
  const int n_tiles = (T + 127) / 128;
  const int my_tiles = n_tiles > (int)blockIdx.x ? (n_tiles - 1 - (int)blockIdx.x) / (int)gridDim.x + 1 : 0;
  auto load_z = [&](int it) {
    const int t = (int)blockIdx.x + it * (int)gridDim.x;
    mbar_arrive_expect_tx(&bar_z, KCH * 16384);
    for (int kc = 0; kc < KCH; ++kc) tma_load_2d(sZ + kc * 16384, &tmDZ, &bar_z, kc * 64, t * 128);
  };
  if (threadIdx.x == 0) {
    mbar_init(&bar_w, 1);
    mbar_init(&bar_z, 1);
    fence_barrier_init();
    mbar_arrive_expect_tx(&bar_w, 3 * W_BYTES);
    for (int kc = 0; kc < KCH; ++kc)
      for (int nc = 0; nc < KCH; ++nc) {
        tma_load_2d(sW2 + (kc * KCH + nc) * 8192, &tmW2, &bar_w, nc * 64, kc * 64);
        tma_load_2d(sW1 + (kc * KCH + nc) * 8192, &tmW1, &bar_w, nc * 64, kc * 64);
        tma_load_2d(sWo + (kc * KCH + nc) * 8192, &tmWo, &bar_w, nc * 64, kc * 64);
      }
    if (my_tiles > 0) load_z(0);
  }
  for (int i = threadIdx.x; i < D; i += kBlockThreads) {
    s_lnw[i] = p.ln_w[i];
    s_ck[i] = drop_col_key((uint32_t)i);
  }
  __syncthreads();
  const int wg = threadIdx.x >> 7, t = threadIdx.x & 127;
  const int fr = frag_row(t), fc = frag_col(t);
  const float ks_ = p.drop_p > 0.f ? 1.f / (1.f - p.drop_p) : 1.f;
  const uint32_t thr = p.drop_p > 0.f ? (uint32_t)(p.drop_p * 4294967296.0) : 0u;
  const unsigned long long seed_eff = p.seed + ((p.drop_p > 0.f && p.seed_ptr) ? *p.seed_ptr : 0ull);
  const float inv_d = 1.f / (float)feat_count(D, p.hd_valid);
  float cw[R / 2], cb[R / 2];   // LayerNorm parameter gradients of this thread's columns, summed over its rows and tiles
  acc_zero(cw);
  acc_zero(cb);
  mbar_wait(&bar_w, 0);
  for (int it = 0; it < my_tiles; ++it) {
    const int tile = (int)blockIdx.x + it * (int)gridDim.x;
    const int ra = tile * 128 + 64 * wg + fr;
    float rm[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) rm[h] = (p.rowmask == nullptr || (ra + 8 * h < T && p.rowmask[ra + 8 * h])) ? 1.f : 0.f;
    // ---- dzm = dz * pad (kept for the residual branch), d_t = dropout2'(dzm)
    float dzm[R];
    mbar_wait(&bar_z, it & 1);
    frag_load_tile(sZ, 64 * wg + fr, dzm);
    named_bar_sync(1, kBlockThreads);   // the dz tile has been read
    if (threadIdx.x == 0 && it + 1 < my_tiles) load_z(it + 1);
    uint32_t pk[R / 2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const uint32_t rk2 = p.drop_p > 0.f ? drop_row_key(seed_eff, p.off2, row_token(p.row_tok, ra + 8 * h, T)) : 0u;
#pragma unroll
      for (int j = 0; j < R / 4; ++j) {
        const int i = 4 * j + 2 * h, c = 8 * j + fc;
        dzm[i] *= rm[h];
        dzm[i + 1] *= rm[h];
        float v0 = dzm[i], v1 = dzm[i + 1];
        if (p.drop_p > 0.f) {
          v0 = drop_mix(rk2, s_ck[c]) >= thr ? v0 * ks_ : 0.f;
          v1 = drop_mix(rk2, s_ck[c + 1]) >= thr ? v1 * ks_ : 0.f;
        }
        pk[2 * j + h] = pack_bf16(v0, v1);
      }
    }
    if (p.d_t != nullptr) frag_store_bf16(pk, p.d_t, D, ra, T);
    // ---- du = (d_t W2) * [u != 0] / keep
    float acc[R];
    wg_gemm_rs_w<D, KCH>(acc, pk, smem_u32(sW2));
    {
      const int fcol = fc;
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int r = ra + 8 * h;
        const __nv_bfloat16* urow = p.u + (size_t)(r < T ? r : 0) * D + fcol;
#pragma unroll
        for (int j = 0; j < R / 4; ++j) {
          const uint32_t w = r < T ? *reinterpret_cast<const uint32_t*>(urow + 8 * j) : 0u;
          const int i = 4 * j + 2 * h;
          // bf16 zero test on the raw halves (-0 cannot occur after ReLU)
          pk[2 * j + h] = pack_bf16((w & 0x7fffu) ? acc[i] * ks_ : 0.f, (w & 0x7fff0000u) ? acc[i + 1] * ks_ : 0.f);
        }
      }
    }
    frag_store_bf16(pk, p.du, D, ra, T);
    // ---- dy = du W1 + dzm ; dh = LayerNorm2-backward(dy) ; LN parameter gradients
    wg_gemm_rs_w<D, KCH>(acc, pk, smem_u32(sW1));
#pragma unroll
    for (int i = 0; i < R; ++i) acc[i] += dzm[i];   // acc = dy
    {
      float hv[R];
      frag_load_bf16(p.h, D, ra, T, hv);
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int r = ra + 8 * h;
        const bool ok = r < T;
        const float rs = ok ? p.rstd[r] : 0.f, nmr = ok ? -p.mean[r] * rs : 0.f;
        float s1 = 0.f, s2 = 0.f;
#pragma unroll
        for (int j = 0; j < R / 4; ++j)
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int i = 4 * j + 2 * h + e;
            const float g = acc[i] * s_lnw[8 * j + fc + e], hh = fmaf(hv[i], rs, nmr);
            s1 += g;
            s2 = fmaf(g, hh, s2);
            if (ok) {
              cw[2 * j + e] = fmaf(acc[i], hh, cw[2 * j + e]);
              cb[2 * j + e] += acc[i];
            }
          }
        const float m1 = quad_sum(s1) * inv_d, m2 = quad_sum(s2) * inv_d;
#pragma unroll
        for (int j = 0; j < R / 4; ++j) {
          float tt[2];
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int i = 4 * j + 2 * h + e, c = 8 * j + fc + e;
            tt[e] = rs * (acc[i] * s_lnw[c] - m1 - fmaf(hv[i], rs, nmr) * m2);
            if (!feat_valid(c, p.hd_valid)) tt[e] = 0.f;   // padded inputs of the LayerNorm do not exist: no gradient
          }
          pk[2 * j + h] = pack_bf16(tt[0], tt[1]);
        }
      }
    }
    frag_store_bf16(pk, p.dh, D, ra, T);
    // ---- d_o = dh Wo
    wg_gemm_rs_w<D, KCH>(acc, pk, smem_u32(sWo));
    frag_pack(acc, pk);
    frag_store_bf16(pk, p.d_o, D, ra, T);
  }
  frag_colsum_commit<R>(cw, cb, s_red, p.dln_w, p.dln_b, kBlockThreads);
}

template <int KCH>
static int launch_post_attn_bwd(const CUtensorMap& tmDZ, const CUtensorMap& tmW2, const CUtensorMap& tmW1,
                                const CUtensorMap& tmWo, const PostAttnBwdParams& p, cudaStream_t st) {
  const int smem = 3 * KCH * KCH * 8192 + KCH * 128 * 128 + 1024;
  auto kern = post_attn_bwd_kernel<KCH>;
  RP_CUDA_CHECK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  const int n_tiles = (p.T + 127) / 128;
  const int grid = n_tiles < sm_count() ? n_tiles : sm_count();
  kern<<<grid, kBlockThreads, smem, st>>>(tmDZ, tmW2, tmW1, tmWo, p);
  RP_LAUNCH_CHECK();
  return RP_OK;
}

}  // namespace rp

using namespace rp;

// dz, u, h bf16 [T, d]; mean / rstd fp32 [T] (LayerNorm2 statistics saved by rp_post_attn_train); ln_w fp32 [d]; w2, w1, wo bf16
// [d, d] (row = output feature); rowmask optional uint8 [T].  Dropout site 2 is regenerated from (seed + *seed_ptr, drop_off2,
// element index) exactly as rp_post_attn_train / rp_gemm drew it; site 1 is encoded in the zeros of u.
// Outputs bf16 [T, d]: d_t (may be NULL when drop_p == 0 and rowmask == NULL: then d_t == dz), du, dh, d_o (none may alias an
// input); dln_w / dln_b fp32 [d] are ACCUMULATED (one atomic per column and CTA).  d in {64, 128}.
static int post_attn_bwd(const void* dz, const void* u, const void* h, const float* mean, const float* rstd, const float* ln_w,
                         const void* w2, const void* w1, const void* wo, const uint8_t* rowmask, int T, int d, float drop_p,
                         unsigned long long seed, unsigned long long drop_off2, const unsigned long long* seed_ptr, void* d_t,
                         void* du, void* dh, void* d_o, float* dln_w, float* dln_b, int hd_valid, const int32_t* n_rows_dev,
                         const int32_t* row_tok, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (!dz || !u || !h || !mean || !rstd || !ln_w || !w2 || !w1 || !wo || !du || !dh || !d_o || !dln_w || !dln_b || T <= 0)
    return RP_EINVAL;
  if (d != 64 && d != 128) return RP_ESHAPE;
  if (drop_p < 0.f || drop_p >= 1.f || (drop_off2 & 3)) return RP_EINVAL;
  if (hd_valid < 0 || hd_valid > 128 || (hd_valid > 0 && d % (hd_valid <= 64 ? 64 : 128))) return RP_ESHAPE;
  if (!d_t && (drop_p > 0.f || rowmask)) return RP_EINVAL;
  if (d_t == dz || du == dz || dh == dz || d_o == dz) return RP_EINVAL;
  CUtensorMap tmDZ, tmW2, tmW1, tmWo;
  int rc;
  if ((rc = make_tmap_bf16(&tmDZ, dz, T, d, d, 128)) != RP_OK) return rc;
  if ((rc = make_tmap_bf16(&tmW2, w2, d, d, d, 64)) != RP_OK) return rc;
  if ((rc = make_tmap_bf16(&tmW1, w1, d, d, d, 64)) != RP_OK) return rc;
  if ((rc = make_tmap_bf16(&tmWo, wo, d, d, d, 64)) != RP_OK) return rc;
  PostAttnBwdParams p;
  p.u = reinterpret_cast<const __nv_bfloat16*>(u); p.h = reinterpret_cast<const __nv_bfloat16*>(h);
  p.mean = mean; p.rstd = rstd; p.ln_w = ln_w; p.rowmask = rowmask;
  p.d_t = reinterpret_cast<__nv_bfloat16*>(d_t); p.du = reinterpret_cast<__nv_bfloat16*>(du);
  p.dh = reinterpret_cast<__nv_bfloat16*>(dh); p.d_o = reinterpret_cast<__nv_bfloat16*>(d_o);
  p.dln_w = dln_w; p.dln_b = dln_b; p.drop_p = drop_p; p.seed = seed; p.off2 = drop_off2; p.seed_ptr = seed_ptr; p.T = T;
  p.hd_valid = hd_valid; p.n_rows_dev = n_rows_dev; p.row_tok = row_tok;
  return d == 64 ? launch_post_attn_bwd<1>(tmDZ, tmW2, tmW1, tmWo, p, stream)
                 : launch_post_attn_bwd<2>(tmDZ, tmW2, tmW1, tmWo, p, stream);
}

RP_API int rp_post_attn_bwd(const void* dz, const void* u, const void* h, const float* mean, const float* rstd, const float* ln_w,
                            const void* w2, const void* w1, const void* wo, const uint8_t* rowmask, int T, int d, float drop_p,
                            unsigned long long seed, unsigned long long drop_off2, const unsigned long long* seed_ptr, void* d_t,
                            void* du, void* dh, void* d_o, float* dln_w, float* dln_b, int hd_valid, void* stream_) {
  return post_attn_bwd(dz, u, h, mean, rstd, ln_w, w2, w1, wo, rowmask, T, d, drop_p, seed, drop_off2, seed_ptr, d_t, du, dh, d_o,
                       dln_w, dln_b, hd_valid, nullptr, nullptr, stream_);
}

// Packed rows: the first *n_rows_dev rows only, dropout keyed by row_tok as in rp_post_attn_train_rows.
RP_API int rp_post_attn_bwd_rows(const void* dz, const void* u, const void* h, const float* mean, const float* rstd,
                                 const float* ln_w, const void* w2, const void* w1, const void* wo, int T, int d, float drop_p,
                                 unsigned long long seed, unsigned long long drop_off2, const unsigned long long* seed_ptr,
                                 void* d_t, void* du, void* dh, void* d_o, float* dln_w, float* dln_b, int hd_valid,
                                 const int32_t* n_rows_dev, const int32_t* row_tok, void* stream_) {
  if (!n_rows_dev || !row_tok) return RP_EINVAL;
  return post_attn_bwd(dz, u, h, mean, rstd, ln_w, w2, w1, wo, nullptr, T, d, drop_p, seed, drop_off2, seed_ptr, d_t, du, dh, d_o,
                       dln_w, dln_b, hd_valid, n_rows_dev, row_tok, stream_);
}
