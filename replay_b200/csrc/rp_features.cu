// rp_features.cu - the new-path SASRec input stage with side features (replay/nn/embedding.py, replay/nn/agg.py:44-53,
// replay/nn/sequential/sasrec/agg.py:37-53):
//
//   s_t = E_item[id_t] + sum_cat E_f[id_f,t] + sum_bag bag_f(E_f, ids_f,t) + sum_num v_f,t . W_f^T + b_f + sum_ident v_f,t
//   x_t = dropout(s_t * scale + P[pos0 + t % L])
//
// One warp per token gathers every row, so the summed input is rounded to bf16 once, as the reference rounds nothing.  The
// numerical projections run in the same pass: their summed tensor_dim is at most RP_FEAT_MAX_NUM_COLS, so a lane's dot
// products are a few dozen FMAs per column on a weight slab that stays in L1, while a separate GEMM would need a bf16
// staging copy of the values and a second read-modify-write pass over [T, d].  The dropout stream is rp_embed_fwd's (row
// key = the token index, embedding site 0), so an item-only model and a side-feature model drop the same elements.
//
// Backward (rp_embed_bwd keeps the item table and the positions): dS = scale * dropout'(dx) is scattered into the side
// tables with fp32 atomics (padding rows frozen, mean bags scaled by 1 / count), and written as bf16 next to the gathered
// numerical values, the operands of the weight-gradient GEMM (rp_wgrad_group) that gives dW and db in a fixed order.
//
// The BERT form (template flag BERT; legacy bert4rec/model.py:173-296, BertEmbedding with sum aggregation):
//
//   s_t = E_item[id_t] + sum_cat E_f[id_f,t] + sum_ident v_f,t
//   x_t = dropout(where(token_mask_t, s_t, mask_emb) + P[t % L])        (no sqrt(d) scale; P optional)
//
// Its categorical tables have no padding row (the host passes padding_value = -1), and its dropout is rp_bert_embed_fwd's
// stream.  Backward: dS = dropout'(dx) goes to the side tables at the real, unmasked tokens only; rp_bert_embed_bwd keeps
// the item table, mask_emb and the positions.  The SASRec instantiations compile none of this.
#include "rp_b200.h"
#include "rp_host.h"
#include "rp_philox.cuh"
#include "rp_sm90.cuh"

namespace rp {

struct FeatArgs {
  rp_feature f[RP_FEAT_MAX];
  int n;
};

// true feature index of padded column c (head slots of 64 / 128 columns with hd_valid real features each), -1 for padding
__device__ __forceinline__ int feat_true_col(int c, int hd_valid) {
  if (hd_valid == 0) return c;
  const int slot = hd_valid <= 64 ? 64 : 128, j = c % slot;
  return j < hd_valid ? (c / slot) * hd_valid + j : -1;
}

__device__ __forceinline__ bool feat_live(int id, const rp_feature& f) {
  return id != f.padding_value && id >= 0 && id < f.n_rows;
}

template <int VEC>
__device__ __forceinline__ void add_row(float* acc, const __nv_bfloat16* row, float w) {
#pragma unroll
  for (int i = 0; i < VEC; i += 2) {
    const float2 v = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(row + i));
    acc[i] += v.x * w;
    acc[i + 1] += v.y * w;
  }
}

// acc[0, VEC) += sum_f term_f(t) over columns [c0, c0 + VEC) (the kinds of rp_feature_embed_fwd; BERT: CAT and IDENT)
template <int VEC, bool BERT>
__device__ __forceinline__ void add_features(float* acc, const FeatArgs& fa, int t, int c0, int hd_valid) {
  constexpr int D = VEC * 32;
  for (int k = 0; k < fa.n; ++k) {
    const rp_feature& f = fa.f[k];
    if (f.kind == RP_FEAT_CAT || (!BERT && (f.kind == RP_FEAT_BAG_SUM || f.kind == RP_FEAT_BAG_MEAN))) {
      const int32_t* v = reinterpret_cast<const int32_t*>(f.values) + (size_t)t * f.width;
      const __nv_bfloat16* tab = reinterpret_cast<const __nv_bfloat16*>(f.table);
      float bag[VEC];
#pragma unroll
      for (int i = 0; i < VEC; ++i) bag[i] = 0.f;
      int cnt = 0;
      for (int j = 0; j < f.width; ++j) {
        const int id = v[j];
        if (!feat_live(id, f)) continue;
        add_row<VEC>(bag, tab + (size_t)id * D + c0, 1.f);
        ++cnt;
      }
      const float w = (f.kind == RP_FEAT_BAG_MEAN && cnt > 0) ? 1.f / (float)cnt : 1.f;
#pragma unroll
      for (int i = 0; i < VEC; ++i) acc[i] += bag[i] * w;
    } else if (!BERT && f.kind == RP_FEAT_NUM) {
      const float* v = reinterpret_cast<const float*>(f.values) + (size_t)t * f.width;
      const float* W = reinterpret_cast<const float*>(f.table);
#pragma unroll
      for (int i = 0; i < VEC; ++i) acc[i] += f.bias[c0 + i];
      for (int j = 0; j < f.width; ++j) {
        const float vj = v[j];
#pragma unroll
        for (int i = 0; i < VEC; ++i) acc[i] += vj * W[(size_t)(c0 + i) * f.width + j];
      }
    } else {  // RP_FEAT_IDENT: the values are the embedding (true features only; padded columns stay zero)
      const float* v = reinterpret_cast<const float*>(f.values) + (size_t)t * f.width;
#pragma unroll
      for (int i = 0; i < VEC; ++i) {
        const int tc = feat_true_col(c0 + i, hd_valid);
        if (tc >= 0) acc[i] += v[tc];
      }
    }
  }
}

// row r of the output is token row_tok[r] (packed rows, *n_rows_dev of them) or token r (row_tok == null, n_tok rows)
// BERT: tok_mask / mask_emb replace the masked tokens' sum, pos may be null, scale is not applied (only CAT and IDENT kinds)
template <int VEC, bool BERT>
__global__ void __launch_bounds__(256, VEC >= 16 ? 2 : 4) feature_embed_fwd_kernel(
    const __nv_bfloat16* __restrict__ item, const float* __restrict__ pos, const int32_t* __restrict__ ids, const __grid_constant__ FeatArgs fa,
    int n_tok, int L, int hd_valid, int pos0, float scale, float drop_p, unsigned long long seed, unsigned long long drop_off,
    const unsigned long long* __restrict__ seed_ptr, const int32_t* __restrict__ row_tok, const int32_t* __restrict__ n_rows_dev,
    const uint8_t* __restrict__ tok_mask, const __nv_bfloat16* __restrict__ mask_emb, __nv_bfloat16* __restrict__ out) {
  if (drop_p > 0.f && seed_ptr) seed += *seed_ptr;
  constexpr int D = VEC * 32;
  const int n = n_rows_dev ? *n_rows_dev : n_tok;
  const int lane = threadIdx.x & 31, wpb = blockDim.x >> 5;
  const int c0 = lane * VEC;
  const uint32_t thr = drop_p > 0.f ? (uint32_t)(drop_p * 4294967296.0) : 0u;
  const float ks = drop_p > 0.f ? 1.f / (1.f - drop_p) : 1.f;
  for (int r = blockIdx.x * wpb + (threadIdx.x >> 5); r < n; r += gridDim.x * wpb) {
    const int t = row_tok ? row_tok[r] : r;
    float acc[VEC];
#pragma unroll
    for (int i = 0; i < VEC; ++i) acc[i] = 0.f;
    // BERT's <MASK> and pad tokens take mask_emb in place of the whole sum, so nothing else is gathered for them
    const bool masked = BERT && !tok_mask[t];
    add_row<VEC>(acc, masked ? mask_emb + c0 : item + (size_t)ids[t] * D + c0, 1.f);
    if (!masked) add_features<VEC, BERT>(acc, fa, t, c0, hd_valid);
    if (BERT) {
      if (pos) {
        const float* p = pos + (size_t)(t % L) * D + c0;
#pragma unroll
        for (int i = 0; i < VEC; ++i) acc[i] += p[i];
      }
    } else {
      const float* p = pos + (size_t)(pos0 + t % L) * D + c0;
#pragma unroll
      for (int i = 0; i < VEC; ++i) acc[i] = acc[i] * scale + p[i];
    }
    if (drop_p > 0.f) {
      const uint32_t rk = drop_row_key(seed, drop_off, (unsigned long long)t);
#pragma unroll
      for (int i = 0; i < VEC; ++i) acc[i] = drop_mix(rk, drop_col_key((uint32_t)(c0 + i))) >= thr ? acc[i] * ks : 0.f;
    }
    __nv_bfloat16* o = out + (size_t)r * D + c0;
#pragma unroll
    for (int i = 0; i < VEC; i += 2) *reinterpret_cast<uint32_t*>(o + i) = pack_bf16(acc[i], acc[i + 1]);
  }
}

template <int VEC>
__device__ __forceinline__ void scatter_row(float* dst, const float* g, float w) {
  if constexpr (VEC % 4 == 0) {
#pragma unroll
    for (int i = 0; i < VEC; i += 4) atomicAdd(reinterpret_cast<float4*>(dst + i), make_float4(g[i] * w, g[i + 1] * w, g[i + 2] * w, g[i + 3] * w));
  } else {
#pragma unroll
    for (int i = 0; i < VEC; i += 2) atomicAdd(reinterpret_cast<float2*>(dst + i), make_float2(g[i] * w, g[i + 1] * w));
  }
}

// BERT: only tokens with pad_mask && tok_mask reach the tables (a masked token's sum was replaced by mask_emb); CAT only
template <int VEC, bool BERT>
__global__ void __launch_bounds__(256, VEC >= 16 ? 2 : 4) feature_embed_bwd_kernel(
    const __nv_bfloat16* __restrict__ dx, const __grid_constant__ FeatArgs fa, int n_tok, float scale, float drop_p, unsigned long long seed,
    unsigned long long drop_off, const unsigned long long* __restrict__ seed_ptr, const int32_t* __restrict__ row_tok,
    const int32_t* __restrict__ n_rows_dev, __nv_bfloat16* __restrict__ d_s, __nv_bfloat16* __restrict__ v_rows, int v_ld,
    const uint8_t* __restrict__ pad_mask, const uint8_t* __restrict__ tok_mask) {
  if (drop_p > 0.f && seed_ptr) seed += *seed_ptr;
  constexpr int D = VEC * 32;
  const int n = n_rows_dev ? *n_rows_dev : n_tok;
  const int lane = threadIdx.x & 31, wpb = blockDim.x >> 5;
  const int c0 = lane * VEC;
  const uint32_t thr = drop_p > 0.f ? (uint32_t)(drop_p * 4294967296.0) : 0u;
  const float ks = (drop_p > 0.f ? 1.f / (1.f - drop_p) : 1.f) * scale;
  for (int r = blockIdx.x * wpb + (threadIdx.x >> 5); r < n; r += gridDim.x * wpb) {
    const int t = row_tok ? row_tok[r] : r;
    if (BERT && !(pad_mask[t] && tok_mask[t])) continue;
    float g[VEC];
    const __nv_bfloat16* gx = dx + (size_t)r * D + c0;
#pragma unroll
    for (int i = 0; i < VEC; i += 2) {
      const float2 v = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(gx + i));
      g[i] = v.x * ks;
      g[i + 1] = v.y * ks;
    }
    if (drop_p > 0.f) {
      const uint32_t rk = drop_row_key(seed, drop_off, (unsigned long long)t);
#pragma unroll
      for (int i = 0; i < VEC; ++i)
        if (drop_mix(rk, drop_col_key((uint32_t)(c0 + i))) < thr) g[i] = 0.f;
    }
    if (!BERT && d_s) {
      __nv_bfloat16* o = d_s + (size_t)r * D + c0;
#pragma unroll
      for (int i = 0; i < VEC; i += 2) *reinterpret_cast<uint32_t*>(o + i) = pack_bf16(g[i], g[i + 1]);
    }
    if (!BERT && v_rows)  // zero the staging row first: its numerical columns are written below, the padding columns stay zero
      for (int j = lane; j < v_ld; j += 32) v_rows[(size_t)r * v_ld + j] = __float2bfloat16(0.f);
    __syncwarp();
    for (int k = 0; k < fa.n; ++k) {
      const rp_feature& f = fa.f[k];
      if (f.kind == RP_FEAT_CAT || (!BERT && (f.kind == RP_FEAT_BAG_SUM || f.kind == RP_FEAT_BAG_MEAN))) {
        const int32_t* v = reinterpret_cast<const int32_t*>(f.values) + (size_t)t * f.width;
        float w = 1.f;
        if (!BERT && f.kind == RP_FEAT_BAG_MEAN) {
          int cnt = 0;
          for (int j = 0; j < f.width; ++j) cnt += feat_live(v[j], f);
          w = cnt > 0 ? 1.f / (float)cnt : 0.f;
        }
        for (int j = 0; j < f.width; ++j) {
          const int id = v[j];
          if (feat_live(id, f)) scatter_row<VEC>(f.d_table + (size_t)id * D + c0, g, w);
        }
      } else if (!BERT && f.kind == RP_FEAT_NUM && v_rows) {
        const float* v = reinterpret_cast<const float*>(f.values) + (size_t)t * f.width;
        for (int j = lane; j < f.width; j += 32) v_rows[(size_t)r * v_ld + f.val_col + j] = __float2bfloat16(v[j]);
      }
    }
  }
}

// ---- ConcatAggregator (replay/nn/agg.py:56-109): every feature at its own width, concatenated in the order the host gives
// (the reference sorts by feature name), then Linear(sum of widths, d) on the tensor cores (rp_gemm).  One warp per row and
// one column per lane and step: segment widths are arbitrary (11, 13, ...), so nothing is vector-loaded and neither the side
// tables nor the segment offsets need padding.  Each segment value is summed in fp32 and rounded to bf16 once.
struct ConcatArgs {
  rp_feature f[RP_FEAT_MAX];
  int col[RP_FEAT_MAX], dim[RP_FEAT_MAX];   // first column and width of feature k's segment
  int n, item_col;
};

// padded column of true feature j (the inverse of feat_true_col)
__device__ __forceinline__ int feat_pad_col(int j, int hd_valid) {
  if (hd_valid == 0) return j;
  return (j / hd_valid) * (hd_valid <= 64 ? 64 : 128) + j % hd_valid;
}

// x[r, :] = [segments | zeros up to kp] for row r (token row_tok[r] on packed rows, *n_rows_dev of them)
__global__ void __launch_bounds__(256) concat_gather_kernel(
    const __nv_bfloat16* __restrict__ item, const int32_t* __restrict__ ids, const __grid_constant__ ConcatArgs ca, int n_tok,
    int D, int d_true, int hd_valid, int width, int kp, const int32_t* __restrict__ row_tok,
    const int32_t* __restrict__ n_rows_dev, __nv_bfloat16* __restrict__ x) {
  const int n = n_rows_dev ? *n_rows_dev : n_tok;
  const int lane = threadIdx.x & 31, wpb = blockDim.x >> 5;
  for (int r = blockIdx.x * wpb + (threadIdx.x >> 5); r < n; r += gridDim.x * wpb) {
    const int t = row_tok ? row_tok[r] : r;
    __nv_bfloat16* o = x + (size_t)r * kp;
    for (int c = width + lane; c < kp; c += 32) o[c] = __float2bfloat16(0.f);
    const __nv_bfloat16* it = item + (size_t)ids[t] * D;
    for (int j = lane; j < d_true; j += 32) o[ca.item_col + j] = it[feat_pad_col(j, hd_valid)];
    for (int k = 0; k < ca.n; ++k) {
      const rp_feature& f = ca.f[k];
      const int w = ca.dim[k];
      __nv_bfloat16* seg = o + ca.col[k];
      if (f.kind == RP_FEAT_CAT || f.kind == RP_FEAT_BAG_SUM || f.kind == RP_FEAT_BAG_MEAN) {
        const int32_t* v = reinterpret_cast<const int32_t*>(f.values) + (size_t)t * f.width;
        const __nv_bfloat16* tab = reinterpret_cast<const __nv_bfloat16*>(f.table);
        int cnt = 0;
        for (int i = 0; i < f.width; ++i) cnt += feat_live(v[i], f);
        const float s = (f.kind == RP_FEAT_BAG_MEAN && cnt > 0) ? 1.f / (float)cnt : 1.f;
        for (int j = lane; j < w; j += 32) {
          float acc = 0.f;
          for (int i = 0; i < f.width; ++i) {
            const int id = v[i];
            if (feat_live(id, f)) acc += __bfloat162float(tab[(size_t)id * w + j]);
          }
          seg[j] = __float2bfloat16(acc * s);
        }
      } else if (f.kind == RP_FEAT_NUM) {   // v . W^T + b at the feature's own width, W fp32 [w, tensor_dim]
        const float* v = reinterpret_cast<const float*>(f.values) + (size_t)t * f.width;
        const float* W = reinterpret_cast<const float*>(f.table);
        for (int j = lane; j < w; j += 32) {
          float acc = f.bias[j];
          for (int i = 0; i < f.width; ++i) acc += v[i] * W[(size_t)j * f.width + i];
          seg[j] = __float2bfloat16(acc);
        }
      } else {   // RP_FEAT_IDENT: the values themselves (width == w)
        const float* v = reinterpret_cast<const float*>(f.values) + (size_t)t * f.width;
        for (int j = lane; j < w; j += 32) seg[j] = __float2bfloat16(v[j]);
      }
    }
  }
}

// out[r] = dropout(y[r] * scale + pos[pos0 + t % L]), y fp32 [rows, D] = the projection (bias included); the dropout stream of
// rp_embed_fwd (row key = token t, embedding site drop_off), so a concat model drops what the item-only model drops
template <int VEC>
__global__ void __launch_bounds__(256) concat_embed_fwd_kernel(
    const float* __restrict__ y, const float* __restrict__ pos, int n_tok, int L, int pos0, float scale, float drop_p,
    unsigned long long seed, unsigned long long drop_off, const unsigned long long* __restrict__ seed_ptr,
    const int32_t* __restrict__ row_tok, const int32_t* __restrict__ n_rows_dev, __nv_bfloat16* __restrict__ out) {
  if (drop_p > 0.f && seed_ptr) seed += *seed_ptr;
  constexpr int D = VEC * 32;
  const int n = n_rows_dev ? *n_rows_dev : n_tok;
  const int lane = threadIdx.x & 31, wpb = blockDim.x >> 5;
  const int c0 = lane * VEC;
  const uint32_t thr = drop_p > 0.f ? (uint32_t)(drop_p * 4294967296.0) : 0u;
  const float ks = drop_p > 0.f ? 1.f / (1.f - drop_p) : 1.f;
  for (int r = blockIdx.x * wpb + (threadIdx.x >> 5); r < n; r += gridDim.x * wpb) {
    const int t = row_tok ? row_tok[r] : r;
    const float* yr = y + (size_t)r * D + c0;
    const float* p = pos + (size_t)(pos0 + t % L) * D + c0;
    float acc[VEC];
#pragma unroll
    for (int i = 0; i < VEC; ++i) acc[i] = yr[i] * scale + p[i];
    if (drop_p > 0.f) {
      const uint32_t rk = drop_row_key(seed, drop_off, (unsigned long long)t);
#pragma unroll
      for (int i = 0; i < VEC; ++i) acc[i] = drop_mix(rk, drop_col_key((uint32_t)(c0 + i))) >= thr ? acc[i] * ks : 0.f;
    }
    __nv_bfloat16* o = out + (size_t)r * D + c0;
#pragma unroll
    for (int i = 0; i < VEC; i += 2) *reinterpret_cast<uint32_t*>(o + i) = pack_bf16(acc[i], acc[i + 1]);
  }
}

// dX = dY . W (bf16 [rows, kp]) into the tables: the item segment into d_item (pad_id frozen), categorical segments into their
// d_table (padding rows frozen, mean bags by 1 / count); numerical values staged into v_rows for their dW / db
__global__ void __launch_bounds__(256) concat_scatter_kernel(
    const __nv_bfloat16* __restrict__ dx, const int32_t* __restrict__ ids, float* __restrict__ d_item, int pad_id,
    const __grid_constant__ ConcatArgs ca, int n_tok, int D, int d_true, int hd_valid, int kp, const int32_t* __restrict__ row_tok,
    const int32_t* __restrict__ n_rows_dev, __nv_bfloat16* __restrict__ v_rows, int v_ld) {
  const int n = n_rows_dev ? *n_rows_dev : n_tok;
  const int lane = threadIdx.x & 31, wpb = blockDim.x >> 5;
  for (int r = blockIdx.x * wpb + (threadIdx.x >> 5); r < n; r += gridDim.x * wpb) {
    const int t = row_tok ? row_tok[r] : r;
    const __nv_bfloat16* g = dx + (size_t)r * kp;
    const int id = ids[t];
    if (id != pad_id) {
      float* dst = d_item + (size_t)id * D;
      for (int j = lane; j < d_true; j += 32) atomicAdd(dst + feat_pad_col(j, hd_valid), __bfloat162float(g[ca.item_col + j]));
    }
    if (v_rows)   // zero the staging row first: its numerical columns are written below, the other columns stay zero
      for (int j = lane; j < v_ld; j += 32) v_rows[(size_t)r * v_ld + j] = __float2bfloat16(0.f);
    __syncwarp();
    for (int k = 0; k < ca.n; ++k) {
      const rp_feature& f = ca.f[k];
      const int w = ca.dim[k];
      const __nv_bfloat16* seg = g + ca.col[k];
      if (f.kind == RP_FEAT_CAT || f.kind == RP_FEAT_BAG_SUM || f.kind == RP_FEAT_BAG_MEAN) {
        const int32_t* v = reinterpret_cast<const int32_t*>(f.values) + (size_t)t * f.width;
        float s = 1.f;
        if (f.kind == RP_FEAT_BAG_MEAN) {
          int cnt = 0;
          for (int i = 0; i < f.width; ++i) cnt += feat_live(v[i], f);
          s = cnt > 0 ? 1.f / (float)cnt : 0.f;
        }
        for (int i = 0; i < f.width; ++i) {
          const int fid = v[i];
          if (!feat_live(fid, f)) continue;
          float* dst = f.d_table + (size_t)fid * w;
          for (int j = lane; j < w; j += 32) atomicAdd(dst + j, __bfloat162float(seg[j]) * s);
        }
      } else if (f.kind == RP_FEAT_NUM && v_rows) {
        const float* v = reinterpret_cast<const float*>(f.values) + (size_t)t * f.width;
        for (int j = lane; j < f.width; j += 32) v_rows[(size_t)r * v_ld + f.val_col + j] = __float2bfloat16(v[j]);
      }
    }
  }
}


// ---- TwoTower's item tower input (replay/nn/sequential/twotower/model.py ItemTower.forward -> embedder -> SumAggregator):
//
//   X0[r] = E_item[i] + sum_f term_f(reader_f[i]),   i = item_of_slot[r] (compacted candidates) or item0 + r (the catalog)
//
// No scale, position or dropout.  The reader's values are indexed by item id, so the feature terms are add_features' own.
// Rows from *n_slots on are written as zeros, as rp_tower_compact leaves its rows there.
template <int VEC>
__global__ void __launch_bounds__(256, VEC >= 16 ? 2 : 4) item_feature_fwd_kernel(
    const __nv_bfloat16* __restrict__ item, const __grid_constant__ FeatArgs fa, int n_rows, int item0, int hd_valid,
    const int32_t* __restrict__ item_of_slot, const int32_t* __restrict__ n_slots, __nv_bfloat16* __restrict__ out) {
  constexpr int D = VEC * 32;
  const int live = item_of_slot ? min(*n_slots, n_rows) : n_rows;
  const int lane = threadIdx.x & 31, wpb = blockDim.x >> 5;
  const int c0 = lane * VEC;
  for (int r = blockIdx.x * wpb + (threadIdx.x >> 5); r < n_rows; r += gridDim.x * wpb) {
    float acc[VEC];
#pragma unroll
    for (int i = 0; i < VEC; ++i) acc[i] = 0.f;
    if (r < live) {
      const int t = item_of_slot ? item_of_slot[r] : item0 + r;
      add_row<VEC>(acc, item + (size_t)t * D + c0, 1.f);
      add_features<VEC, false>(acc, fa, t, c0, hd_valid);
    }
    __nv_bfloat16* o = out + (size_t)r * D + c0;
#pragma unroll
    for (int i = 0; i < VEC; i += 2) *reinterpret_cast<uint32_t*>(o + i) = pack_bf16(acc[i], acc[i + 1]);
  }
}

// Full-catalog backward of the categorical tables in a fixed order (rp_item_feature_plan): pass 1 sums each chunk's entries,
// partial[c] = sum_e w_e * dx[item_e]; pass 2 adds each (feature, table row) group's chunk partials, in chunk order, into its
// d_table row.  Every group has one owner, so the stores are plain and the result is the same bits on every run.
template <int VEC>
__global__ void __launch_bounds__(256) item_feature_chunk_kernel(const __nv_bfloat16* __restrict__ dx,
                                                                 const rp_item_feature_plan plan) {
  constexpr int D = VEC * 32;
  const int lane = threadIdx.x & 31, wpb = blockDim.x >> 5;
  const int c0 = lane * VEC;
  for (int c = blockIdx.x * wpb + (threadIdx.x >> 5); c < plan.n_chunks; c += gridDim.x * wpb) {
    float acc[VEC];
#pragma unroll
    for (int i = 0; i < VEC; ++i) acc[i] = 0.f;
    for (int e = plan.chunk_off[c]; e < plan.chunk_off[c + 1]; ++e)
      add_row<VEC>(acc, dx + (size_t)plan.ent_item[e] * D + c0, plan.ent_w[e]);
    float* p = plan.partial + (size_t)c * D + c0;
#pragma unroll
    for (int i = 0; i < VEC; ++i) p[i] = acc[i];
  }
}

template <int VEC>
__global__ void __launch_bounds__(256) item_feature_group_kernel(const __grid_constant__ FeatArgs fa,
                                                                 const rp_item_feature_plan plan) {
  constexpr int D = VEC * 32;
  const int lane = threadIdx.x & 31, wpb = blockDim.x >> 5;
  const int c0 = lane * VEC;
  for (int g = blockIdx.x * wpb + (threadIdx.x >> 5); g < plan.n_groups; g += gridDim.x * wpb) {
    float acc[VEC];
#pragma unroll
    for (int i = 0; i < VEC; ++i) acc[i] = 0.f;
    for (int c = plan.grp_chunk[g]; c < plan.grp_chunk[g + 1]; ++c) {
      const float* p = plan.partial + (size_t)c * D + c0;
#pragma unroll
      for (int i = 0; i < VEC; ++i) acc[i] += p[i];
    }
    float* dst = fa.f[plan.grp_feat[g]].d_table + (size_t)plan.grp_row[g] * D + c0;
#pragma unroll
    for (int i = 0; i < VEC; ++i) dst[i] += acc[i];
  }
}

}  // namespace rp

using namespace rp;

#define RP_FEAT_DISPATCH(d, CALL)                      \
  switch (d) {                                         \
    case 64: { constexpr int VEC = 2; CALL; } break;   \
    case 128: { constexpr int VEC = 4; CALL; } break;  \
    case 256: { constexpr int VEC = 8; CALL; } break;  \
    case 512: { constexpr int VEC = 16; CALL; } break; \
    default: return RP_ESHAPE;                         \
  }

static inline int feat_grid(long long rows) {   // one warp per row, about 8 blocks of 8 warps per SM
  long long b = (rows + 7) / 8;
  const long long cap = (long long)sm_count() * 8;
  return (int)(b > cap ? cap : (b < 1 ? 1 : b));
}

// shared argument checks: RP_EINVAL for a null pointer or unknown kind, RP_ESHAPE for a size the kernels do not take
// bert: the BERT form, which takes the CAT and IDENT kinds only
static int feat_args(const rp_feature* feats, int n_feats, int d, int hd_valid, bool bwd, int v_ld, FeatArgs* fa,
                     bool bert = false) {
  if (n_feats < 0 || n_feats > RP_FEAT_MAX || (n_feats > 0 && !feats)) return n_feats < 0 || n_feats > RP_FEAT_MAX ? RP_ESHAPE : RP_EINVAL;
  if (hd_valid < 0 || hd_valid > 128 || (hd_valid > 0 && d % (hd_valid <= 64 ? 64 : 128))) return RP_ESHAPE;
  const int d_true = hd_valid ? d / (hd_valid <= 64 ? 64 : 128) * hd_valid : d;
  int num_cols = 0;
  fa->n = n_feats;
  for (int k = 0; k < n_feats; ++k) {
    const rp_feature& f = feats[k];
    if (!f.values) return RP_EINVAL;
    if (bert && f.kind != RP_FEAT_CAT && f.kind != RP_FEAT_IDENT) return RP_EINVAL;
    if (f.width <= 0) return RP_ESHAPE;
    switch (f.kind) {
      case RP_FEAT_CAT:
      case RP_FEAT_BAG_SUM:
      case RP_FEAT_BAG_MEAN:
        if (!f.table || (bwd && !f.d_table)) return RP_EINVAL;
        if (f.n_rows <= 0 || (f.kind == RP_FEAT_CAT && f.width != 1)) return RP_ESHAPE;
        break;
      case RP_FEAT_NUM:
        if (!f.table || !f.bias) return RP_EINVAL;
        if (f.val_col != num_cols) return RP_ESHAPE;   // consecutive columns of the staging rows, in feature order
        num_cols += f.width;
        break;
      case RP_FEAT_IDENT:
        if (f.width != d_true) return RP_ESHAPE;
        break;
      default:
        return RP_EINVAL;
    }
    fa->f[k] = f;
  }
  if (num_cols > RP_FEAT_MAX_NUM_COLS) return RP_ESHAPE;
  if (bwd && num_cols > 0 && (v_ld < num_cols || v_ld % 8)) return RP_ESHAPE;
  return RP_OK;
}

static int feature_fwd(const void* item_table, const float* pos, const int32_t* ids, const rp_feature* feats, int n_feats,
                       const int32_t* row_tok, const int32_t* n_rows_dev, int T, int L, int d, int hd_valid, int pos0,
                       float scale, float drop_p, unsigned long long seed, unsigned long long drop_off,
                       const unsigned long long* seed_ptr, void* out, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (!item_table || !pos || !ids || !out || T <= 0 || L <= 0 || pos0 < 0) return RP_EINVAL;
  if (drop_p < 0.f || drop_p >= 1.f) return RP_EINVAL;
  FeatArgs fa;
  const int rc = feat_args(feats, n_feats, d, hd_valid, false, 0, &fa);
  if (rc != RP_OK) return rc;
  const int grid = feat_grid(T);
  RP_FEAT_DISPATCH(d, (feature_embed_fwd_kernel<VEC, false><<<grid, 256, 0, stream>>>(
                          reinterpret_cast<const __nv_bfloat16*>(item_table), pos, ids, fa, T, L, hd_valid, pos0, scale, drop_p,
                          seed, drop_off, seed_ptr, row_tok, n_rows_dev, nullptr, nullptr, reinterpret_cast<__nv_bfloat16*>(out))));
  RP_LAUNCH_CHECK();
  return RP_OK;
}

static int feature_bwd(const void* dx, const rp_feature* feats, int n_feats, const int32_t* row_tok, const int32_t* n_rows_dev,
                       int T, int d, int hd_valid, float scale, float drop_p, unsigned long long seed,
                       unsigned long long drop_off, const unsigned long long* seed_ptr, void* d_s, void* v_rows, int v_ld,
                       void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (!dx || T <= 0) return RP_EINVAL;
  if (drop_p < 0.f || drop_p >= 1.f) return RP_EINVAL;
  FeatArgs fa;
  const int rc = feat_args(feats, n_feats, d, hd_valid, true, v_ld, &fa);
  if (rc != RP_OK) return rc;
  bool has_num = false;
  for (int k = 0; k < n_feats; ++k) has_num |= feats[k].kind == RP_FEAT_NUM;
  if (has_num && (!d_s || !v_rows)) return RP_EINVAL;
  const int grid = feat_grid(T);
  RP_FEAT_DISPATCH(d, (feature_embed_bwd_kernel<VEC, false><<<grid, 256, 0, stream>>>(
                          reinterpret_cast<const __nv_bfloat16*>(dx), fa, T, scale, drop_p, seed, drop_off, seed_ptr, row_tok,
                          n_rows_dev, reinterpret_cast<__nv_bfloat16*>(d_s), reinterpret_cast<__nv_bfloat16*>(v_rows), v_ld,
                          nullptr, nullptr)));
  RP_LAUNCH_CHECK();
  return RP_OK;
}

RP_API int rp_feature_embed_fwd(const void* item_table, const float* pos, const int32_t* ids, const rp_feature* feats,
                                int n_feats, int T, int L, int d, int hd_valid, int pos0, float scale, float drop_p,
                                unsigned long long seed, unsigned long long drop_off, const unsigned long long* seed_ptr,
                                void* out, void* stream) {
  return feature_fwd(item_table, pos, ids, feats, n_feats, nullptr, nullptr, T, L, d, hd_valid, pos0, scale, drop_p, seed,
                     drop_off, seed_ptr, out, stream);
}

RP_API int rp_feature_embed_fwd_rows(const void* item_table, const float* pos, const int32_t* ids, const rp_feature* feats,
                                     int n_feats, const int32_t* row_tok, const int32_t* n_rows_dev, int T, int L, int d,
                                     int hd_valid, int pos0, float scale, float drop_p, unsigned long long seed,
                                     unsigned long long drop_off, const unsigned long long* seed_ptr, void* out, void* stream) {
  if (!row_tok || !n_rows_dev) return RP_EINVAL;
  return feature_fwd(item_table, pos, ids, feats, n_feats, row_tok, n_rows_dev, T, L, d, hd_valid, pos0, scale, drop_p, seed,
                     drop_off, seed_ptr, out, stream);
}

RP_API int rp_feature_embed_bwd(const void* dx, const rp_feature* feats, int n_feats, int T, int d, int hd_valid, float scale,
                                float drop_p, unsigned long long seed, unsigned long long drop_off,
                                const unsigned long long* seed_ptr, void* d_s, void* v_rows, int v_ld, void* stream) {
  return feature_bwd(dx, feats, n_feats, nullptr, nullptr, T, d, hd_valid, scale, drop_p, seed, drop_off, seed_ptr, d_s, v_rows,
                     v_ld, stream);
}

RP_API int rp_feature_embed_bwd_rows(const void* dx, const rp_feature* feats, int n_feats, const int32_t* row_tok,
                                     const int32_t* n_rows_dev, int T, int d, int hd_valid, float scale, float drop_p,
                                     unsigned long long seed, unsigned long long drop_off, const unsigned long long* seed_ptr,
                                     void* d_s, void* v_rows, int v_ld, void* stream) {
  if (!row_tok || !n_rows_dev) return RP_EINVAL;
  return feature_bwd(dx, feats, n_feats, row_tok, n_rows_dev, T, d, hd_valid, scale, drop_p, seed, drop_off, seed_ptr, d_s,
                     v_rows, v_ld, stream);
}

// ---- the BERT form (legacy BERT4Rec's BertEmbedding over side features): see the top of this file and include/rp_b200.h
RP_API int rp_bert_feature_embed_fwd(const void* item_table, const void* mask_emb, const float* pos, const int32_t* ids,
                                     const uint8_t* tok_mask, const rp_feature* feats, int n_feats, int T, int L, int d,
                                     int hd_valid, float drop_p, unsigned long long seed, unsigned long long drop_off,
                                     const unsigned long long* seed_ptr, void* out, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  // pos == null: no positional term (enable_positional_embedding=False)
  if (!item_table || !mask_emb || !ids || !tok_mask || !out || T <= 0 || L <= 0) return RP_EINVAL;
  if (drop_p < 0.f || drop_p >= 1.f) return RP_EINVAL;
  if (T % L != 0) return RP_ESHAPE;
  FeatArgs fa;
  const int rc = feat_args(feats, n_feats, d, hd_valid, false, 0, &fa, true);
  if (rc != RP_OK) return rc;
  const int grid = feat_grid(T);
  RP_FEAT_DISPATCH(d, (feature_embed_fwd_kernel<VEC, true><<<grid, 256, 0, stream>>>(
                          reinterpret_cast<const __nv_bfloat16*>(item_table), pos, ids, fa, T, L, hd_valid, 0, 1.f, drop_p, seed,
                          drop_off, seed_ptr, nullptr, nullptr, tok_mask, reinterpret_cast<const __nv_bfloat16*>(mask_emb),
                          reinterpret_cast<__nv_bfloat16*>(out))));
  RP_LAUNCH_CHECK();
  return RP_OK;
}

RP_API int rp_bert_feature_embed_bwd(const void* dx, const uint8_t* pad_mask, const uint8_t* tok_mask, const rp_feature* feats,
                                     int n_feats, int T, int d, int hd_valid, float drop_p, unsigned long long seed,
                                     unsigned long long drop_off, const unsigned long long* seed_ptr, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (!dx || !pad_mask || !tok_mask || T <= 0) return RP_EINVAL;
  if (drop_p < 0.f || drop_p >= 1.f) return RP_EINVAL;
  FeatArgs fa;
  const int rc = feat_args(feats, n_feats, d, hd_valid, true, 0, &fa, true);
  if (rc != RP_OK) return rc;
  const int grid = feat_grid(T);
  RP_FEAT_DISPATCH(d, (feature_embed_bwd_kernel<VEC, true><<<grid, 256, 0, stream>>>(
                          reinterpret_cast<const __nv_bfloat16*>(dx), fa, T, 1.f, drop_p, seed, drop_off, seed_ptr, nullptr,
                          nullptr, nullptr, nullptr, 0, pad_mask, tok_mask)));
  RP_LAUNCH_CHECK();
  return RP_OK;
}

// ---- ConcatAggregator: see the ConcatArgs comment above and include/rp_b200.h
// RP_EINVAL for a null pointer or unknown kind; RP_ESHAPE unless the segments (the item's d_true columns at item_col, feature
// k's seg_dim[k] at seg_col[k]) tile [0, width) exactly, kp is a multiple of 64 in [width, RP_CONCAT_MAX_COLS], identity
// widths equal their segment and the numerical columns are consecutive (at most RP_FEAT_MAX_NUM_COLS)
static int concat_args(const rp_feature* feats, const int* seg_col, const int* seg_dim, int n_feats, int item_col, int d,
                       int hd_valid, int kp, bool bwd, ConcatArgs* ca, int* d_true, int* width) {
  if (n_feats < 0 || n_feats > RP_FEAT_MAX) return RP_ESHAPE;
  if (n_feats > 0 && (!feats || !seg_col || !seg_dim)) return RP_EINVAL;
  if (d != 64 && d != 128 && d != 256 && d != 512) return RP_ESHAPE;
  if (hd_valid < 0 || hd_valid > 128 || (hd_valid > 0 && d % (hd_valid <= 64 ? 64 : 128))) return RP_ESHAPE;
  *d_true = hd_valid ? d / (hd_valid <= 64 ? 64 : 128) * hd_valid : d;
  if (kp <= 0 || kp % 64 || kp > RP_CONCAT_MAX_COLS) return RP_ESHAPE;
  // the segments tile [0, width): sorted by first column, each starts where the previous one ends
  int lo[RP_FEAT_MAX + 1], hi[RP_FEAT_MAX + 1];
  lo[0] = item_col;
  hi[0] = item_col + *d_true;
  int num_cols = 0;
  ca->n = n_feats;
  ca->item_col = item_col;
  for (int k = 0; k < n_feats; ++k) {
    const rp_feature& f = feats[k];
    const int w = seg_dim[k];
    if (!f.values) return RP_EINVAL;
    if (f.width <= 0 || w <= 0 || seg_col[k] < 0) return RP_ESHAPE;
    switch (f.kind) {
      case RP_FEAT_CAT:
      case RP_FEAT_BAG_SUM:
      case RP_FEAT_BAG_MEAN:
        if (!f.table || (bwd && !f.d_table)) return RP_EINVAL;
        if (f.n_rows <= 0 || (f.kind == RP_FEAT_CAT && f.width != 1)) return RP_ESHAPE;
        break;
      case RP_FEAT_NUM:
        if (!f.table || !f.bias) return RP_EINVAL;
        if (f.val_col != num_cols) return RP_ESHAPE;
        num_cols += f.width;
        break;
      case RP_FEAT_IDENT:
        if (f.width != w) return RP_ESHAPE;
        break;
      default:
        return RP_EINVAL;
    }
    ca->f[k] = f;
    ca->col[k] = seg_col[k];
    ca->dim[k] = w;
    lo[k + 1] = seg_col[k];
    hi[k + 1] = seg_col[k] + w;
  }
  if (num_cols > RP_FEAT_MAX_NUM_COLS) return RP_ESHAPE;
  int end = 0;
  for (int done = 0; done <= n_feats; ++done) {   // n <= 17 segments: find the one starting at `end`, n times
    int next = -1;
    for (int k = 0; k <= n_feats; ++k)
      if (lo[k] == end) next = k;
    if (next < 0) return RP_ESHAPE;
    end = hi[next];
  }
  if (end > kp) return RP_ESHAPE;
  *width = end;
  return RP_OK;
}

static int concat_gather(const void* item_table, const int32_t* ids, const rp_feature* feats, const int* seg_col,
                         const int* seg_dim, int n_feats, int item_col, const int32_t* row_tok, const int32_t* n_rows_dev,
                         int T, int d, int hd_valid, int kp, void* x, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (!item_table || !ids || !x || T <= 0) return RP_EINVAL;
  ConcatArgs ca;
  int d_true, width;
  const int rc = concat_args(feats, seg_col, seg_dim, n_feats, item_col, d, hd_valid, kp, false, &ca, &d_true, &width);
  if (rc != RP_OK) return rc;
  concat_gather_kernel<<<feat_grid(T), 256, 0, stream>>>(reinterpret_cast<const __nv_bfloat16*>(item_table), ids, ca, T, d,
                                                         d_true, hd_valid, width, kp, row_tok, n_rows_dev,
                                                         reinterpret_cast<__nv_bfloat16*>(x));
  RP_LAUNCH_CHECK();
  return RP_OK;
}

RP_API int rp_concat_gather(const void* item_table, const int32_t* ids, const rp_feature* feats, const int* seg_col,
                            const int* seg_dim, int n_feats, int item_col, int T, int d, int hd_valid, int kp, void* x,
                            void* stream) {
  return concat_gather(item_table, ids, feats, seg_col, seg_dim, n_feats, item_col, nullptr, nullptr, T, d, hd_valid, kp, x,
                       stream);
}

RP_API int rp_concat_gather_rows(const void* item_table, const int32_t* ids, const rp_feature* feats, const int* seg_col,
                                 const int* seg_dim, int n_feats, int item_col, const int32_t* row_tok,
                                 const int32_t* n_rows_dev, int T, int d, int hd_valid, int kp, void* x, void* stream) {
  if (!row_tok || !n_rows_dev) return RP_EINVAL;
  return concat_gather(item_table, ids, feats, seg_col, seg_dim, n_feats, item_col, row_tok, n_rows_dev, T, d, hd_valid, kp, x,
                       stream);
}

RP_API int rp_concat_embed_fwd(const float* y, const float* pos, const int32_t* row_tok, const int32_t* n_rows_dev, int T,
                               int L, int d, int pos0, float scale, float drop_p, unsigned long long seed,
                               unsigned long long drop_off, const unsigned long long* seed_ptr, void* out, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (!y || !pos || !out || T <= 0 || L <= 0 || pos0 < 0 || (!row_tok != !n_rows_dev)) return RP_EINVAL;
  if (drop_p < 0.f || drop_p >= 1.f) return RP_EINVAL;
  const int grid = feat_grid(T);
  RP_FEAT_DISPATCH(d, (concat_embed_fwd_kernel<VEC><<<grid, 256, 0, stream>>>(y, pos, T, L, pos0, scale, drop_p, seed,
                                                                              drop_off, seed_ptr, row_tok, n_rows_dev,
                                                                              reinterpret_cast<__nv_bfloat16*>(out))));
  RP_LAUNCH_CHECK();
  return RP_OK;
}

RP_API int rp_concat_scatter(const void* dx, const int32_t* ids, float* d_item, int pad_id, const rp_feature* feats,
                             const int* seg_col, const int* seg_dim, int n_feats, int item_col, const int32_t* row_tok,
                             const int32_t* n_rows_dev, int T, int d, int hd_valid, int kp, void* v_rows, int v_ld,
                             void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (!dx || !ids || !d_item || T <= 0 || (!row_tok != !n_rows_dev)) return RP_EINVAL;
  ConcatArgs ca;
  int d_true, width;
  const int rc = concat_args(feats, seg_col, seg_dim, n_feats, item_col, d, hd_valid, kp, true, &ca, &d_true, &width);
  if (rc != RP_OK) return rc;
  int num_cols = 0;
  for (int k = 0; k < n_feats; ++k) num_cols += feats[k].kind == RP_FEAT_NUM ? feats[k].width : 0;
  if (num_cols > 0 && !v_rows) return RP_EINVAL;
  if (v_rows && (v_ld < num_cols || v_ld % 8)) return RP_ESHAPE;
  concat_scatter_kernel<<<feat_grid(T), 256, 0, stream>>>(reinterpret_cast<const __nv_bfloat16*>(dx), ids, d_item, pad_id, ca,
                                                          T, d, d_true, hd_valid, kp, row_tok, n_rows_dev,
                                                          reinterpret_cast<__nv_bfloat16*>(v_rows), v_ld);
  RP_LAUNCH_CHECK();
  return RP_OK;
}

// ---- TwoTower's item tower input: see item_feature_fwd_kernel above and include/rp_b200.h
RP_API int rp_item_feature_embed_fwd(const void* item_table, const rp_feature* feats, int n_feats, const int32_t* item_of_slot,
                                     const int32_t* n_slots, int n_rows, int item0, int d, int hd_valid, void* out,
                                     void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (!item_table || !out || n_rows <= 0 || item0 < 0 || (item_of_slot && !n_slots)) return RP_EINVAL;
  FeatArgs fa;
  const int rc = feat_args(feats, n_feats, d, hd_valid, false, 0, &fa);
  if (rc != RP_OK) return rc;
  const int grid = feat_grid(n_rows);
  RP_FEAT_DISPATCH(d, (item_feature_fwd_kernel<VEC><<<grid, 256, 0, stream>>>(
                          reinterpret_cast<const __nv_bfloat16*>(item_table), fa, n_rows, item0, hd_valid, item_of_slot, n_slots,
                          reinterpret_cast<__nv_bfloat16*>(out))));
  RP_LAUNCH_CHECK();
  return RP_OK;
}

RP_API int rp_item_feature_embed_bwd(const void* dx, const rp_feature* feats, int n_feats, const int32_t* item_of_slot,
                                     const int32_t* n_slots, int n_rows, int d, int hd_valid, const rp_item_feature_plan* plan,
                                     void* v_rows, int v_ld, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (!dx || n_rows <= 0 || (item_of_slot && !n_slots) || (!item_of_slot && !plan)) return RP_EINVAL;
  FeatArgs fa;
  const int rc = feat_args(feats, n_feats, d, hd_valid, true, v_ld, &fa);
  if (rc != RP_OK) return rc;
  bool has_num = false;
  for (int k = 0; k < n_feats; ++k) has_num |= feats[k].kind == RP_FEAT_NUM;
  if (has_num && item_of_slot && !v_rows) return RP_EINVAL;
  const int grid = feat_grid(n_rows);
  if (item_of_slot) {   // at most cap rows, one slot per item: fp32 atomics into the table rows, values staged per slot
    RP_FEAT_DISPATCH(d, (feature_embed_bwd_kernel<VEC, false><<<grid, 256, 0, stream>>>(
                            reinterpret_cast<const __nv_bfloat16*>(dx), fa, n_rows, 1.f, 0.f, 0ull, 0ull, nullptr, item_of_slot,
                            n_slots, nullptr, reinterpret_cast<__nv_bfloat16*>(v_rows), v_ld, nullptr, nullptr)));
    RP_LAUNCH_CHECK();
    return RP_OK;
  }
  if (plan->n_chunks < 0 || plan->n_groups < 0) return RP_ESHAPE;
  if (plan->n_chunks > 0 && (!plan->ent_item || !plan->ent_w || !plan->chunk_off || !plan->partial)) return RP_EINVAL;
  if (plan->n_groups > 0 && (!plan->grp_chunk || !plan->grp_feat || !plan->grp_row)) return RP_EINVAL;
  if (has_num && v_rows) {   // the values of the numerical features only: no table row is touched here
    FeatArgs nf;
    nf.n = 0;
    for (int k = 0; k < n_feats; ++k)
      if (feats[k].kind == RP_FEAT_NUM) nf.f[nf.n++] = feats[k];
    RP_FEAT_DISPATCH(d, (feature_embed_bwd_kernel<VEC, false><<<grid, 256, 0, stream>>>(
                            reinterpret_cast<const __nv_bfloat16*>(dx), nf, n_rows, 1.f, 0.f, 0ull, 0ull, nullptr, nullptr,
                            nullptr, nullptr, reinterpret_cast<__nv_bfloat16*>(v_rows), v_ld, nullptr, nullptr)));
    RP_LAUNCH_CHECK();
  }
  if (plan->n_chunks > 0) {
    RP_FEAT_DISPATCH(d, (item_feature_chunk_kernel<VEC><<<feat_grid(plan->n_chunks), 256, 0, stream>>>(
                            reinterpret_cast<const __nv_bfloat16*>(dx), *plan)));
    RP_LAUNCH_CHECK();
  }
  if (plan->n_groups > 0) {
    RP_FEAT_DISPATCH(d, (item_feature_group_kernel<VEC><<<feat_grid(plan->n_groups), 256, 0, stream>>>(fa, *plan)));
    RP_LAUNCH_CHECK();
  }
  return RP_OK;
}
