// rp_attention.cu - padded-sequence multi-head attention for L <= 512, head_dim 64 or 128 (SASRec causal + key-padding, BERT4Rec key-padding):
// fused forward on wgmma (S = Q.K^T in registers -> masked softmax in registers -> P bf16 as the register A operand of O = P.V),
// the row-wise softmax backward that sits between the batched backward GEMMs (rp_gemm), and the fused backward (below).
//
// Replaces torch.nn.MultiheadAttention's scaled-dot-product core as configured by the reference:
//   replay/nn/sequential/sasrec/transformer.py:36-46,99-106 + replay/nn/mask.py:18-51 (float [B*H,L,L] mask never built)
//   replay/models/nn/sequential/sasrec/model.py:407-414,435 (bool causal mask, pad keys NOT masked)
//   replay/models/nn/sequential/bert4rec/model.py:471,494 (key_padding_mask only)
// Fully masked query rows produce a zero output (torch >= 2.5 safe-softmax semantics of the training path).
#include "rp_host.h"
#include "rp_philox.cuh"
#include "rp_sm90.cuh"

namespace rp {

struct AttnParams {
  int B, H, L, Lp;             // Lp = round_up(L, 64): row pitch / row count of the saved probability buffers
  int causal, mask_pad_keys;
  float scale;                 // 1/sqrt(head_dim)
  const uint8_t* pad_mask;     // [B*L] 1 = real token
  __nv_bfloat16* out;          // [B*L, ldo] ; head h writes columns [h*HD, (h+1)*HD)
  int ldo;
  __nv_bfloat16* p_save;       // [B*H, Lp, Lp] unnormalised exp(s - max) (bf16) or null
  float* inv_sum;              // [B*H, Lp] 1 / row sum (0 for fully masked rows)
  float* m_save;               // [B*H, Lp] row max in exp2 units (max * scale * log2e), for the fused backward; or null
  int q_c0, k_c0, v_c0;        // column offsets of head 0 inside the Q / K / V 2-D arrays
  float drop_p;
  unsigned long long seed, drop_off;
  const unsigned long long* seed_ptr;
  // packed rows (training, head_dim 64, L <= 256): sequence b owns rows [seq_off[b], seq_off[b] + L - seq_first[b]) of q / k / v
  // / out, its positions seq_first[b] .. L - 1; null = padded rows b * L + position
  const int32_t* seq_first;
  const int32_t* seq_off;
};

static constexpr float kLog2eA = 1.4426950408889634f;

static constexpr int kAfThreads = 256;  // two warpgroups: query rows [0, 64) and [64, 128) of the tile
static constexpr int kAfVStages = 3;    // V ring of attn_fwd_kernel<128, 2>: 64-key stages of 16 KB

// KB = number of 256-key blocks the CTA keeps resident (1: L <= 256, 2: L <= 512).  Q, K and V of the tile stay in shared
// memory; each warpgroup walks the visible keys in 64-key chunks twice: pass 1 takes the row max of S = Q.K^T, pass 2
// recomputes the chunk, forms P = exp(S - max) in registers (saved un-dropped to p_save if asked, then dropped) and
// accumulates O += P.V with P as the register A operand.  Chunks entirely above the causal diagonal of a warpgroup's rows
// are skipped (their P is zero).
//
// <128, 2> (STREAM_V): 512 keys of K and V at 128 head dims do not both fit in shared memory.  Q and K stay resident, so
// pass 1 is the same; V streams through a ring of kAfVStages 64-key stages (TMA box [64 rows x 64 columns], tmV built with a
// 64-row box), loaded by thread 0 ahead of pass 2.  Both warpgroups walk every loaded chunk of the tile - a warpgroup whose
// rows see none of the chunk's keys skips the MMA - and every thread releases a stage once its wgmma on it has completed,
// so the "empty" barrier always counts kAfThreads arrivals and thread 0 refills the stage after both warpgroups let it go.
// <64, 1> (81 KB of shared memory) is held to 128 registers so that two CTAs share an SM: one's loads and softmax overlap
// the other's MMAs.
template <int HD, int KB>
__global__ void __launch_bounds__(kAfThreads, (HD == 64 && KB == 1) ? 2 : 1)
attn_fwd_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
                const __grid_constant__ CUtensorMap tmV, const AttnParams p) {
  constexpr int HC = HD / 64;                 // 64-wide head-dim chunks
  constexpr int Q_BYTES = HC * 128 * 128;     // [128 x HD]
  constexpr int KV_CHUNK = KB * 256 * 128;    // one 64-wide head-dim chunk of all resident keys
  constexpr int KV_BYTES = HC * KV_CHUNK;     // [256*KB x HD]
  constexpr bool STREAM_V = HD == 128 && KB == 2;
  constexpr int V_STAGE = HC * 64 * 128;      // one 64-key chunk of V: HC boxes of [64 x 64], 8 KB apart
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sQ = smem;
  uint8_t* sK = sQ + Q_BYTES;
  uint8_t* sV = sK + KV_BYTES;                // STREAM_V: the ring, then its full / empty barriers
  uint64_t* v_full = reinterpret_cast<uint64_t*>(sV + kAfVStages * V_STAGE);
  uint64_t* v_empty = v_full + kAfVStages;
  __shared__ __align__(16) uint32_t s_colkey[256 * KB];   // dropout key of every key position
  __shared__ uint8_t s_keyok[256 * KB];                    // key position is real (j < L, and not padding if masked)
  __shared__ uint64_t bar_load;

  const int q0 = blockIdx.x * 128, h = blockIdx.y, b = blockIdx.z;
  const int bz = b * p.H + h;
  const int L = p.L;
  // packed rows: the sequence's rows hold positions first .. L - 1 from row seq_off[b] on.  The CTA's window starts `lead`
  // rows earlier, at the 64-aligned position `shift`, so that its 64-key chunks cover the same positions as in the padded
  // layout (every row sums the same products in the same order); the lead rows belong to the sequence before and are
  // masked as keys and never stored.  Local index = position - shift; masks and dropout keys use the position.
  const bool packed = p.seq_first != nullptr;
  const int first = packed ? p.seq_first[b] : 0;
  const int lead = first & 63, shift = first - lead;
  const int n = L - shift;
  const int row0 = packed ? p.seq_off[b] - lead : b * L;
  if (packed && q0 >= n) return;   // no live query in this tile: nothing reads its rows
  // Inference: a query tile whose rows are ALL padding (left-padded windows: the first tile of every user with at most L - 128
  // items) produces nothing anybody reads - the new path masks pad positions as keys and never queries them, the legacy
  // path zeroes pad rows after the block.  Such a CTA writes zeros and leaves before any load or MMA.  (Training keeps the
  // rows: the backward reads their saved statistics.)
  if (p.pad_mask && p.inv_sum == nullptr && p.p_save == nullptr && p.m_save == nullptr) {
    const int r = q0 + (int)threadIdx.x;
    const int live = (threadIdx.x < 128 && r < L) ? (p.pad_mask[(size_t)b * L + r] != 0) : 0;
    if (!__syncthreads_or(live)) {
      // 128 rows x HD bf16 of this head: 16-byte stores, HD / 8 per row
      constexpr int PER_ROW = HD / 8;
      for (int i = threadIdx.x; i < 128 * PER_ROW; i += blockDim.x) {
        const int rr = q0 + i / PER_ROW;
        if (rr < L)
          *reinterpret_cast<uint4*>(p.out + ((size_t)b * L + rr) * p.ldo + h * HD + (i % PER_ROW) * 8) = make_uint4(0u, 0u, 0u, 0u);
      }
      return;
    }
  }
  const int nk = p.causal ? min(n, q0 + 128) : n;  // keys that can be visible to this query tile
  const int nk32 = (nk + 31) & ~31;                // extent of the saved probability rows
  const int n_boxes = (nk32 + 127) / 128;
  const int n64 = (nk32 + 63) / 64;

  // STREAM_V: 64-key chunk ch of V into stage ch % kAfVStages
  auto v_load = [&](int ch) {
    uint64_t* full = v_full + ch % kAfVStages;
    mbar_arrive_expect_tx(full, V_STAGE);
    for (int c = 0; c < HC; ++c)
      tma_load_2d(sV + (ch % kAfVStages) * V_STAGE + c * 8192, &tmV, full, p.v_c0 + h * HD + c * 64, row0 + ch * 64);
  };
  if (threadIdx.x == 0) {
    mbar_init(&bar_load, 1);
    if constexpr (STREAM_V)
      for (int s = 0; s < kAfVStages; ++s) {
        mbar_init(v_full + s, 1);
        mbar_init(v_empty + s, kAfThreads);
      }
    fence_barrier_init();
    mbar_arrive_expect_tx(&bar_load, HC * 128 * 128 + (STREAM_V ? 1 : 2) * HC * n_boxes * 128 * 128);
    for (int c = 0; c < HC; ++c) {
      tma_load_2d(sQ + c * 16384, &tmQ, &bar_load, p.q_c0 + h * HD + c * 64, row0 + q0);
      for (int bx = 0; bx < n_boxes; ++bx) {
        tma_load_2d(sK + c * KV_CHUNK + bx * 16384, &tmK, &bar_load, p.k_c0 + h * HD + c * 64, row0 + bx * 128);
        if constexpr (!STREAM_V)
          tma_load_2d(sV + c * KV_CHUNK + bx * 16384, &tmV, &bar_load, p.v_c0 + h * HD + c * 64, row0 + bx * 128);
      }
    }
    if constexpr (STREAM_V)
      for (int ch = 0; ch < min(kAfVStages, n64); ++ch) v_load(ch);
  }
  for (int j = threadIdx.x; j < 256 * KB; j += kAfThreads) {
    s_colkey[j] = p.drop_p > 0.f ? drop_col_key((uint32_t)(shift + j)) : 0u;
    s_keyok[j] = (j >= lead && j < n) && (!p.mask_pad_keys || p.pad_mask[(size_t)b * L + shift + j] != 0);
  }
  __syncthreads();

  const int t = threadIdx.x & 127, wg = threadIdx.x >> 7;
  const int fr = frag_row(t), fc = frag_col(t);
  const int ia = q0 + 64 * wg + fr, ib = ia + 8;   // the two query rows of this thread
  const int wg_last = q0 + 64 * wg + 63;           // last query row of the warpgroup
  const int n_live = p.causal ? min(n64, wg_last / 64 + 1) : n64;  // chunks with a visible key for some row of the warpgroup
  const float sl2 = p.scale * kLog2eA;
  const bool drop = p.drop_p > 0.f;
  const uint32_t thr = drop ? (uint32_t)(p.drop_p * 4294967296.0) : 0u;
  const float ks_drop = drop ? 1.f / (1.f - p.drop_p) : 1.f;
  const unsigned long long seed_eff = p.seed + ((drop && p.seed_ptr) ? *p.seed_ptr : 0ull);
  const uint32_t rk_a = drop ? drop_row_key(seed_eff, p.drop_off, (unsigned long long)bz * p.Lp + (unsigned long long)(shift + ia)) : 0u;
  const uint32_t rk_b = drop ? drop_row_key(seed_eff, p.drop_off, (unsigned long long)bz * p.Lp + (unsigned long long)(shift + ib)) : 0u;
  auto visible = [&](int key, int i) -> bool { return s_keyok[key] && (!p.causal || key <= i); };
  const uint32_t q_base = smem_u32(sQ) + wg * 8192;
  auto qk_chunk = [&](float (&sacc)[32], int j0) {
    wg_fence();
#pragma unroll
    for (int c = 0; c < HC; ++c)
#pragma unroll
      for (int ks = 0; ks < 4; ++ks)
        WgmmaSS<64>::template run<0, 0>(sacc, desc_k(q_base + c * 16384 + ks * 32),
                                        desc_k(smem_u32(sK) + c * KV_CHUNK + j0 * 128 + ks * 32), (c | ks) != 0);
    wg_commit();
    wg_wait<0>();
    wg_fence_acc(sacc);
  };
  mbar_wait(&bar_load, 0);
  if constexpr (!STREAM_V) {
    if (packed) {
      // rows [n, n_boxes * 128) of the loaded boxes belong to the next sequence or to no sequence (stale rows past the packed
      // count, possibly not finite): their probabilities are zero, but 0 * Inf / NaN in O += P.V is not, so the value rows are
      // cleared (the lead rows are rows of the sequence before: finite)
      const int n_pad = n_boxes * 128 - n;
      for (int i = threadIdx.x; i < HC * max(n_pad, 0) * 8; i += kAfThreads) {
        const int c = i / (max(n_pad, 1) * 8), r = n + (i / 8) % max(n_pad, 1);
        *reinterpret_cast<uint4*>(sV + c * KV_CHUNK + r * 128 + (i % 8) * 16) = make_uint4(0u, 0u, 0u, 0u);
      }
      fence_proxy_async();
      __syncthreads();
    }
  }

  // ---- pass 1: row max over the visible keys
  float mxa = -INFINITY, mxb = -INFINITY;
  for (int ch = 0; ch < n_live; ++ch) {
    float sacc[32];
    qk_chunk(sacc, ch * 64);
#pragma unroll
    for (int j = 0; j < 8; ++j)
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int key = ch * 64 + 8 * j + fc + e;
        if (visible(key, ia)) mxa = fmaxf(mxa, sacc[4 * j + e]);
        if (visible(key, ib)) mxb = fmaxf(mxb, sacc[4 * j + 2 + e]);
      }
  }
#pragma unroll
  for (int o = 1; o <= 2; o <<= 1) {
    mxa = fmaxf(mxa, __shfl_xor_sync(0xffffffffu, mxa, o));
    mxb = fmaxf(mxb, __shfl_xor_sync(0xffffffffu, mxb, o));
  }
  const float moa = (mxa == -INFINITY) ? 0.f : mxa * sl2, mob = (mxb == -INFINITY) ? 0.f : mxb * sl2;

  // ---- pass 2: P = exp2(S * scale * log2e - max), row sums, optional copy of the un-dropped P, O += P.V
  const bool own_a = ia >= lead && ia < n, own_b = ib >= lead && ib < n;   // rows of this sequence
  // saved probability of query row i, key `key` (formed where it is stored: two row pointers held across pass 2 would
  // cost the registers that let attn_fwd_kernel<64, 1> run two CTAs per SM)
  auto p_at = [&](int i, int key) { return reinterpret_cast<uint32_t*>(p.p_save + ((size_t)bz * p.Lp + i) * p.Lp + key); };
  float oacc[HD / 2];
  acc_zero(oacc);
  float suma = 0.f, sumb = 0.f;
  // STREAM_V: hand stage ch back once this thread's wgmma on it has completed; thread 0 refills it with chunk ch + kAfVStages
  // after all kAfThreads threads have
  auto v_release = [&](int ch) {
    mbar_arrive(v_empty + ch % kAfVStages);
    if (threadIdx.x == 0 && ch + kAfVStages < n64) {
      mbar_wait(v_empty + ch % kAfVStages, (ch / kAfVStages) & 1);
      v_load(ch + kAfVStages);
    }
    __syncwarp();
  };
  const int n_walk = STREAM_V ? n64 : n_live;
  for (int ch = 0; ch < n_walk; ++ch) {
    if constexpr (STREAM_V) {
      mbar_wait(v_full + ch % kAfVStages, (ch / kAfVStages) & 1);
      if (ch >= n_live) {
        v_release(ch);
        continue;
      }
    }
    float sacc[32];
    qk_chunk(sacc, ch * 64);
    uint32_t pk[16];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int key = ch * 64 + 8 * j + fc;
      float ea[2], eb[2];
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        ea[e] = visible(key + e, ia) ? ex2f(fmaf(sacc[4 * j + e], sl2, -moa)) : 0.f;
        eb[e] = visible(key + e, ib) ? ex2f(fmaf(sacc[4 * j + 2 + e], sl2, -mob)) : 0.f;
        suma += ea[e];
        sumb += eb[e];
      }
      if (key < nk32) {
        if (p.p_save && own_a) *p_at(ia, key) = pack_bf16(ea[0], ea[1]);
        if (p.p_save && own_b) *p_at(ib, key) = pack_bf16(eb[0], eb[1]);
      }
      if (drop) {
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const uint32_t ck = s_colkey[key + e];
          ea[e] = drop_mix(rk_a, ck) >= thr ? ea[e] * ks_drop : 0.f;
          eb[e] = drop_mix(rk_b, ck) >= thr ? eb[e] * ks_drop : 0.f;
        }
      }
      pk[2 * j] = pack_bf16(ea[0], ea[1]);
      pk[2 * j + 1] = pack_bf16(eb[0], eb[1]);
    }
    wg_fence();
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {  // 16 keys per step: A fragment = P columns [16 kk, 16 kk + 16) of the chunk
      const uint32_t a[4] = {pk[4 * kk], pk[4 * kk + 1], pk[4 * kk + 2], pk[4 * kk + 3]};
      if constexpr (STREAM_V)
        WgmmaRS<HD>::template run<1>(oacc, a, desc_mn(smem_u32(sV) + (ch % kAfVStages) * V_STAGE + kk * 2048, 8192), 1);
      else
        WgmmaRS<HD>::template run<1>(oacc, a, desc_mn(smem_u32(sV) + (ch * 4 + kk) * 2048, KV_CHUNK), 1);
    }
    wg_commit();
    wg_wait<0>();
    wg_fence_acc(oacc);
    if constexpr (STREAM_V) v_release(ch);
  }
  // probability rows of the chunks above the diagonal of this warpgroup are zero
  for (int ch = n_live; ch < n64; ++ch)
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int key = ch * 64 + 8 * j + fc;
      if (key < nk32) {
        if (p.p_save && own_a) *p_at(ia, key) = 0u;
        if (p.p_save && own_b) *p_at(ib, key) = 0u;
      }
    }
#pragma unroll
  for (int o = 1; o <= 2; o <<= 1) {
    suma += __shfl_xor_sync(0xffffffffu, suma, o);
    sumb += __shfl_xor_sync(0xffffffffu, sumb, o);
  }
  const float inva = suma > 0.f ? 1.f / suma : 0.f, invb = sumb > 0.f ? 1.f / sumb : 0.f;
  if (fc == 0) {
    if (own_a) {
      if (p.inv_sum) p.inv_sum[(size_t)bz * p.Lp + ia] = inva;
      if (p.m_save) p.m_save[(size_t)bz * p.Lp + ia] = moa;
    }
    if (own_b) {
      if (p.inv_sum) p.inv_sum[(size_t)bz * p.Lp + ib] = invb;
      if (p.m_save) p.m_save[(size_t)bz * p.Lp + ib] = mob;
    }
  }
  // ---- O = (P.V) / sum
#pragma unroll
  for (int j = 0; j < HD / 8; ++j) {
    const int c = h * HD + 8 * j + fc;
    if (own_a) *reinterpret_cast<uint32_t*>(p.out + ((size_t)row0 + ia) * p.ldo + c) = pack_bf16(oacc[4 * j] * inva, oacc[4 * j + 1] * inva);
    if (own_b) *reinterpret_cast<uint32_t*>(p.out + ((size_t)row0 + ib) * p.ldo + c) = pack_bf16(oacc[4 * j + 2] * invb, oacc[4 * j + 3] * invb);
  }
}

// Row-wise softmax backward between the batched GEMMs.  One warp per (batch*head, query) row.
//   in : p_save  = exp(s - max) (bf16), inv_sum, dpd = dO.V^T (bf16, w.r.t. the dropped & rescaled probabilities)
//   out: ds (over dpd) = P * (dP - sum_j P_j dP_j) * scale      with P = p_save * inv_sum, dP = dpd * mask / keep
//        pd (over p_save) = P * mask / keep                       (A operand of dV = Pd^T . dO)
template <int NK>  // 128-column blocks per row: Lp <= 128 * NK
__global__ void attn_softmax_bwd_kernel(__nv_bfloat16* __restrict__ p_save, __nv_bfloat16* __restrict__ dpd,
                                        const float* __restrict__ inv_sum, int BH, int L, int Lp, float scale,
                                        float drop_p, unsigned long long seed, unsigned long long drop_off,
                                        const unsigned long long* __restrict__ seed_ptr) {
  if (drop_p > 0.f && seed_ptr) seed += *seed_ptr;
  const int lane = threadIdx.x & 31;
  const int wpb = blockDim.x >> 5;
  const uint32_t thr = drop_p > 0.f ? (uint32_t)(drop_p * 4294967296.0) : 0u;
  const float ksd = drop_p > 0.f ? 1.f / (1.f - drop_p) : 1.f;
  const long long n_rows = (long long)BH * L;
  uint32_t colkey[4 * NK];  // the lane's columns are the same in every row
#pragma unroll
  for (int k = 0; k < NK; ++k)
#pragma unroll
    for (int q = 0; q < 4; ++q) colkey[k * 4 + q] = drop_col_key((uint32_t)(k * 128 + lane * 4 + q));
  for (long long r = (long long)blockIdx.x * wpb + (threadIdx.x >> 5); r < n_rows; r += (long long)gridDim.x * wpb) {
    const int bz = (int)(r / L), i = (int)(r % L);
    const size_t base = ((size_t)bz * Lp + i) * Lp;
    const uint32_t row_key = drop_row_key(seed, drop_off, (unsigned long long)bz * Lp + (unsigned long long)i);
    const float inv = inv_sum[(size_t)bz * Lp + i];
    // lane owns columns [4*lane + 128*k, +4), k < NK   (columns >= L hold zeros and are never written)
    float P[4 * NK], dP[4 * NK], keep[4 * NK];
    float dot = 0.f;
#pragma unroll
    for (int k = 0; k < NK; ++k) {
      const int j0 = k * 128 + lane * 4;
#pragma unroll
      for (int q = 0; q < 4; ++q) { P[k * 4 + q] = 0.f; dP[k * 4 + q] = 0.f; keep[k * 4 + q] = 0.f; }
      if (j0 < L) {
        const uint2 pr = *reinterpret_cast<const uint2*>(p_save + base + j0);
        const uint2 dr = *reinterpret_cast<const uint2*>(dpd + base + j0);
        const __nv_bfloat162* ph = reinterpret_cast<const __nv_bfloat162*>(&pr);
        const __nv_bfloat162* dh = reinterpret_cast<const __nv_bfloat162*>(&dr);
        const float2 p0 = __bfloat1622float2(ph[0]), p1 = __bfloat1622float2(ph[1]);
        const float2 d0 = __bfloat1622float2(dh[0]), d1 = __bfloat1622float2(dh[1]);
        const float pv[4] = {p0.x, p0.y, p1.x, p1.y}, dv[4] = {d0.x, d0.y, d1.x, d1.y};
        uint32_t rv[4] = {0xffffffffu, 0xffffffffu, 0xffffffffu, 0xffffffffu};
        if (drop_p > 0.f) {
#pragma unroll
          for (int q = 0; q < 4; ++q) rv[q] = drop_mix(row_key, colkey[k * 4 + q]);
        }
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const bool in = (j0 + q) < L;
          keep[k * 4 + q] = (in && rv[q] >= thr) ? ksd : 0.f;
          P[k * 4 + q] = in ? pv[q] * inv : 0.f;
          dP[k * 4 + q] = dv[q] * keep[k * 4 + q];
          dot += P[k * 4 + q] * dP[k * 4 + q];
        }
      }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) dot += __shfl_xor_sync(0xffffffffu, dot, o);
#pragma unroll
    for (int k = 0; k < NK; ++k) {
      const int j0 = k * 128 + lane * 4;
      if (j0 < L) {
        float ds[4], pd[4];
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          ds[q] = P[k * 4 + q] * (dP[k * 4 + q] - dot) * scale;
          pd[q] = P[k * 4 + q] * keep[k * 4 + q];
        }
        uint2 w0, w1;
        w0.x = pack_bf16(ds[0], ds[1]); w0.y = pack_bf16(ds[2], ds[3]);
        w1.x = pack_bf16(pd[0], pd[1]); w1.y = pack_bf16(pd[2], pd[3]);
        *reinterpret_cast<uint2*>(dpd + base + j0) = w0;
        *reinterpret_cast<uint2*>(p_save + base + j0) = w1;
      }
    }
  }
}


// ------------------------------------------------------------------------------------------------------------------
// predict(): only the LAST position of every sequence is scored, so in the last transformer block a single query row per
// (sequence, head) attends to the keys - a memory-bound GEMV pair, one warp per (b, h).
//   q    bf16 [B, H*HD]   (compact: one row per sequence)
//   k, v bf16 rows b*L + j of 2-D arrays with pitches ldk / ldv, head h at columns x_c0 + h*HD
//   out  bf16 [B, H*HD]
// Visible keys: j < L (the query is the last position, so causal masking is a no-op) and, if mask_pad_keys, pad[b*L+j].
// ------------------------------------------------------------------------------------------------------------------
template <int HD>
__global__ void attn_last_kernel(const __nv_bfloat16* __restrict__ q, const __nv_bfloat16* __restrict__ k,
                                 const __nv_bfloat16* __restrict__ v, long long ldk, long long ldv, int k_c0, int v_c0,
                                 const uint8_t* __restrict__ pad_mask, int B, int H, int L, int mask_pad_keys, float scale,
                                 __nv_bfloat16* __restrict__ out) {
  constexpr int PER = HD / 32;  // output columns per lane
  __shared__ float s_q[8][HD];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const int bh = blockIdx.x * (blockDim.x >> 5) + w;
  if (bh >= B * H) return;
  const int b = bh / H, h = bh % H;
  for (int c = lane; c < HD; c += 32) s_q[w][c] = __bfloat162float(q[(size_t)b * H * HD + h * HD + c]) * scale;
  __syncwarp();
  // scores: lane owns keys lane, lane+32, ...
  float sc[16];  // L <= 512
  float mx = -INFINITY;
#pragma unroll
  for (int i = 0; i < 16; ++i) {
    const int j = i * 32 + lane;
    sc[i] = -INFINITY;
    if (j < L && (!mask_pad_keys || pad_mask[(size_t)b * L + j])) {
      const uint4* kr = reinterpret_cast<const uint4*>(k + ((size_t)b * L + j) * ldk + k_c0 + h * HD);
      float acc = 0.f;
#pragma unroll
      for (int c8 = 0; c8 < HD / 8; ++c8) {
        const uint4 raw = kr[c8];
        const __nv_bfloat162* h2 = reinterpret_cast<const __nv_bfloat162*>(&raw);
#pragma unroll
        for (int t = 0; t < 4; ++t) {
          const float2 f = __bfloat1622float2(h2[t]);
          acc = fmaf(f.x, s_q[w][c8 * 8 + 2 * t], fmaf(f.y, s_q[w][c8 * 8 + 2 * t + 1], acc));
        }
      }
      sc[i] = acc;
      mx = fmaxf(mx, acc);
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  float sum = 0.f;
#pragma unroll
  for (int i = 0; i < 16; ++i) {
    sc[i] = (sc[i] == -INFINITY) ? 0.f : __expf(sc[i] - mx);
    sum += sc[i];
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
  const float inv = sum > 0.f ? 1.f / sum : 0.f;  // no visible key -> zero output (safe-softmax semantics)
  // P.V: every lane accumulates the value rows of ITS keys (independent 16-byte loads, nothing serialised on a broadcast of
  // p_j), then a reduce-scatter butterfly over the lanes leaves HD/32 finished output columns per lane
  float o[HD];
#pragma unroll
  for (int c = 0; c < HD; ++c) o[c] = 0.f;
#pragma unroll
  for (int i = 0; i < 16; ++i) {
    const int j = i * 32 + lane;
    if (j < L && sc[i] != 0.f) {
      const uint4* vr = reinterpret_cast<const uint4*>(v + ((size_t)b * L + j) * ldv + v_c0 + h * HD);
      const float pj = sc[i];
#pragma unroll
      for (int c8 = 0; c8 < HD / 8; ++c8) {
        const uint4 raw = vr[c8];
        const __nv_bfloat162* h2 = reinterpret_cast<const __nv_bfloat162*>(&raw);
#pragma unroll
        for (int t = 0; t < 4; ++t) {
          const float2 f = __bfloat1622float2(h2[t]);
          o[c8 * 8 + 2 * t] = fmaf(pj, f.x, o[c8 * 8 + 2 * t]);
          o[c8 * 8 + 2 * t + 1] = fmaf(pj, f.y, o[c8 * 8 + 2 * t + 1]);
        }
      }
    }
  }
  int base = 0;
#define RP_RS_STEP(OFF, N)                                                     \
  {                                                                            \
    const bool up = (lane & OFF) != 0;                                         \
    _Pragma("unroll") for (int c = 0; c < N; ++c) {                            \
      const float send = up ? o[c] : o[c + N];                                 \
      const float recv = __shfl_xor_sync(0xffffffffu, send, OFF);              \
      o[c] = (up ? o[c + N] : o[c]) + recv;                                    \
    }                                                                          \
    base += up ? N : 0;                                                        \
  }
  RP_RS_STEP(16, HD / 2)
  RP_RS_STEP(8, HD / 4)
  RP_RS_STEP(4, HD / 8)
  RP_RS_STEP(2, HD / 16)
  RP_RS_STEP(1, HD / 32)
#undef RP_RS_STEP
  __nv_bfloat16* op = out + (size_t)b * H * HD + h * HD + base;
#pragma unroll
  for (int c = 0; c < PER; c += 2) *reinterpret_cast<uint32_t*>(op + c) = pack_bf16(o[c] * inv, o[c + 1] * inv);
}

}  // namespace rp

using namespace rp;

RP_API int rp_attn_last(const void* q, const void* k, const void* v, long long ldk, long long ldv, int k_c0, int v_c0,
                        const uint8_t* pad_mask, int B, int H, int L, int head_dim, int mask_pad_keys, void* out,
                        float scale_in, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (!q || !k || !v || !pad_mask || !out) return RP_EINVAL;
  if (B <= 0 || H <= 0 || L <= 0 || L > 512) return RP_ESHAPE;
  if ((ldk & 7) || (ldv & 7) || (k_c0 & 7) || (v_c0 & 7)) return RP_EALIGN;
  const float scale = scale_in > 0.f ? scale_in : 1.f / sqrtf((float)head_dim);
  const int blocks = (B * H + 7) / 8;
  const __nv_bfloat16 *qq = reinterpret_cast<const __nv_bfloat16*>(q), *kk = reinterpret_cast<const __nv_bfloat16*>(k),
                      *vv = reinterpret_cast<const __nv_bfloat16*>(v);
  if (head_dim == 64)
    attn_last_kernel<64><<<blocks, 256, 0, stream>>>(qq, kk, vv, ldk, ldv, k_c0, v_c0, pad_mask, B, H, L, mask_pad_keys, scale,
                                                     reinterpret_cast<__nv_bfloat16*>(out));
  else if (head_dim == 128)
    attn_last_kernel<128><<<blocks, 256, 0, stream>>>(qq, kk, vv, ldk, ldv, k_c0, v_c0, pad_mask, B, H, L, mask_pad_keys, scale,
                                                      reinterpret_cast<__nv_bfloat16*>(out));
  else
    return RP_ESHAPE;
  RP_LAUNCH_CHECK();
  return RP_OK;
}

struct rp_attn_desc {
  const void* q; long long q_rows, q_cols, ldq; int q_c0;
  const void* k; long long k_rows, k_cols, ldk; int k_c0;
  const void* v; long long v_rows, v_cols, ldv; int v_c0;
  int B, H, L, head_dim;
  int causal, mask_pad_keys;
  const uint8_t* pad_mask;
  void* out; int ldo;
  void* p_save; float* inv_sum;
  float drop_p; unsigned long long seed, drop_off; const unsigned long long* seed_ptr;
  float* m_save;
  float scale;
  const int32_t* seq_first; const int32_t* seq_off;
};

RP_API int rp_attn_fwd(const rp_attn_desc* a, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (!a || !a->q || !a->k || !a->v || !a->out || !a->pad_mask) return RP_EINVAL;
  if (a->L <= 0 || a->L > 512 || a->B <= 0 || a->H <= 0) return RP_ESHAPE;
  if (a->head_dim != 64 && a->head_dim != 128) return RP_ESHAPE;
  if (a->ldo % 8 != 0) return RP_EALIGN;
  AttnParams p;
  p.B = a->B; p.H = a->H; p.L = a->L; p.Lp = (a->L + 63) & ~63;
  p.causal = a->causal; p.mask_pad_keys = a->mask_pad_keys;
  p.scale = a->scale > 0.f ? a->scale : 1.f / sqrtf((float)a->head_dim);
  p.pad_mask = a->pad_mask;
  p.out = reinterpret_cast<__nv_bfloat16*>(a->out); p.ldo = a->ldo;
  p.p_save = reinterpret_cast<__nv_bfloat16*>(a->p_save); p.inv_sum = a->inv_sum; p.m_save = a->m_save;
  p.q_c0 = a->q_c0; p.k_c0 = a->k_c0; p.v_c0 = a->v_c0;
  p.drop_p = a->drop_p; p.seed = a->seed; p.drop_off = a->drop_off; p.seed_ptr = a->seed_ptr;
  p.seq_first = a->seq_first; p.seq_off = a->seq_off;
  if ((a->seq_first == nullptr) != (a->seq_off == nullptr)) return RP_EINVAL;
  if (a->seq_first && (a->head_dim != 64 || a->L > 256)) return RP_ESHAPE;
  if (a->seq_first && !a->causal) return RP_EINVAL;   // a lead row is never a visible key only under the causal mask
  CUtensorMap tmQ, tmK, tmV;
  int rc;
  if ((rc = make_tmap_bf16(&tmQ, a->q, a->q_rows, a->q_cols, a->ldq, 128)) != RP_OK) return rc;
  if ((rc = make_tmap_bf16(&tmK, a->k, a->k_rows, a->k_cols, a->ldk, 128)) != RP_OK) return rc;
  const bool stream_v = a->L > 256 && a->head_dim == 128;   // V through the 64-key ring of attn_fwd_kernel<128, 2>
  if ((rc = make_tmap_bf16(&tmV, a->v, a->v_rows, a->v_cols, a->ldv, stream_v ? 64 : 128)) != RP_OK) return rc;
  dim3 grid((a->L + 127) / 128, a->H, a->B);
  if (stream_v) {
    const int smem = 2 * (16384 + 65536) + kAfVStages * (16384 + 2 * 8) + 1024;
    RP_CUDA_CHECK(cudaFuncSetAttribute(attn_fwd_kernel<128, 2>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    attn_fwd_kernel<128, 2><<<grid, kAfThreads, smem, stream>>>(tmQ, tmK, tmV, p);
  } else if (a->L > 256) {
    const int smem = 16384 + 2 * 65536 + 1024;
    RP_CUDA_CHECK(cudaFuncSetAttribute(attn_fwd_kernel<64, 2>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    attn_fwd_kernel<64, 2><<<grid, kAfThreads, smem, stream>>>(tmQ, tmK, tmV, p);
  } else if (a->head_dim == 64) {
    const int smem = 16384 + 2 * 32768 + 1024;
    RP_CUDA_CHECK(cudaFuncSetAttribute(attn_fwd_kernel<64, 1>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    attn_fwd_kernel<64, 1><<<grid, kAfThreads, smem, stream>>>(tmQ, tmK, tmV, p);
  } else {
    const int smem = 2 * (16384 + 2 * 32768) + 1024;
    RP_CUDA_CHECK(cudaFuncSetAttribute(attn_fwd_kernel<128, 1>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    attn_fwd_kernel<128, 1><<<grid, kAfThreads, smem, stream>>>(tmQ, tmK, tmV, p);
  }
  RP_LAUNCH_CHECK();
  return RP_OK;
}

RP_API int rp_attn_softmax_bwd(void* p_save, void* dpd, const float* inv_sum, int BH, int L, float scale, float drop_p,
                               unsigned long long seed, unsigned long long drop_off, const unsigned long long* seed_ptr,
                               void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (!p_save || !dpd || !inv_sum || BH <= 0 || L <= 0 || L > 512) return RP_EINVAL;
  const int Lp = (L + 63) & ~63;
  const long long rows = (long long)BH * L;
  long long blocks = (rows + 7) / 8;
  const long long cap = (long long)sm_count() * 16;
  if (blocks > cap) blocks = cap;
  if (L > 256)
    attn_softmax_bwd_kernel<4><<<(int)blocks, 256, 0, stream>>>(reinterpret_cast<__nv_bfloat16*>(p_save),
                                                                reinterpret_cast<__nv_bfloat16*>(dpd), inv_sum, BH, L, Lp, scale,
                                                                drop_p, seed, drop_off, seed_ptr);
  else
    attn_softmax_bwd_kernel<2><<<(int)blocks, 256, 0, stream>>>(reinterpret_cast<__nv_bfloat16*>(p_save),
                                                                reinterpret_cast<__nv_bfloat16*>(dpd), inv_sum, BH, L, Lp, scale,
                                                                drop_p, seed, drop_off, seed_ptr);
  RP_LAUNCH_CHECK();
  return RP_OK;
}

// ==================================================================================================================
// Fused attention backward on wgmma for L <= 256, head_dim 64: one CTA per (sequence, head).
//
// Replaces autograd's backward of torch.nn.MultiheadAttention's SDPA core
// (replay/nn/sequential/sasrec/transformer.py:99-106, models/nn/sequential/sasrec/model.py:435, bert4rec/model.py:494)
// without materialising the [B*H, L, L] probability / gradient matrices the un-fused path needs.
//
// Q, K, V, dO and O of the (sequence, head) stay in shared memory.  The two warpgroups work on 64-row blocks:
//   phase 1, rows = keys (block kb):   for every 64-query step qs
//     S^T = K_kb . Q_qs^T, dP^T = V_kb . dO_qs^T       (registers)
//     P = exp2(s*sl2 - m_i) * inv_i (masked), dS = P * (dP * dropmask/keep - delta_i) * scale, Pd = P * dropmask/keep
//     dV_kb += Pd^T . dO_qs,  dK_kb += dS^T . Q_qs    (bf16 Pd^T / dS^T as register A operands)
//   phase 2, rows = queries (block qb): dQ_qb += dS_(qb,kb) . K_kb for every visible 64-key block kb
//     causal: phase 1 also stores each bf16 dS^T block in shared memory (the causal triangle, at most 10 blocks of 8 KB, in
//             place of O, which is dead once delta is formed), and phase 2 reads it as an MN-major A operand: MMAs only
//     non-causal: 16 blocks do not fit beside the operands; phase 2 recomputes S, dP and dS with rows = queries
// Every gradient element is summed by one warpgroup in a fixed order (deterministic, no atomics); causally empty blocks
// are skipped.  Row statistics m_i (max in exp2 units) and inv_i (1/rowsum) come from the forward; delta_i = sum_c dO[i,c] O[i,c].

namespace rp {

struct AttnBwdParams {
  int B, H, L, Lp;
  int causal, mask_pad_keys;
  float scale;
  const uint8_t* pad_mask;
  const float* m_save;         // [B*H, Lp]
  const float* inv_sum;        // [B*H, Lp]
  __nv_bfloat16* dQ; int ld_dq, dq_c0;   // outputs: rows b*L + i, columns x_c0 + h*64
  __nv_bfloat16* dK; int ld_dk, dk_c0;
  __nv_bfloat16* dV; int ld_dv, dv_c0;
  int q_c0, k_c0, v_c0;        // column offsets of head 0 inside the Q / K / V arrays (tensor maps)
  float drop_p;
  unsigned long long seed, drop_off;
  const unsigned long long* seed_ptr;
  const int32_t* seq_first;    // packed rows as in AttnParams (then the five maps are 2-D over the rows), or null
  const int32_t* seq_off;
};

static constexpr int kAbThreads = 256;   // two warpgroups

// the five 3-D tensor maps [B][L][columns] (box 128 rows x 64 columns, rows >= L out of bounds: zero-filled)
struct AttnBwdMaps {
  CUtensorMap q, k, v, d_o, o;
};

// dS and Pd of the 64 x 64 block held as an accumulator fragment pair (S, dP).  KEYS_ROWS: fragment rows are keys, columns
// queries (phase 1); otherwise rows are queries, columns keys (phase 2).  r0 / c0: first row / column position of the block.
// FULL: every (query, key) pair of the block is visible, so no element is tested.
// Results packed as bf16 A fragments: pk_s = dS, pk_p = Pd (element order of the accumulator).
template <bool KEYS_ROWS, bool FULL>
__device__ __forceinline__ void attn_bwd_block(const float (&sa)[32], const float (&dpa)[32], uint32_t (&pk_s)[16], uint32_t (&pk_p)[16],
                                               const float4* __restrict__ s_stat, const uint8_t* __restrict__ s_keyok,
                                               const uint32_t* __restrict__ s_colkey, int r0, int c0, int L, bool causal,
                                               float sl2, float scale, bool drop, uint32_t thr, float ks_drop) {
  const int t = threadIdx.x & 127;
  const int fr = frag_row(t), fc = frag_col(t);
  const float keep_s = ks_drop * scale;
#pragma unroll
  for (int q = 0; q < 8; ++q)
#pragma unroll
    for (int h = 0; h < 2; ++h) {   // h: fragment row fr (0) or fr + 8 (1)
      float ds2[2], pd2[2];
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int rr = r0 + fr + 8 * h, cc = c0 + 8 * q + fc + e;
        const int i = KEYS_ROWS ? cc : rr, j = KEYS_ROWS ? rr : cc;   // query, key
        const float4 st = s_stat[i];   // m, 1/sum, delta * scale, row key (bits)
        const float pr = ex2f(fmaf(sa[4 * q + 2 * h + e], sl2, -st.x)) * st.y;
        float kp = ks_drop, kps = keep_s;
        if (drop) {
          const bool keep = drop_mix(__float_as_uint(st.w), s_colkey[j]) >= thr;
          kp = keep ? ks_drop : 0.f;
          kps = keep ? keep_s : 0.f;
        }
        const bool vis = FULL || (s_keyok[j] && i < L && (!causal || j <= i));
        ds2[e] = vis ? pr * fmaf(dpa[4 * q + 2 * h + e], kps, -st.z) : 0.f;
        pd2[e] = vis ? pr * kp : 0.f;
      }
      pk_s[2 * q + h] = pack_bf16(ds2[0], ds2[1]);
      pk_p[2 * q + h] = pack_bf16(pd2[0], pd2[1]);
    }
}

template <bool CAUSAL>
__global__ void __launch_bounds__(kAbThreads, 1)
attn_bwd_kernel(const __grid_constant__ AttnBwdMaps tm, const AttnBwdParams p) {
  constexpr int HD = 64;
  constexpr int TILE = 128 * 128;  // bytes of one [128 rows x 64 bf16] swizzled tile; 64-row block b at + b * 8192
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sQ = smem;               // 2 tiles each (rows 0-127, 128-255)
  uint8_t* sdO = sQ + 2 * TILE;
  uint8_t* sK = sdO + 2 * TILE;
  uint8_t* sV = sK + 2 * TILE;
  uint8_t* sO = sV + 2 * TILE;
  uint8_t* sdS = sO;                // causal: dS^T block (kb, qs), kb <= qs, at + ds_blk(kb, qs) * 8192 (O is dead by then)
  __shared__ float4 s_stat[256];    // per query: m, 1/sum, delta * scale, dropout row key
  __shared__ uint8_t s_keyok[256];
  __shared__ uint8_t s_kok32[8];    // all 32 keys [32 g, 32 g + 32) are real
  __shared__ __align__(16) uint32_t s_colkey[256];
  __shared__ uint64_t bar_load;

  const int h = blockIdx.x % p.H, b = blockIdx.x / p.H;
  const int bz = b * p.H + h;
  // packed rows: the window of attn_fwd_kernel (lead rows of the sequence before, then positions first .. p.L - 1); L is
  // its length, local index = position - shift.  Causal only: a query before `lead` sees no key, a key before it is masked.
  const bool packed = p.seq_first != nullptr;
  const int first = packed ? p.seq_first[b] : 0;
  const int lead = first & 63, shift = first - lead;
  const int L = p.L - shift;
  const int row0 = packed ? p.seq_off[b] - lead : b * p.L;
  if (packed && first == p.L) return;
  const int n_t = (L + 127) / 128;  // 128-row tiles
  const int n_blk = (L + 63) / 64;  // 64-row blocks
  const bool drop = p.drop_p > 0.f;

  if (threadIdx.x == 0) {
    mbar_init(&bar_load, 1);
    fence_barrier_init();
    mbar_arrive_expect_tx(&bar_load, 5 * n_t * TILE);
    for (int t = 0; t < n_t; ++t) {
      if (packed) {
        tma_load_2d(sK + t * TILE, &tm.k, &bar_load, p.k_c0 + h * HD, row0 + t * 128);
        tma_load_2d(sQ + t * TILE, &tm.q, &bar_load, p.q_c0 + h * HD, row0 + t * 128);
        tma_load_2d(sV + t * TILE, &tm.v, &bar_load, p.v_c0 + h * HD, row0 + t * 128);
        tma_load_2d(sdO + t * TILE, &tm.d_o, &bar_load, h * HD, row0 + t * 128);
        tma_load_2d(sO + t * TILE, &tm.o, &bar_load, h * HD, row0 + t * 128);
        continue;
      }
      tma_load_3d(sK + t * TILE, &tm.k, &bar_load, p.k_c0 + h * HD, t * 128, b);
      tma_load_3d(sQ + t * TILE, &tm.q, &bar_load, p.q_c0 + h * HD, t * 128, b);
      tma_load_3d(sV + t * TILE, &tm.v, &bar_load, p.v_c0 + h * HD, t * 128, b);
      tma_load_3d(sdO + t * TILE, &tm.d_o, &bar_load, h * HD, t * 128, b);
      tma_load_3d(sO + t * TILE, &tm.o, &bar_load, h * HD, t * 128, b);
    }
  }
  __syncthreads();
  {
    // row statistics of this (sequence, head): m, 1/sum from the forward, delta = sum_c dO[i,c] O[i,c], the dropout keys
    const int i = threadIdx.x, ti = i >> 7, r = i & 127;
    const unsigned long long seed_eff = p.seed + ((drop && p.seed_ptr) ? *p.seed_ptr : 0ull);
    float m = 0.f, inv = 0.f, dl = 0.f;
    if (i >= lead && i < L) {
      m = p.m_save[(size_t)bz * p.Lp + i];
      inv = p.inv_sum[(size_t)bz * p.Lp + i];
    }
    const uint32_t rk = drop_row_key(seed_eff, p.drop_off, (unsigned long long)bz * p.Lp + (unsigned long long)(shift + i));
    const bool key_ok = i >= lead && i < L && (!p.mask_pad_keys || p.pad_mask[(size_t)b * p.L + shift + i] != 0);
    s_keyok[i] = key_ok;
    const bool all_ok = __all_sync(0xffffffffu, key_ok);
    if ((i & 31) == 0) s_kok32[i >> 5] = all_ok;
    s_colkey[i] = drop_col_key((uint32_t)(shift + i));
    mbar_wait(&bar_load, 0);
    if (ti < n_t) {
#pragma unroll
      for (int c = 0; c < HD / 8; ++c) {
        const uint4 ov = *reinterpret_cast<const uint4*>(sO + ti * TILE + sw128_off((uint32_t)r, (uint32_t)c));
        const uint4 dv = *reinterpret_cast<const uint4*>(sdO + ti * TILE + sw128_off((uint32_t)r, (uint32_t)c));
        const __nv_bfloat162* o2 = reinterpret_cast<const __nv_bfloat162*>(&ov);
        const __nv_bfloat162* d2 = reinterpret_cast<const __nv_bfloat162*>(&dv);
#pragma unroll
        for (int t = 0; t < 4; ++t) {
          const float2 a = __bfloat1622float2(o2[t]), g = __bfloat1622float2(d2[t]);
          dl = fmaf(a.x, g.x, fmaf(a.y, g.y, dl));
        }
      }
    }
    s_stat[i] = make_float4(m, inv, dl * p.scale, __uint_as_float(rk));
  }
  if (packed) {
    // rows [L, n_t * 128) of the tiles belong to the next sequence or to no sequence (stale rows past the packed count): every
    // probability that touches them is zero, but 0 * Inf / NaN in the MMAs is not, so the operand rows are cleared
    __syncthreads();   // the statistics above have read sO / sdO
    const int n_pad = n_t * 128 - L;
    for (int i = threadIdx.x; i < 4 * n_pad * 8; i += kAbThreads) {
      const int a = i / (n_pad * 8), r = L + (i / 8) % n_pad;
      uint8_t* base = a == 0 ? sQ : a == 1 ? sK : a == 2 ? sV : sdO;
      *reinterpret_cast<uint4*>(base + r * 128 + (i % 8) * 16) = make_uint4(0u, 0u, 0u, 0u);
    }
    fence_proxy_async();
  }
  __syncthreads();

  const int wg = threadIdx.x >> 7, t = threadIdx.x & 127;
  const int fr = frag_row(t), fc = frag_col(t);
  const float sl2 = p.scale * kLog2eA;
  const uint32_t thr = drop ? (uint32_t)(p.drop_p * 4294967296.0) : 0u;
  const float ks_drop = drop ? 1.f / (1.f - p.drop_p) : 1.f;
  const uint32_t aQ = smem_u32(sQ), adO = smem_u32(sdO), aK = smem_u32(sK), aV = smem_u32(sV);
  // S-type products of two 64-row blocks: X_x . Y_y^T (both K-major over the 64 head dims)
  auto qk = [&](float (&acc)[32], uint32_t x, uint32_t y) {
#pragma unroll
    for (int ks = 0; ks < 4; ++ks) WgmmaSS<64>::template run<0, 0>(acc, desc_k(x + ks * 32), desc_k(y + ks * 32), ks != 0);
  };
  auto store_rows = [&](const float (&acc)[32], __nv_bfloat16* base, int ld, int c0, int r0) {
    const int ra = r0 + fr, rb = ra + 8;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int c = c0 + h * HD + 8 * j + fc;
      if (ra >= lead && ra < L) *reinterpret_cast<uint32_t*>(base + ((size_t)row0 + ra) * ld + c) = pack_bf16(acc[4 * j], acc[4 * j + 1]);
      if (rb >= lead && rb < L) *reinterpret_cast<uint32_t*>(base + ((size_t)row0 + rb) * ld + c) = pack_bf16(acc[4 * j + 2], acc[4 * j + 3]);
    }
  };
  // every (query, key) pair of block (query block qb, key block kb) is visible: all its keys are real, all its queries are
  // rows < L, and under the causal mask it lies below the diagonal
  auto block_full = [&](int qb, int kb) -> bool {
    return s_kok32[2 * kb] && s_kok32[2 * kb + 1] && (qb + 1) * 64 <= L && (!CAUSAL || kb < qb);
  };
  auto ds_blk = [](int kb, int qs) { return (uint32_t)(qs * (qs + 1) / 2 + kb) * 8192u; };
  // blocks of this warpgroup: wg and 3 - wg (balances the causal triangle)
#pragma unroll 1
  for (int u = 0; u < 2; ++u) {
    const int kb = u == 0 ? wg : 3 - wg;
    if (kb >= n_blk) continue;
    // ---- phase 1: rows = keys of block kb
    float dk[32], dv[32];
    acc_zero(dk);
    acc_zero(dv);
#pragma unroll 1
    for (int qs = CAUSAL ? kb : 0; qs < n_blk; ++qs) {
      float sa[32], dpa[32];
      wg_fence();
      qk(sa, aK + kb * 8192, aQ + qs * 8192);
      qk(dpa, aV + kb * 8192, adO + qs * 8192);
      wg_commit();
      wg_wait<0>();
      wg_fence_acc(sa);
      wg_fence_acc(dpa);
      uint32_t pk_s[16], pk_p[16];
      if (block_full(qs, kb))
        attn_bwd_block<true, true>(sa, dpa, pk_s, pk_p, s_stat, s_keyok, s_colkey, kb * 64, qs * 64, L, CAUSAL, sl2, p.scale, drop,
                                   thr, ks_drop);
      else
        attn_bwd_block<true, false>(sa, dpa, pk_s, pk_p, s_stat, s_keyok, s_colkey, kb * 64, qs * 64, L, CAUSAL, sl2, p.scale, drop,
                                    thr, ks_drop);
      if constexpr (CAUSAL) {
        // dS^T as a swizzled [64 keys x 64 queries] tile: row fr (+ 8), 16-byte chunk q, bf16 pair at fc
        uint8_t* blk = sdS + ds_blk(kb, qs);
#pragma unroll
        for (int q = 0; q < 8; ++q)
#pragma unroll
          for (int hr = 0; hr < 2; ++hr)
            *reinterpret_cast<uint32_t*>(blk + sw128_off((uint32_t)(fr + 8 * hr), (uint32_t)q) + fc * 2) = pk_s[2 * q + hr];
      }
      wg_fence();
#pragma unroll
      for (int kk = 0; kk < 4; ++kk) {   // contraction over the 64 queries of the step
        const uint32_t ap[4] = {pk_p[4 * kk], pk_p[4 * kk + 1], pk_p[4 * kk + 2], pk_p[4 * kk + 3]};
        const uint32_t as[4] = {pk_s[4 * kk], pk_s[4 * kk + 1], pk_s[4 * kk + 2], pk_s[4 * kk + 3]};
        WgmmaRS<64>::template run<1>(dv, ap, desc_mn(adO + qs * 8192 + kk * 2048, 8192), 1);
        WgmmaRS<64>::template run<1>(dk, as, desc_mn(aQ + qs * 8192 + kk * 2048, 8192), 1);
      }
      wg_commit();
      wg_wait<0>();
      wg_fence_acc(dk);
      wg_fence_acc(dv);
    }
    store_rows(dk, p.dK, p.ld_dk, p.dk_c0, kb * 64);
    store_rows(dv, p.dV, p.ld_dv, p.dv_c0, kb * 64);
  }
  if constexpr (CAUSAL) {
    // phase 2 reads the dS^T blocks through the async proxy, some of them written by the other warpgroup
    fence_proxy_async();
    __syncthreads();
  }
  const uint32_t adS = smem_u32(sdS);
#pragma unroll 1
  for (int u = 0; u < 2; ++u) {
    const int qb = u == 0 ? wg : 3 - wg;
    if (qb >= n_blk) continue;
    // ---- phase 2: rows = queries of block qb
    float dq[32];
    acc_zero(dq);
    if constexpr (CAUSAL) {
      // one commit group per key block, one wait for all of them (a single group spanning the loop makes ptxas serialise
      // the wgmmas)
#pragma unroll 1
      for (int kb = 0; kb <= qb; ++kb) {
        wg_fence();
#pragma unroll
        for (int kk = 0; kk < 4; ++kk)   // contraction over the 64 keys of the block
          WgmmaSS<64>::template run<1, 1>(dq, desc_mn(adS + ds_blk(kb, qb) + kk * 2048, 8192),
                                          desc_mn(aK + kb * 8192 + kk * 2048, 8192), 1);
        wg_commit();
      }
      wg_wait<0>();
      wg_fence_acc(dq);
    } else {
#pragma unroll 1
      for (int kb = 0; kb < n_blk; ++kb) {
        float sa[32], dpa[32];
        wg_fence();
        qk(sa, aQ + qb * 8192, aK + kb * 8192);
        qk(dpa, adO + qb * 8192, aV + kb * 8192);
        wg_commit();
        wg_wait<0>();
        wg_fence_acc(sa);
        wg_fence_acc(dpa);
        uint32_t pk_s[16], pk_p[16];
        if (block_full(qb, kb))
          attn_bwd_block<false, true>(sa, dpa, pk_s, pk_p, s_stat, s_keyok, s_colkey, qb * 64, kb * 64, L, false, sl2, p.scale, drop,
                                      thr, ks_drop);
        else
          attn_bwd_block<false, false>(sa, dpa, pk_s, pk_p, s_stat, s_keyok, s_colkey, qb * 64, kb * 64, L, false, sl2, p.scale, drop,
                                       thr, ks_drop);
        wg_fence();
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) {   // contraction over the 64 keys of the block
          const uint32_t as[4] = {pk_s[4 * kk], pk_s[4 * kk + 1], pk_s[4 * kk + 2], pk_s[4 * kk + 3]};
          WgmmaRS<64>::template run<1>(dq, as, desc_mn(aK + kb * 8192 + kk * 2048, 8192), 1);
        }
        wg_commit();
        wg_wait<0>();
        wg_fence_acc(dq);
      }
    }
    store_rows(dq, p.dQ, p.ld_dq, p.dq_c0, qb * 64);
  }
}

}  // namespace rp

using namespace rp;

struct rp_attn_bwd_desc {
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
  float scale;
  const int32_t* seq_first; const int32_t* seq_off;
};

RP_API int rp_attn_bwd(const rp_attn_bwd_desc* a, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (!a || !a->q || !a->k || !a->v || !a->d_out || !a->out || !a->pad_mask || !a->m_save || !a->inv_sum || !a->dq || !a->dk ||
      !a->dv)
    return RP_EINVAL;
  if (a->L <= 0 || a->L > 256 || a->B <= 0 || a->H <= 0 || a->head_dim != 64) return RP_ESHAPE;
  if ((a->ld_dq & 7) || (a->ld_dk & 7) || (a->ld_dv & 7) || (a->ldo & 7) || (a->ld_do & 7) || (a->dq_c0 & 7) || (a->dk_c0 & 7) ||
      (a->dv_c0 & 7))
    return RP_EALIGN;
  AttnBwdParams p;
  p.B = a->B; p.H = a->H; p.L = a->L; p.Lp = (a->L + 63) & ~63;
  p.causal = a->causal; p.mask_pad_keys = a->mask_pad_keys;
  p.scale = a->scale > 0.f ? a->scale : 1.f / sqrtf((float)a->head_dim);
  p.pad_mask = a->pad_mask;
  p.m_save = a->m_save; p.inv_sum = a->inv_sum;
  p.dQ = reinterpret_cast<__nv_bfloat16*>(a->dq); p.ld_dq = a->ld_dq; p.dq_c0 = a->dq_c0;
  p.dK = reinterpret_cast<__nv_bfloat16*>(a->dk); p.ld_dk = a->ld_dk; p.dk_c0 = a->dk_c0;
  p.dV = reinterpret_cast<__nv_bfloat16*>(a->dv); p.ld_dv = a->ld_dv; p.dv_c0 = a->dv_c0;
  p.q_c0 = a->q_c0; p.k_c0 = a->k_c0; p.v_c0 = a->v_c0;
  p.drop_p = a->drop_p; p.seed = a->seed; p.drop_off = a->drop_off; p.seed_ptr = a->seed_ptr;
  p.seq_first = a->seq_first; p.seq_off = a->seq_off;
  if ((a->seq_first == nullptr) != (a->seq_off == nullptr)) return RP_EINVAL;
  if (a->seq_first && !a->causal) return RP_EINVAL;
  AttnBwdMaps tm;
  int rc;
  const uint64_t B = (uint64_t)a->B, L = (uint64_t)a->L;
  if ((uint64_t)a->q_rows < B * L || (uint64_t)a->k_rows < B * L || (uint64_t)a->v_rows < B * L || (uint64_t)a->do_rows < B * L)
    return RP_ESHAPE;
  if (a->seq_first) {
    // packed rows: 2-D maps over the row arrays (a window starts inside the sequence before - at a negative row for the first
    // sequence: zero-filled - and may run into the next sequence's rows, which the kernel clears)
    if ((rc = make_tmap_bf16(&tm.q, a->q, a->q_rows, a->q_cols, a->ldq, 128)) != RP_OK) return rc;
    if ((rc = make_tmap_bf16(&tm.k, a->k, a->k_rows, a->k_cols, a->ldk, 128)) != RP_OK) return rc;
    if ((rc = make_tmap_bf16(&tm.v, a->v, a->v_rows, a->v_cols, a->ldv, 128)) != RP_OK) return rc;
    if ((rc = make_tmap_bf16(&tm.d_o, a->d_out, a->do_rows, a->do_cols, a->ld_do, 128)) != RP_OK) return rc;
    if ((rc = make_tmap_bf16(&tm.o, a->out, a->do_rows, (uint64_t)a->H * 64, a->ldo, 128)) != RP_OK) return rc;
  } else {
    if ((rc = make_tmap_bf16_seq(&tm.q, a->q, B, L, a->q_cols, a->ldq, 128)) != RP_OK) return rc;
    if ((rc = make_tmap_bf16_seq(&tm.k, a->k, B, L, a->k_cols, a->ldk, 128)) != RP_OK) return rc;
    if ((rc = make_tmap_bf16_seq(&tm.v, a->v, B, L, a->v_cols, a->ldv, 128)) != RP_OK) return rc;
    if ((rc = make_tmap_bf16_seq(&tm.d_o, a->d_out, B, L, a->do_cols, a->ld_do, 128)) != RP_OK) return rc;
    if ((rc = make_tmap_bf16_seq(&tm.o, a->out, B, L, (uint64_t)a->H * 64, a->ldo, 128)) != RP_OK) return rc;
  }
  // Q, dO, K, V (2 tiles each), then O (2 tiles) or, causal, the dS^T triangle of up to 10 64 x 64 blocks in its place
  const int smem = 8 * 128 * 128 + (a->causal ? 10 * 8192 : 2 * 128 * 128) + 1024;
  if (a->causal) {
    RP_CUDA_CHECK(cudaFuncSetAttribute(attn_bwd_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    attn_bwd_kernel<true><<<a->B * a->H, kAbThreads, smem, stream>>>(tm, p);
  } else {
    RP_CUDA_CHECK(cudaFuncSetAttribute(attn_bwd_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    attn_bwd_kernel<false><<<a->B * a->H, kAbThreads, smem, stream>>>(tm, p);
  }
  RP_LAUNCH_CHECK();
  return RP_OK;
}
