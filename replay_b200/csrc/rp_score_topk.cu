// rp_score_topk.cu - fused predict head:  scores = Hq[B,d] . E[I,d]^T  ->  seen-item mask  ->  per-row top-K.
//
// Replaces, for one batch of users, the reference chain
//   EmbeddingTyingHead.forward            replay/nn/head.py:29-34   (legacy: models/nn/sequential/sasrec/model.py:286-307)
//   SeenItemsFilter._compute_scores       replay/nn/lightning/postprocessor/seen_items.py:56-83
//   torch.topk(logits, k, dim=1)          replay/nn/lightning/callback/predictions_callback.py:90
// without ever materialising the [B, |I|] logits.
//
// Kernel 1 (score_topk_kernel): one CTA = 128 users x a contiguous range of 128-item tiles.
//   thread 0    TMA: user tile A (resident in smem) + ring of item-table K-chunks [128 items x 64]
//   warpgroups  wgmma: S[128x128] fp32 in registers (warpgroup g: users [64 g, 64 g + 64)); each 64-column half of the
//   0 and 1     tile goes through a shared-memory stage, then thread = (user row, 32-column part): seen-mask via a cursor
//               into the user's sorted seen list, running top-K (sorted, registers), partial top-K per (user, split, part)
// Kernel 2 (topk_merge_kernel): one warp per user merges the per-split partial lists (score desc, column asc).
// This register path serves K <= 32; 32 < K <= 1024 runs score_topk_wide_kernel + topk_wide_merge_kernel (see "wide K").
#include <cfloat>

#include "rp_host.h"
#include "rp_sm90.cuh"

namespace rp {

static constexpr int kTileM = 128;   // users per CTA
static constexpr int kTileN = 128;   // items per MMA tile
static constexpr int kChunkBytes = 128 * 128;  // [128 rows x 64 bf16]
static constexpr int kNoId = 0x7fffffff;

// Per-thread running top-K kept in registers.  The K live entries occupy slots [KMAX-K, KMAX) in descending order so
// that the admission threshold is always the statically indexed last slot; slots below hold +inf sentinels that never
// move.  (A runtime-indexed v[K-1] would push the whole structure into local memory.)
template <int KMAX>
struct TopK {
  float v[KMAX];
  int id[KMAX];
  __device__ __forceinline__ void init(int K) {
#pragma unroll
    for (int i = 0; i < KMAX; ++i) {
      v[i] = (i < KMAX - K) ? INFINITY : -INFINITY;
      id[i] = kNoId;
    }
  }
  __device__ __forceinline__ float thr() const { return v[KMAX - 1]; }
  // sorted insert (descending, earlier insert wins ties because columns arrive in ascending order)
  __device__ __forceinline__ void insert(float x, int xi) {
#pragma unroll
    for (int i = 0; i < KMAX; ++i) {
      const bool gt = x > v[i];
      const float tv = gt ? v[i] : x;
      const int ti = gt ? id[i] : xi;
      v[i] = gt ? x : v[i];
      id[i] = gt ? xi : id[i];
      x = tv;
      xi = ti;
    }
  }
};

// order-preserving float <-> unsigned key (0 is below every float, so a zero-filled array means "no threshold yet")
__device__ __forceinline__ uint32_t f2key(float f) {
  const uint32_t b = __float_as_uint(f);
  return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}
__device__ __forceinline__ float key2f(uint32_t k) {
  return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k);
}

static constexpr int kEpiThreads = 256;   // the two warpgroups
static constexpr int kColParts = 2;       // 32-column parts of each 64-column half: one running top-K per (row, part)
static constexpr int kThreads = kEpiThreads;
static constexpr int kStagePitch = 64 + 4;

// One 32-column chunk of one row (thread).  FAST PATH: the maxima of the four 8-column groups against the admission threshold -
// the values are never modified or copied.  Seen / out-of-catalog columns are
// NOT masked here: a masked column only matters if it would be admitted, and then the slow path drops it from the hit mask (a
// spurious slow-path entry costs about what masking every chunk that holds a seen item would).  SLOW PATH (a group maximum
// beats the threshold): stage that group's 8 values in shared memory so that ONE insert site serves a runtime column index,
// build the hit mask, drop masked columns, insert.
template <int KMAX>
__device__ __forceinline__ void score_chunk(const uint32_t (&raw)[32], uint32_t kill, float thr, float gthr, int col0,
                                            TopK<KMAX>& top, float* sc, bool live, uint32_t* row_thr_u) {
  // maxima of the four 8-column groups: the slow path then stages and scans only the group(s) that hold a candidate
  float g[4];
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const float a = fmaxf(__uint_as_float(raw[8 * k]), __uint_as_float(raw[8 * k + 1]));
    const float b = fmaxf(__uint_as_float(raw[8 * k + 2]), __uint_as_float(raw[8 * k + 3]));
    const float c = fmaxf(__uint_as_float(raw[8 * k + 4]), __uint_as_float(raw[8 * k + 5]));
    const float d = fmaxf(__uint_as_float(raw[8 * k + 6]), __uint_as_float(raw[8 * k + 7]));
    g[k] = fmaxf(fmaxf(a, b), fmaxf(c, d));
  }
  const float m = fmaxf(fmaxf(g[0], g[1]), fmaxf(g[2], g[3]));
  if (m > thr) {
    const float before = top.thr();
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      if (g[k] > thr) {  // stage this group's 8 values so that ONE insert site serves a runtime column index
        uint32_t hit = 0;
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          sc[i * kEpiThreads] = __uint_as_float(raw[8 * k + i]);
          hit |= (__uint_as_float(raw[8 * k + i]) > thr) ? (1u << i) : 0u;
        }
        hit &= ~(kill >> (8 * k));
        while (hit) {
          const int i = __ffs(hit) - 1;
          hit &= hit - 1;
          const float val = sc[i * kEpiThreads];
          if (val > fmaxf(top.thr(), gthr)) top.insert(val, col0 + 8 * k + i);
        }
      }
    }
    // publish an improved K-th best (only once the list holds K real entries, i.e. its last slot is finite)
    if (live && top.thr() > before && top.thr() > -INFINITY) atomicMax(row_thr_u, f2key(top.thr()));
  }
}


template <int KCH /* d / 64 */, int NSTAGE, int KMAX>
__global__ void __launch_bounds__(kThreads, 1)
score_topk_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                  const int32_t* __restrict__ seen_sorted, int S, int n_users, int n_items, int K, int n_splits,
                  const float* __restrict__ bias, float* __restrict__ part_vals, int32_t* __restrict__ part_ids,
                  uint32_t* __restrict__ row_thr /* [n_users] shared K-th-best keys, zero-filled */) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sA = smem;                          // KCH chunks of 16 KB
  uint8_t* sB = smem + KCH * kChunkBytes;      // NSTAGE chunks of 16 KB
  float* stage = reinterpret_cast<float*>(sB + NSTAGE * kChunkBytes);   // [128 x kStagePitch] fp32: one 64-column half
  __shared__ uint64_t bar_a, bar_full[NSTAGE], bar_empty[NSTAGE];
  __shared__ float s_scratch[8 * kEpiThreads];  // [i][thread]: one 8-column group staged for the insert path

  const int lane = threadIdx.x & 31;
  const int user_tile = blockIdx.x / n_splits, split = blockIdx.x % n_splits;
  const int u0 = user_tile * kTileM;
  const int n_tiles_total = (n_items + kTileN - 1) / kTileN;
  const int t_begin = (int)(((long long)n_tiles_total * split) / n_splits);
  const int t_end = (int)(((long long)n_tiles_total * (split + 1)) / n_splits);

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
  // the ring of item-table chunks is fed by thread 0: chunk i -> stage i % NSTAGE once the 8 warps released its previous use
  const int n_chunks = (t_end - t_begin) * KCH;
  auto issue = [&](int i) {
    const uint32_t s = i % NSTAGE;
    mbar_wait(&bar_empty[s], ((i / NSTAGE) & 1) ^ 1);
    mbar_arrive_expect_tx(&bar_full[s], kChunkBytes);
    tma_load_2d(sB + s * kChunkBytes, &tmB, &bar_full[s], (i % KCH) * 64, (t_begin + i / KCH) * kTileN);
  };
  if (threadIdx.x == 0) {
    mbar_arrive_expect_tx(&bar_a, KCH * kChunkBytes);
    for (int kc = 0; kc < KCH; ++kc) tma_load_2d(sA + kc * kChunkBytes, &tmA, &bar_a, kc * 64, u0);
    for (int i = 0; i < NSTAGE && i < n_chunks; ++i) issue(i);
  }
  const int wg = threadIdx.x >> 7, ft = threadIdx.x & 127;
  const int fr = frag_row(ft), fc = frag_col(ft);
  // row-wise part: thread = (user row, 32-column part of the staged half)
  const int row = ft, part = wg;
  const int u = u0 + row;
  const bool live = u < n_users;
  float* sc = s_scratch + threadIdx.x;  // element q of this thread at sc[q * kEpiThreads]
  TopK<KMAX> top;
  top.init(K);
  // cursor into this user's sorted seen list (ascending, kNoId = padding).  The next entry is prefetched one step ahead
  // so that the (rare, per thread) advance never waits on a dependent global load inside the tile loop.
  const int32_t* sp = seen_sorted ? seen_sorted + (size_t)(live ? u : 0) * S : nullptr;
  int ci = 0;
  int next_seen = kNoId, pre_seen = kNoId;
  if (sp && live) {
    const int first_col = t_begin * kTileN;
    int lo = 0, hi = S;  // lower_bound(first_col), once per CTA
    while (lo < hi) {
      const int mid = (lo + hi) >> 1;
      if (sp[mid] < first_col) lo = mid + 1; else hi = mid;
    }
    ci = lo;
    next_seen = ci < S ? sp[ci] : kNoId;
    pre_seen = ci + 1 < S ? sp[ci + 1] : kNoId;
  }
  // K-th best already secured for this row by ANY thread / CTA working on it (other column parts and item splits):
  // anything strictly below it cannot reach the final top-K, so it never enters the insert path.  The shared value is
  // read one tile AHEAD (a stale threshold is only weaker, never wrong), so its L2 round trip is off the per-tile path.
  uint32_t gk = live ? *reinterpret_cast<volatile uint32_t*>(row_thr + u) : 0u;
  float gthr = -INFINITY;
  mbar_wait(&bar_a, 0);
  uint32_t it = 0;
  for (int t = t_begin, j = 0; t < t_end; ++t, ++j) {
    if ((j & 3) == 0) {  // refresh every 4th tile: the shared threshold moves slowly once the lists are full
      gthr = gk != 0u ? key2f(gk - 1u) : -INFINITY;  // largest value strictly below the shared K-th best
      // ... except around zero: below a published +0 lies -0, and below -0 or a denormal lies a denormal, which
      // --use_fast_math compares as 0, so "0 > gthr" would reject the zeros that win an exact-zero tie at the K-th place on
      // their smaller column.  -FLT_MIN (normal, never flushed) admits them; a lower threshold only admits more, never wrong.
      if (fabsf(gthr) < FLT_MIN) gthr = -FLT_MIN;
      if (live) gk = *reinterpret_cast<volatile uint32_t*>(row_thr + u);  // lands long before its use 4 tiles later
    }
    float acc[kTileN / 2];
    for (int kc = 0; kc < KCH; ++kc, ++it) {
      const uint32_t s = it % NSTAGE, ph = (it / NSTAGE) & 1;
      mbar_wait(&bar_full[s], ph);
      const uint32_t a0 = smem_u32(sA + kc * kChunkBytes) + wg * 8192, b0 = smem_u32(sB + s * kChunkBytes);
      wg_fence();
#pragma unroll
      for (int ks = 0; ks < 4; ++ks)
        WgmmaSS<kTileN>::template run<0, 0>(acc, desc_k(a0 + ks * 32), desc_k(b0 + ks * 32), (kc | ks) != 0);
      wg_commit();
      wg_wait<0>();
      wg_fence_acc(acc);
      __syncwarp();
      if (lane == 0) mbar_arrive(&bar_empty[s]);
      if (threadIdx.x == 0 && (int)it + NSTAGE < n_chunks) issue((int)it + NSTAGE);
    }
#pragma unroll
    for (int half = 0; half < 2; ++half) {
      named_bar_sync(1, kEpiThreads);   // the stage's previous readers are done
      {
        const int r = 64 * wg + fr;
#pragma unroll
        for (int q = 0; q < 8; ++q) {
          const int jj = 8 * half + q;
          *reinterpret_cast<float2*>(stage + r * kStagePitch + 8 * q + fc) = make_float2(acc[4 * jj], acc[4 * jj + 1]);
          *reinterpret_cast<float2*>(stage + (r + 8) * kStagePitch + 8 * q + fc) = make_float2(acc[4 * jj + 2], acc[4 * jj + 3]);
        }
      }
      named_bar_sync(1, kEpiThreads);
      uint32_t raw[32];
      stage_ld32(stage + row * kStagePitch + part * 32, raw);
      const int col0 = t * kTileN + half * 64 + part * 32;
      // seen items of this 32-column chunk as a bit mask (also skips entries that belong to the other column part);
      // columns beyond the catalog (ragged last tile) are "seen" too
      uint32_t kill = 0;
      while (next_seen < col0 + 32) {
        if (next_seen >= col0) kill |= 1u << (next_seen - col0);
        next_seen = pre_seen;
        ++ci;
        pre_seen = ci + 1 < S ? sp[ci + 1] : kNoId;
      }
      if (col0 + 32 > n_items) kill |= (col0 >= n_items) ? 0xffffffffu : (0xffffffffu << (n_items - col0));
      const float thr = live ? fmaxf(top.thr(), gthr) : INFINITY;  // rows beyond the batch never enter the insert path
      if (bias == nullptr) {
        score_chunk(raw, kill, thr, gthr, col0, top, sc, live, row_thr + u);
      } else {  // biased head (BERT4Rec): warp-uniform 16-byte loads, bias padded to a multiple of 128 entries
#pragma unroll
        for (int q = 0; q < 32; q += 4) {
          const float4 b4 = __ldg(reinterpret_cast<const float4*>(bias + col0 + q));
          raw[q] = __float_as_uint(__uint_as_float(raw[q]) + b4.x);
          raw[q + 1] = __float_as_uint(__uint_as_float(raw[q + 1]) + b4.y);
          raw[q + 2] = __float_as_uint(__uint_as_float(raw[q + 2]) + b4.z);
          raw[q + 3] = __float_as_uint(__uint_as_float(raw[q + 3]) + b4.w);
        }
        score_chunk(raw, kill, thr, gthr, col0, top, sc, live, row_thr + u);
      }
    }
  }
  if (live) {
    float* pv = part_vals + (((size_t)u * n_splits + split) * kColParts + part) * K;
    int32_t* pi = part_ids + (((size_t)u * n_splits + split) * kColParts + part) * K;
#pragma unroll
    for (int i = 0; i < KMAX; ++i)
      if (i >= KMAX - K) {
        pv[i - (KMAX - K)] = top.v[i];
        pi[i - (KMAX - K)] = top.id[i];
      }
  }
}

// one warp per user: merge n_splits sorted partial lists -> final top-K; ties: smaller column first.
// Slots that no finite candidate fills (fewer than K unmasked items) are filled with the user's masked columns in
// ascending order, score -inf (torch.topk would return arbitrary -inf entries there).
__global__ void topk_merge_kernel(const float* __restrict__ part_vals, const int32_t* __restrict__ part_ids,
                                  const int32_t* __restrict__ seen_sorted, int S, int n_users, int n_items, int K,
                                  int n_splits, const int64_t* __restrict__ candidates, int64_t* __restrict__ out_ids,
                                  float* __restrict__ out_scores) {
  const int u = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (u >= n_users) return;
  const int n = n_splits * K;
  const float* pv = part_vals + (size_t)u * n;
  const int32_t* pi = part_ids + (size_t)u * n;
  // each lane owns candidates lane, lane+32, ...  ; consumed ones are flagged by setting id to kNoId+(-inf)
  float last_v = INFINITY;
  int last_id = -1;
  int n_out = 0;
  for (int k = 0; k < K; ++k) {
    // best candidate strictly after (last_v, last_id) in (score desc, id asc) order
    float bv = -INFINITY;
    int bi = kNoId;
    for (int i = lane; i < n; i += 32) {
      const float v = pv[i];
      const int id = pi[i];
      if (id == kNoId) continue;
      const bool after = (v < last_v) || (v == last_v && id > last_id);
      if (!after) continue;
      if (v > bv || (v == bv && id < bi)) {
        bv = v;
        bi = id;
      }
    }
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) {
      const float ov = __shfl_xor_sync(0xffffffffu, bv, off);
      const int oi = __shfl_xor_sync(0xffffffffu, bi, off);
      if (ov > bv || (ov == bv && oi < bi)) {
        bv = ov;
        bi = oi;
      }
    }
    if (bi == kNoId) break;
    if (lane == 0) {
      out_ids[(size_t)u * K + k] = candidates ? candidates[bi] : (int64_t)bi;
      out_scores[(size_t)u * K + k] = bv;
    }
    last_v = bv;
    last_id = bi;
    ++n_out;
  }
  if (n_out < K && lane == 0) {
    int ci = 0;
    int prev = -1;
    for (int k = n_out; k < K; ++k) {
      int col = kNoId;
      while (seen_sorted && ci < S) {
        const int c = seen_sorted[(size_t)u * S + ci++];
        if (c != prev && c < n_items) {
          col = c;
          prev = c;
          break;
        }
      }
      out_ids[(size_t)u * K + k] = (col == kNoId) ? -1 : (candidates ? candidates[col] : (int64_t)col);
      out_scores[(size_t)u * K + k] = -INFINITY;
    }
  }
}

// Prepare the seen lists for score_topk: int64 ids [B,S] -> int32 columns sorted ascending, padding = kNoId.
// Ids outside [0, item_count) are padding (seen_items.py:62).  With inv_map (candidates_to_score) an id becomes its
// position in the candidate list (or padding when it is not a candidate).  One block per user, bitonic sort in smem.
template <int SPAD>
__global__ void seen_prepare_kernel(const int64_t* __restrict__ seen, int S, int item_count,
                                    const int32_t* __restrict__ inv_map, int32_t* __restrict__ out) {
  __shared__ int32_t buf[SPAD];
  const int u = blockIdx.x;
  for (int i = threadIdx.x; i < SPAD; i += blockDim.x) {
    int32_t v = kNoId;
    if (i < S) {
      const int64_t id = seen[(size_t)u * S + i];
      if (id >= 0 && id < item_count) {
        v = (int32_t)id;
        if (inv_map) {
          v = inv_map[v];
          if (v < 0) v = kNoId;
        }
      }
    }
    buf[i] = v;
  }
  __syncthreads();
  for (int k = 2; k <= SPAD; k <<= 1) {
    for (int jj = k >> 1; jj > 0; jj >>= 1) {
      for (int i = threadIdx.x; i < SPAD; i += blockDim.x) {
        const int ixj = i ^ jj;
        if (ixj > i) {
          const bool up = (i & k) == 0;
          const int32_t a = buf[i], b = buf[ixj];
          if ((a > b) == up) {
            buf[i] = b;
            buf[ixj] = a;
          }
        }
      }
      __syncthreads();
    }
  }
  for (int i = threadIdx.x; i < S; i += blockDim.x) out[(size_t)u * S + i] = buf[i];
}

static int choose_splits(int n_user_tiles, int n_item_tiles) {
  const int sms = sm_count();
  int p = sms / n_user_tiles;
  if (p < 1) p = 1;
  if (p > n_item_tiles) p = n_item_tiles;
  if (p > 64) p = 64;
  return p;
}

template <int KCH, int NSTAGE>
static int launch_score_topk(const CUtensorMap& tmA, const CUtensorMap& tmB, const int32_t* seen_sorted, int S, int B,
                             int I, int K, int n_splits, const float* bias, float* pv, int32_t* pi, uint32_t* row_thr,
                             cudaStream_t stream) {
  const int smem = (KCH + NSTAGE) * kChunkBytes + 128 * kStagePitch * 4 + 1024;
  const int grid = ((B + kTileM - 1) / kTileM) * n_splits;
  if (K <= 10) {
    auto kern = score_topk_kernel<KCH, NSTAGE, 10>;
    RP_CUDA_CHECK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    kern<<<grid, kThreads, smem, stream>>>(tmA, tmB, seen_sorted, S, B, I, K, n_splits, bias, pv, pi, row_thr);
  } else if (K <= 16) {
    auto kern = score_topk_kernel<KCH, NSTAGE, 16>;
    RP_CUDA_CHECK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    kern<<<grid, kThreads, smem, stream>>>(tmA, tmB, seen_sorted, S, B, I, K, n_splits, bias, pv, pi, row_thr);
  } else {
    auto kern = score_topk_kernel<KCH, NSTAGE, 32>;
    RP_CUDA_CHECK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    kern<<<grid, kThreads, smem, stream>>>(tmA, tmB, seen_sorted, S, B, I, K, n_splits, bias, pv, pi, row_thr);
  }
  RP_LAUNCH_CHECK();
  return RP_OK;
}

// ---------------------------------------------------------------------------------------------------------- wide K
// 32 < K <= 1024: a K-entry sorted list no longer fits in registers.  Each (user, item split) instead owns a candidate
// buffer of C >= K + 64 entries in the workspace.  An entry is one 64-bit key: f2key(score) in the high word, ~column in the
// low word, so descending key order is exactly (score desc, column asc) and no two keys are equal - the result is exact
// and deterministic although entries arrive in buffer slots through shared-memory atomics.
//   score_topk_wide_kernel  same CTA, tile loop and admission threshold as score_topk_kernel; an admitted value takes a slot
//                           of its row's buffer.  When a half-tile leaves some row with more than C - 64 entries (one half-tile
//                           adds at most 64 per row) the CTA compacts those rows, one warp per row: a radix select keeps
//                           exactly the K largest keys, and the K-th becomes the row's threshold and is published to row_thr.
//   topk_wide_merge_kernel  one CTA per user: radix select of the top K keys over the n_splits buffers, bitonic sort.
static constexpr int kWideMaxK = 1024;
static constexpr long long kWideMaxEntries = 65536;   // per user over all splits: bounds the workspace and the merge's reads

// C: at least 2K (a compaction every ~K admissions) and K + 64 (room for one more half-tile after a compaction), rounded up
// to a power of two so that a capped split count fills exactly kWideMaxEntries - the workspace then grows with K.
static int wide_capacity(int K) {
  int c = 128;
  while (c < 2 * K || c < K + 64) c <<= 1;
  return c;
}
static int wide_splits(int n_user_tiles, int n_item_tiles, int C) {
  const int p = choose_splits(n_user_tiles, n_item_tiles);
  const int cap = (int)(kWideMaxEntries / C);
  return p > cap ? cap : p;
}
// workspace layout: candidate keys [n_users * p][C], counts [n_users][64], shared thresholds [n_users]
static size_t wide_layout_bytes(int n_users, int n_item_tiles, int C) {
  const int p = wide_splits((n_users + kTileM - 1) / kTileM, n_item_tiles, C);
  return (size_t)n_users * p * C * 8 + (size_t)n_users * 64 * 4 + (size_t)n_users * 4;
}

__device__ __forceinline__ uint64_t wide_key(uint32_t score_bits, int col) {
  if (score_bits == 0x80000000u) score_bits = 0u;  // -0 == +0: one key, so equal scores tie-break on the column alone
  return ((uint64_t)f2key(__uint_as_float(score_bits)) << 32) | (uint32_t)~col;
}

// One warp, a 256-bin histogram of the keys that match the current prefix: the bin b that holds the need-th largest key.
// Lane l owns bins [8 l, 8 l + 8).  Returns b, the number of keys in higher bins (above) and the count of bin b (in_b).
__device__ __forceinline__ void radix_find_bin(const uint32_t* hist, int need, int lane, int& b, int& above, int& in_b) {
  uint32_t h[8];
  uint32_t s = 0;
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    h[j] = hist[8 * lane + j];
    s += h[j];
  }
  uint32_t suf = s;  // inclusive suffix sum over lanes >= lane
#pragma unroll
  for (int off = 1; off < 32; off <<= 1) {
    const uint32_t v = __shfl_down_sync(0xffffffffu, suf, off);
    if (lane + off < 32) suf += v;
  }
  const uint32_t excl = suf - s;
  int my_b = 0, my_above = 0, my_in = 0;
  const bool mine = excl < (uint32_t)need && (uint32_t)need <= suf;
  if (mine) {
    uint32_t acc = excl;
#pragma unroll
    for (int j = 7; j >= 0; --j) {
      if (acc + h[j] >= (uint32_t)need) {
        my_b = 8 * lane + j;
        my_above = (int)acc;
        my_in = (int)h[j];
        break;
      }
      acc += h[j];
    }
  }
  const int src = __ffs(__ballot_sync(0xffffffffu, mine)) - 1;
  b = __shfl_sync(0xffffffffu, my_b, src);
  above = __shfl_sync(0xffffffffu, my_above, src);
  in_b = __shfl_sync(0xffffffffu, my_in, src);
}

// One warp: keep exactly the K largest of the n > K distinct keys rb[0, n), moved to rb[0, K) (in no particular order).
// Returns the smallest kept key.  hist: 256 words of shared memory owned by this warp.
__device__ __noinline__ uint64_t wide_compact_row(uint64_t* rb, int n, int K, uint32_t* hist, int lane) {
  uint64_t prefix = 0, mask = 0;
  int need = K;
  for (int shift = 56; shift >= 0; shift -= 8) {
#pragma unroll
    for (int j = 0; j < 8; ++j) hist[32 * j + lane] = 0u;
    __syncwarp();
    for (int i0 = lane; i0 < n; i0 += 32 * 8) {  // 8 independent loads in flight before their atomics
      uint64_t k8[8];
#pragma unroll
      for (int q = 0; q < 8; ++q) k8[q] = i0 + 32 * q < n ? rb[i0 + 32 * q] : 0ull;
#pragma unroll
      for (int q = 0; q < 8; ++q)
        if (i0 + 32 * q < n && (k8[q] & mask) == prefix) atomicAdd(hist + ((k8[q] >> shift) & 255u), 1u);
    }
    __syncwarp();
    int b, above, in_b;
    radix_find_bin(hist, need, lane, b, above, in_b);
    __syncwarp();
    need -= above;
    prefix |= (uint64_t)b << shift;
    mask |= (uint64_t)0xff << shift;
    if (in_b == need) break;  // every key of this bin is kept: the kept set is {key : key & mask >= prefix}
  }
  // stable in-place compaction: a lane's write index never exceeds the index any lane reads in this or a later step
  int pos = 0;
  uint64_t mn = ~0ull;
  for (int base = 0; base < n; base += 32) {
    const int i = base + lane;
    const uint64_t key = i < n ? rb[i] : 0ull;
    const bool keep = i < n && (key & mask) >= prefix;
    const uint32_t bal = __ballot_sync(0xffffffffu, keep);
    if (keep) {
      rb[pos + __popc(bal & ((1u << lane) - 1u))] = key;
      mn = key < mn ? key : mn;
    }
    pos += __popc(bal);
  }
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) {
    const uint64_t o = __shfl_xor_sync(0xffffffffu, mn, off);
    mn = o < mn ? o : mn;
  }
  return mn;
}

template <int KCH /* d / 64 */, int NSTAGE>
__global__ void __launch_bounds__(kThreads, 1)
score_topk_wide_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                       const int32_t* __restrict__ seen_sorted, int S, int n_users, int n_items, int K, int C, int n_splits,
                       const float* __restrict__ bias, uint64_t* __restrict__ cand /* [n_users * n_splits][C] */,
                       int32_t* __restrict__ cand_n /* [n_users * n_splits] */,
                       uint32_t* __restrict__ row_thr /* [n_users] shared K-th-best keys, zero-filled */) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sA = smem;                          // KCH chunks of 16 KB
  uint8_t* sB = smem + KCH * kChunkBytes;      // NSTAGE chunks of 16 KB
  float* stage = reinterpret_cast<float*>(sB + NSTAGE * kChunkBytes);   // [128 x kStagePitch] fp32: one 64-column half
  __shared__ uint64_t bar_a, bar_full[NSTAGE], bar_empty[NSTAGE];
  __shared__ int s_cnt[kTileM];                // entries in each row's buffer
  __shared__ float s_thr[kTileM];              // each row's own K-th best (of this split) after its last compaction
  __shared__ uint32_t s_hist[kThreads / 32][256];  // one radix histogram per warp

  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int user_tile = blockIdx.x / n_splits, split = blockIdx.x % n_splits;
  const int u0 = user_tile * kTileM;
  const int n_tiles_total = (n_items + kTileN - 1) / kTileN;
  const int t_begin = (int)(((long long)n_tiles_total * split) / n_splits);
  const int t_end = (int)(((long long)n_tiles_total * (split + 1)) / n_splits);

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
  if (threadIdx.x < kTileM) {
    s_cnt[threadIdx.x] = 0;
    s_thr[threadIdx.x] = -INFINITY;
  }
  __syncthreads();
  const int n_chunks = (t_end - t_begin) * KCH;
  auto issue = [&](int i) {
    const uint32_t s = i % NSTAGE;
    mbar_wait(&bar_empty[s], ((i / NSTAGE) & 1) ^ 1);
    mbar_arrive_expect_tx(&bar_full[s], kChunkBytes);
    tma_load_2d(sB + s * kChunkBytes, &tmB, &bar_full[s], (i % KCH) * 64, (t_begin + i / KCH) * kTileN);
  };
  if (threadIdx.x == 0) {
    mbar_arrive_expect_tx(&bar_a, KCH * kChunkBytes);
    for (int kc = 0; kc < KCH; ++kc) tma_load_2d(sA + kc * kChunkBytes, &tmA, &bar_a, kc * 64, u0);
    for (int i = 0; i < NSTAGE && i < n_chunks; ++i) issue(i);
  }
  const int wg = threadIdx.x >> 7, ft = threadIdx.x & 127;
  const int fr = frag_row(ft), fc = frag_col(ft);
  const int row = ft, part = wg;
  const int u = u0 + row;
  const bool live = u < n_users;
  const size_t list0 = (size_t)u0 * n_splits + split;  // list of row r: list0 + r * n_splits
  uint64_t* rb = cand + (list0 + (size_t)row * n_splits) * C;
  // rows compacted by warp w: w, w + 8, ...  (only rows of users that exist ever hold entries)
  auto compact = [&](int min_count) {
    for (int r = warp; r < kTileM && u0 + r < n_users; r += kThreads / 32) {
      const int n = s_cnt[r];
      if (n > min_count && n > K) {
        const uint64_t kth = wide_compact_row(cand + (list0 + (size_t)r * n_splits) * C, n, K, s_hist[warp], lane);
        if (lane == 0) {
          s_cnt[r] = K;
          s_thr[r] = key2f((uint32_t)(kth >> 32));
          // K entries of this split now lie at or above this score: nothing below it can reach the final top K
          atomicMax(row_thr + u0 + r, (uint32_t)(kth >> 32));
        }
      }
    }
  };
  const int32_t* sp = seen_sorted ? seen_sorted + (size_t)(live ? u : 0) * S : nullptr;
  int ci = 0;
  int next_seen = kNoId, pre_seen = kNoId;
  if (sp && live) {
    const int first_col = t_begin * kTileN;
    int lo = 0, hi = S;
    while (lo < hi) {
      const int mid = (lo + hi) >> 1;
      if (sp[mid] < first_col) lo = mid + 1; else hi = mid;
    }
    ci = lo;
    next_seen = ci < S ? sp[ci] : kNoId;
    pre_seen = ci + 1 < S ? sp[ci + 1] : kNoId;
  }
  uint32_t gk = live ? *reinterpret_cast<volatile uint32_t*>(row_thr + u) : 0u;
  // the shared K-th best itself, compared with >=: "strictly above key2f(gk - 1)" would turn a published +0 into -0 and
  // reject the +0 scores that win an exact-zero tie at the K-th place on their smaller column
  float gmin = -INFINITY;
  mbar_wait(&bar_a, 0);
  uint32_t it = 0;
  for (int t = t_begin, j = 0; t < t_end; ++t, ++j) {
    if ((j & 3) == 0) {
      gmin = gk != 0u ? key2f(gk) : -INFINITY;
      if (live) gk = *reinterpret_cast<volatile uint32_t*>(row_thr + u);
    }
    float acc[kTileN / 2];
    for (int kc = 0; kc < KCH; ++kc, ++it) {
      const uint32_t s = it % NSTAGE, ph = (it / NSTAGE) & 1;
      mbar_wait(&bar_full[s], ph);
      const uint32_t a0 = smem_u32(sA + kc * kChunkBytes) + wg * 8192, b0 = smem_u32(sB + s * kChunkBytes);
      wg_fence();
#pragma unroll
      for (int ks = 0; ks < 4; ++ks)
        WgmmaSS<kTileN>::template run<0, 0>(acc, desc_k(a0 + ks * 32), desc_k(b0 + ks * 32), (kc | ks) != 0);
      wg_commit();
      wg_wait<0>();
      wg_fence_acc(acc);
      __syncwarp();
      if (lane == 0) mbar_arrive(&bar_empty[s]);
      if (threadIdx.x == 0 && (int)it + NSTAGE < n_chunks) issue((int)it + NSTAGE);
    }
#pragma unroll
    for (int half = 0; half < 2; ++half) {
      // the stage's previous readers are done: every thread passed the __syncthreads_or of the previous half
      {
        const int r = 64 * wg + fr;
#pragma unroll
        for (int q = 0; q < 8; ++q) {
          const int jj = 8 * half + q;
          *reinterpret_cast<float2*>(stage + r * kStagePitch + 8 * q + fc) = make_float2(acc[4 * jj], acc[4 * jj + 1]);
          *reinterpret_cast<float2*>(stage + (r + 8) * kStagePitch + 8 * q + fc) = make_float2(acc[4 * jj + 2], acc[4 * jj + 3]);
        }
      }
      named_bar_sync(1, kEpiThreads);
      uint32_t raw[32];
      stage_ld32(stage + row * kStagePitch + part * 32, raw);
      const int col0 = t * kTileN + half * 64 + part * 32;
      uint32_t kill = 0;
      while (next_seen < col0 + 32) {
        if (next_seen >= col0) kill |= 1u << (next_seen - col0);
        next_seen = pre_seen;
        ++ci;
        pre_seen = ci + 1 < S ? sp[ci + 1] : kNoId;
      }
      if (col0 + 32 > n_items) kill |= (col0 >= n_items) ? 0xffffffffu : (0xffffffffu << (n_items - col0));
      if (bias != nullptr) {
#pragma unroll
        for (int q = 0; q < 32; q += 4) {
          const float4 b4 = __ldg(reinterpret_cast<const float4*>(bias + col0 + q));
          raw[q] = __float_as_uint(__uint_as_float(raw[q]) + b4.x);
          raw[q + 1] = __float_as_uint(__uint_as_float(raw[q + 1]) + b4.y);
          raw[q + 2] = __float_as_uint(__uint_as_float(raw[q + 2]) + b4.z);
          raw[q + 3] = __float_as_uint(__uint_as_float(raw[q + 3]) + b4.w);
        }
      }
      // admission: above the row's own K-th best (columns arrive in ascending order, so a tie loses to the list) and at or
      // above the shared K-th best of the other splits (a tie may win there on its smaller column)
      const float own = live ? s_thr[row] : INFINITY;  // rows beyond the batch never admit
      float m = __uint_as_float(raw[0]);
#pragma unroll
      for (int q = 1; q < 32; ++q) m = fmaxf(m, __uint_as_float(raw[q]));
      bool full = false;
      if (m > own && m >= gmin) {
        uint32_t hit = 0;
#pragma unroll
        for (int q = 0; q < 32; ++q) {
          const float v = __uint_as_float(raw[q]);
          hit |= (v > own && v >= gmin) ? (1u << q) : 0u;
        }
        hit &= ~kill;
        if (hit) {
          const int nh = __popc(hit);
          int slot = atomicAdd(&s_cnt[row], nh);
          full = slot + nh > C - 64;
#pragma unroll
          for (int q = 0; q < 32; ++q)
            if (hit & (1u << q)) rb[slot++] = wide_key(raw[q], col0 + q);
        }
      }
      if (__syncthreads_or(full)) {
        compact(C - 64);
        __syncthreads();
      }
    }
  }
  // end of the range: at most K entries per row
  compact(K);
  __syncthreads();
  if (threadIdx.x < kTileM && live) cand_n[list0 + (size_t)row * n_splits] = s_cnt[row];
}

// One CTA per user: the top K keys over the user's n_splits candidate lists, sorted.  Keys below the best K-th score that
// any split published cannot be in the top K and are skipped.  Slots that no finite candidate fills get the user's masked
// columns in ascending order with score -inf, as in topk_merge_kernel.
static constexpr int kMergeThreads = 256;
__global__ void __launch_bounds__(kMergeThreads)
topk_wide_merge_kernel(const uint64_t* __restrict__ cand, const int32_t* __restrict__ cand_n,
                       const uint32_t* __restrict__ row_thr, int C, int n_splits, const int32_t* __restrict__ seen_sorted,
                       int S, int n_items, int K, const int64_t* __restrict__ candidates, int64_t* __restrict__ out_ids,
                       float* __restrict__ out_scores) {
  __shared__ uint32_t hist[256];
  __shared__ uint64_t sel[kWideMaxK];
  __shared__ int s_bin[3], s_nsel;
  const int u = blockIdx.x, tid = threadIdx.x, lane = tid & 31;
  const uint64_t floor_key = (uint64_t)row_thr[u] << 32;
  const uint64_t* lists = cand + (size_t)u * n_splits * C;
  const int32_t* counts = cand_n + (size_t)u * n_splits;
  uint64_t prefix = 0, mask = 0;
  int need = K;
  for (int shift = 56; shift >= 0; shift -= 8) {
    hist[tid] = 0u;
    __syncthreads();
    for (int s = 0; s < n_splits; ++s) {
      const uint64_t* l = lists + (size_t)s * C;
      const int n = counts[s];
      for (int i = tid; i < n; i += kMergeThreads) {
        const uint64_t key = l[i];
        if (key >= floor_key && (key & mask) == prefix) atomicAdd(hist + ((key >> shift) & 255u), 1u);
      }
    }
    __syncthreads();
    if (tid < 32) {
      uint32_t tot = 0;
      for (int j = 0; j < 8; ++j) tot += hist[8 * lane + j];
#pragma unroll
      for (int off = 16; off > 0; off >>= 1) tot += __shfl_xor_sync(0xffffffffu, tot, off);
      int b = 0, above = 0, in_b = (int)tot;  // fewer than `need` keys left: keep them all
      if (tot > (uint32_t)need) radix_find_bin(hist, need, lane, b, above, in_b);
      if (lane == 0) {
        s_bin[0] = tot > (uint32_t)need ? b : -1;
        s_bin[1] = above;
        s_bin[2] = in_b;
      }
    }
    __syncthreads();
    const int b = s_bin[0];
    if (b < 0) break;  // the keys matching the prefix are all kept
    need -= s_bin[1];
    prefix |= (uint64_t)b << shift;
    mask |= (uint64_t)0xff << shift;
    if (s_bin[2] == need) break;
    __syncthreads();  // s_bin is rewritten in the next pass
  }
  if (tid == 0) s_nsel = 0;
  __syncthreads();
  for (int s = 0; s < n_splits; ++s) {
    const uint64_t* l = lists + (size_t)s * C;
    const int n = counts[s];
    for (int i = tid; i < n; i += kMergeThreads) {
      const uint64_t key = l[i];
      if (key >= floor_key && (key & mask) >= prefix) sel[atomicAdd(&s_nsel, 1)] = key;
    }
  }
  __syncthreads();
  const int n_sel = s_nsel;
  int np = 1;
  while (np < n_sel) np <<= 1;
  for (int i = n_sel + tid; i < np; i += kMergeThreads) sel[i] = 0ull;  // 0 is below every key
  __syncthreads();
  for (int k = 2; k <= np; k <<= 1) {  // bitonic sort, descending
    for (int jj = k >> 1; jj > 0; jj >>= 1) {
      for (int i = tid; i < np; i += kMergeThreads) {
        const int ixj = i ^ jj;
        if (ixj > i) {
          const bool up = (i & k) == 0;
          const uint64_t a = sel[i], b = sel[ixj];
          if ((a < b) == up) {
            sel[i] = b;
            sel[ixj] = a;
          }
        }
      }
      __syncthreads();
    }
  }
  for (int k = tid; k < n_sel; k += kMergeThreads) {
    const uint64_t key = sel[k];
    const int col = (int)~(uint32_t)key;
    out_ids[(size_t)u * K + k] = candidates ? candidates[col] : (int64_t)col;
    out_scores[(size_t)u * K + k] = key2f((uint32_t)(key >> 32));
  }
  if (n_sel < K && tid == 0) {
    int ci = 0;
    int prev = -1;
    for (int k = n_sel; k < K; ++k) {
      int col = kNoId;
      while (seen_sorted && ci < S) {
        const int c = seen_sorted[(size_t)u * S + ci++];
        if (c != prev && c < n_items) {
          col = c;
          prev = c;
          break;
        }
      }
      out_ids[(size_t)u * K + k] = (col == kNoId) ? -1 : (candidates ? candidates[col] : (int64_t)col);
      out_scores[(size_t)u * K + k] = -INFINITY;
    }
  }
}

template <int KCH, int NSTAGE>
static int launch_score_topk_wide(const CUtensorMap& tmA, const CUtensorMap& tmB, const int32_t* seen_sorted, int S, int B,
                                  int I, int K, int C, int n_splits, const float* bias, uint64_t* cand, int32_t* cand_n,
                                  uint32_t* row_thr, cudaStream_t stream) {
  const int smem = (KCH + NSTAGE) * kChunkBytes + 128 * kStagePitch * 4 + 1024;
  const int grid = ((B + kTileM - 1) / kTileM) * n_splits;
  auto kern = score_topk_wide_kernel<KCH, NSTAGE>;
  RP_CUDA_CHECK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  kern<<<grid, kThreads, smem, stream>>>(tmA, tmB, seen_sorted, S, B, I, K, C, n_splits, bias, cand, cand_n, row_thr);
  RP_LAUNCH_CHECK();
  return RP_OK;
}

static int score_topk_wide(const CUtensorMap& tmA, const CUtensorMap& tmB, const float* bias, const int32_t* seen_sorted,
                           int S, int n_users, int n_items, int d, int K, const int64_t* candidates, int64_t* out_ids,
                           float* out_scores, void* workspace, cudaStream_t stream) {
  const int ut = (n_users + kTileM - 1) / kTileM, it = (n_items + kTileN - 1) / kTileN;
  const int C = wide_capacity(K), p = wide_splits(ut, it, C);
  uint64_t* cand = reinterpret_cast<uint64_t*>(workspace);
  int32_t* cand_n = reinterpret_cast<int32_t*>(cand + (size_t)n_users * p * C);
  uint32_t* row_thr = reinterpret_cast<uint32_t*>(cand_n + (size_t)n_users * 64);
  RP_CUDA_CHECK(cudaMemsetAsync(row_thr, 0, (size_t)n_users * 4, stream));
  int rc;
  switch (d) {
    case 64: rc = launch_score_topk_wide<1, 8>(tmA, tmB, seen_sorted, S, n_users, n_items, K, C, p, bias, cand, cand_n, row_thr, stream); break;
    case 128: rc = launch_score_topk_wide<2, 8>(tmA, tmB, seen_sorted, S, n_users, n_items, K, C, p, bias, cand, cand_n, row_thr, stream); break;
    case 256: rc = launch_score_topk_wide<4, 6>(tmA, tmB, seen_sorted, S, n_users, n_items, K, C, p, bias, cand, cand_n, row_thr, stream); break;
    default: rc = launch_score_topk_wide<8, 3>(tmA, tmB, seen_sorted, S, n_users, n_items, K, C, p, bias, cand, cand_n, row_thr, stream); break;
  }
  if (rc != RP_OK) return rc;
  topk_wide_merge_kernel<<<n_users, kMergeThreads, 0, stream>>>(cand, cand_n, row_thr, C, p, seen_sorted, S, n_items, K,
                                                                candidates, out_ids, out_scores);
  RP_LAUNCH_CHECK();
  return RP_OK;
}

}  // namespace rp

RP_API size_t rp_score_topk_workspace(int n_users, int n_items, int d, int K) {
  (void)d;
  if (n_users <= 0 || n_items <= 0 || K <= 0) return 0;
  const int ut = (n_users + rp::kTileM - 1) / rp::kTileM, it = (n_items + rp::kTileN - 1) / rp::kTileN;
  if (K > 32) {
    // more users can mean fewer item splits and a smaller layout: take the largest over smaller user-tile counts too, so
    // that the size never shrinks as the call grows (a caller that sized for more users can always serve fewer)
    const int C = rp::wide_capacity(K);
    size_t bytes = rp::wide_layout_bytes(n_users, it, C);
    for (int t = 1; t < ut && t <= rp::sm_count(); ++t) {
      const size_t b = rp::wide_layout_bytes(t * rp::kTileM, it, C);
      bytes = b > bytes ? b : bytes;
    }
    return bytes + 256;
  }
  const int p = rp::choose_splits(ut, it);
  return (size_t)n_users * p * rp::kColParts * K * 8 + (size_t)n_users * 4 + 256;
}

RP_API int rp_seen_prepare(const int64_t* seen_ids, int n_users, int S, int item_count, const int32_t* inv_map,
                    int32_t* out_sorted, void* stream_) {
  using namespace rp;
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (!seen_ids || !out_sorted) return RP_EINVAL;
  if (n_users <= 0 || S <= 0) return RP_ESHAPE;
  if (S <= 64) seen_prepare_kernel<64><<<n_users, 64, 0, stream>>>(seen_ids, S, item_count, inv_map, out_sorted);
  else if (S <= 256) seen_prepare_kernel<256><<<n_users, 128, 0, stream>>>(seen_ids, S, item_count, inv_map, out_sorted);
  else if (S <= 1024) seen_prepare_kernel<1024><<<n_users, 256, 0, stream>>>(seen_ids, S, item_count, inv_map, out_sorted);
  else if (S <= 4096) seen_prepare_kernel<4096><<<n_users, 512, 0, stream>>>(seen_ids, S, item_count, inv_map, out_sorted);
  else return RP_ESHAPE;
  RP_LAUNCH_CHECK();
  return RP_OK;
}

RP_API int rp_score_topk(const void* hq, const void* table, const float* bias, const int32_t* seen_sorted, int S, int n_users,
                  int n_items, int d, int K, const int64_t* candidates, int64_t* out_ids, float* out_scores,
                  void* workspace, size_t workspace_bytes, void* stream_) {
  using namespace rp;
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (!hq || !table || !out_ids || !out_scores || !workspace) return RP_EINVAL;
  if (n_users <= 0 || n_items <= 0 || K <= 0 || K > kWideMaxK || K > n_items) return RP_ESHAPE;
  if (d != 64 && d != 128 && d != 256 && d != 512) return RP_ESHAPE;
  if (seen_sorted && S <= 0) return RP_ESHAPE;
  if (workspace_bytes < rp_score_topk_workspace(n_users, n_items, d, K)) return RP_EWORKSPACE;
  CUtensorMap tmA, tmB;
  int rc;
  if ((rc = make_tmap_bf16(&tmA, hq, n_users, d, d, 128)) != RP_OK) return rc;
  if ((rc = make_tmap_bf16(&tmB, table, n_items, d, d, 128)) != RP_OK) return rc;
  if (K > 32)
    return score_topk_wide(tmA, tmB, bias, seen_sorted, S, n_users, n_items, d, K, candidates, out_ids, out_scores, workspace,
                           stream);
  const int ut = (n_users + kTileM - 1) / kTileM, it = (n_items + kTileN - 1) / kTileN;
  const int p = choose_splits(ut, it);
  float* pv = reinterpret_cast<float*>(workspace);
  int32_t* pi = reinterpret_cast<int32_t*>(pv + (size_t)n_users * p * kColParts * K);
  uint32_t* row_thr = reinterpret_cast<uint32_t*>(pi + (size_t)n_users * p * kColParts * K);
  RP_CUDA_CHECK(cudaMemsetAsync(row_thr, 0, (size_t)n_users * 4, stream));
  switch (d) {
    case 64: rc = launch_score_topk<1, 8>(tmA, tmB, seen_sorted, S, n_users, n_items, K, p, bias, pv, pi, row_thr, stream); break;
    case 128: rc = launch_score_topk<2, 8>(tmA, tmB, seen_sorted, S, n_users, n_items, K, p, bias, pv, pi, row_thr, stream); break;
    case 256: rc = launch_score_topk<4, 6>(tmA, tmB, seen_sorted, S, n_users, n_items, K, p, bias, pv, pi, row_thr, stream); break;
    default: rc = launch_score_topk<8, 3>(tmA, tmB, seen_sorted, S, n_users, n_items, K, p, bias, pv, pi, row_thr, stream); break;
  }
  if (rc != RP_OK) return rc;
  const int threads = 128;
  const int blocks = (n_users * 32 + threads - 1) / threads;
  topk_merge_kernel<<<blocks, threads, 0, stream>>>(pv, pi, seen_sorted, S, n_users, n_items, K, p * kColParts, candidates, out_ids,
                                                    out_scores);
  RP_LAUNCH_CHECK();
  return RP_OK;
}

