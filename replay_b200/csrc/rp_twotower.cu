// rp_twotower.cu - candidate compaction of the TwoTower model's sampled losses (replay/nn/sequential/twotower/model.py:
// get_logits(h, candidates) -> item_tower(candidates)).  The item tower runs only on the distinct items a sampled step
// references: this file flags them in a [n_items] scratch, numbers them in ascending item id (a two-level scan, no host
// synchronisation, so the step stays graph-captured), rewrites the positive labels and the negatives into slot ids, gathers
// the slots' embedding rows as the tower's input and, after the tower's backward, adds each slot's input gradient back into
// the item table's gradient row (one slot per item: no atomics, the same result on every run).
#include <cuda_bf16.h>

#include "rp_host.h"

namespace rp {
namespace tower {

constexpr int kThreads = 256;
constexpr int kPerThread = 16;
constexpr int kTile = kThreads * kPerThread;   // items numbered by one block of the scan

struct CompactArgs {
  const int32_t* labels;
  const int32_t* n_valid;
  int capacity;
  const int64_t* negatives;
  int n_neg, neg_mode, n_neg_rows, seq_len;
  const int32_t* valid_idx;
  int ignore_index, n_items, cap;
};

// the negative row of compacted target t: its position (neg_mode 1) or its sequence (neg_mode 2)
__device__ __forceinline__ long long neg_row(const CompactArgs& a, int t) {
  const int flat = a.valid_idx[t];
  return a.neg_mode == 1 ? flat : flat / a.seq_len;
}

// the entries this step reads: every label t < n_valid, the shared negatives, every per-sequence row, and the
// per-position rows of the valid targets.  Visits each entry once (grid-stride over a flat index).
template <class F>
__device__ __forceinline__ void for_each_entry(const CompactArgs& a, F&& f) {
  const int nv = min(*a.n_valid, a.capacity);
  const long long n_neg_entries = a.neg_mode == 0 ? a.n_neg
                                 : a.neg_mode == 2 ? (long long)a.n_neg_rows * a.n_neg
                                                   : (long long)nv * a.n_neg;
  const long long total = nv + n_neg_entries;
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (long long)gridDim.x * blockDim.x) {
    if (e < nv) {
      f(true, e, (long long)a.labels[e]);
      continue;
    }
    const long long k = e - nv;
    long long idx = k;
    if (a.neg_mode == 1) idx = neg_row(a, (int)(k / a.n_neg)) * a.n_neg + k % a.n_neg;
    f(false, idx, a.negatives[idx]);
  }
}

__device__ __forceinline__ bool ignored(const CompactArgs& a, bool is_label, long long id) {
  return !is_label && a.ignore_index >= 0 && id == (long long)a.ignore_index;
}

__global__ void __launch_bounds__(kThreads) mark_kernel(CompactArgs a, int32_t* flag) {
  for_each_entry(a, [&](bool is_label, long long, long long id) {
    if (ignored(a, is_label, id)) return;
    // an id outside the catalog reads item 0's row in the sampled head (clamp_item): keep item 0 among the candidates
    flag[(id >= 0 && id < a.n_items) ? id : 0] = 1;
  });
}

__device__ __forceinline__ int warp_incl_scan(int v) {
  const int lane = threadIdx.x & 31;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int u = __shfl_up_sync(0xffffffffu, v, o);
    if (lane >= o) v += u;
  }
  return v;
}

// exclusive block scan of one value per thread; *total receives the block's sum
__device__ __forceinline__ int block_excl_scan(int v, int* total) {
  __shared__ int s_warp[kThreads / 32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int incl = warp_incl_scan(v);
  if (lane == 31) s_warp[warp] = incl;
  __syncthreads();
  if (warp == 0) {
    const int w = lane < kThreads / 32 ? s_warp[lane] : 0;
    const int wi = warp_incl_scan(w);
    if (lane < kThreads / 32) s_warp[lane] = wi - w;
    if (lane == 31) *total = wi;
  }
  __syncthreads();
  const int out = s_warp[warp] + incl - v;
  __syncthreads();
  return out;
}

__global__ void __launch_bounds__(kThreads) tile_count_kernel(const int32_t* __restrict__ flag, int n_items, int32_t* tile_sum) {
  const long long base = (long long)blockIdx.x * kTile + (long long)threadIdx.x * kPerThread;
  int c = 0;
#pragma unroll
  for (int j = 0; j < kPerThread; ++j) c += (base + j < n_items) ? flag[base + j] : 0;
  __shared__ int s_total;
  block_excl_scan(c, &s_total);
  if (threadIdx.x == 0) tile_sum[blockIdx.x] = s_total;
}

// slot_of_item (in place over the flags): the flagged item's slot, -1 otherwise; item_of_slot[slot] = item
__global__ void __launch_bounds__(kThreads) tile_assign_kernel(int32_t* flag, int n_items, const int32_t* __restrict__ tile_sum,
                                                              int cap, int32_t* item_of_slot, int32_t* n_slots) {
  // slots before this tile: the sum of the earlier tiles (at most a few hundred), in a fixed order
  int pre = 0;
  for (int b = threadIdx.x; b < (int)blockIdx.x; b += kThreads) pre += tile_sum[b];
  __shared__ int s_total;
  block_excl_scan(pre, &s_total);
  const int before = s_total;
  const long long base = (long long)blockIdx.x * kTile + (long long)threadIdx.x * kPerThread;
  int f[kPerThread];
  int c = 0;
#pragma unroll
  for (int j = 0; j < kPerThread; ++j) {
    f[j] = (base + j < n_items) ? flag[base + j] : 0;
    c += f[j];
  }
  int slot = before + block_excl_scan(c, &s_total);
#pragma unroll
  for (int j = 0; j < kPerThread; ++j) {
    if (base + j >= n_items) break;
    if (f[j] && slot < cap) {
      flag[base + j] = slot;
      item_of_slot[slot] = (int32_t)(base + j);
    } else {
      flag[base + j] = -1;
    }
    slot += f[j];
  }
  if (blockIdx.x == gridDim.x - 1 && threadIdx.x == 0) *n_slots = min(before + s_total, cap);
}

// labels / negatives -> slot ids.  Ignored negatives become `cap` (the head is given ignore_index = cap); ids outside the
// catalog become cap + 1, which the head reads as row 0 = item 0 (flagged by mark_kernel) and never equals a positive.
__global__ void __launch_bounds__(kThreads) remap_kernel(CompactArgs a, const int32_t* __restrict__ slot_of_item,
                                                         int32_t* labels_out, int64_t* negatives_out) {
  for_each_entry(a, [&](bool is_label, long long idx, long long id) {
    long long v;
    if (ignored(a, is_label, id)) v = a.cap;
    else if (id < 0 || id >= a.n_items) v = a.cap + 1;
    else v = slot_of_item[id];
    if (is_label) labels_out[idx] = (int32_t)v;
    else negatives_out[idx] = v;
  });
}

// rows[s] = table[item_of_slot[s]] for s < n_slots, zero rows up to cap (item_of_slot = -1 there); 8 bf16 per thread.
// rows == null: only item_of_slot = -1 from n_slots on (the caller builds the rows itself)
__global__ void __launch_bounds__(kThreads) gather_kernel(const uint4* __restrict__ table, int d8, int cap,
                                                          int32_t* item_of_slot, const int32_t* n_slots, uint4* rows) {
  const int ns = *n_slots;
  const long long total = (long long)cap * d8;
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (long long)gridDim.x * blockDim.x) {
    const int s = (int)(e / d8), c = (int)(e % d8);
    if (s < ns) {
      if (rows) rows[e] = table[(long long)item_of_slot[s] * d8 + c];
    } else {
      if (rows) rows[e] = make_uint4(0u, 0u, 0u, 0u);
      if (c == 0) item_of_slot[s] = -1;
    }
  }
}

// d_table[item_of_slot[s]] += dx[s] (fp32 += bf16), s < *n_slots; identity map when item_of_slot is null
__global__ void __launch_bounds__(kThreads) scatter_kernel(const uint4* __restrict__ dx, const int32_t* __restrict__ item_of_slot,
                                                           const int32_t* n_slots, int n_rows, int d8, float* d_table) {
  const int ns = n_slots ? min(*n_slots, n_rows) : n_rows;
  const long long total = (long long)ns * d8;
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (long long)gridDim.x * blockDim.x) {
    const int s = (int)(e / d8), c = (int)(e % d8);
    const long long item = item_of_slot ? item_of_slot[s] : s;
    const uint4 v = dx[e];
    const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&v);
    float4* dst = reinterpret_cast<float4*>(d_table + (item * d8 + c) * 8);
    float4 lo = dst[0], hi = dst[1];
    const float2 a0 = __bfloat1622float2(h[0]), a1 = __bfloat1622float2(h[1]), a2 = __bfloat1622float2(h[2]),
                 a3 = __bfloat1622float2(h[3]);
    lo.x += a0.x; lo.y += a0.y; lo.z += a1.x; lo.w += a1.y;
    hi.x += a2.x; hi.y += a2.y; hi.z += a3.x; hi.w += a3.y;
    dst[0] = lo;
    dst[1] = hi;
  }
}

static int grid_for(long long work) {
  long long g = (work + kThreads - 1) / kThreads;
  const long long cap = (long long)sm_count() * 8;
  if (g > cap) g = cap;
  return g < 1 ? 1 : (int)g;
}

static int n_tiles(int n_items) { return (n_items + kTile - 1) / kTile; }

}  // namespace tower
}  // namespace rp

using namespace rp::tower;

RP_API size_t rp_tower_compact_workspace(int n_items) {
  if (n_items <= 0) return 0;
  return ((size_t)n_items + (size_t)n_tiles(n_items) + 64) * sizeof(int32_t);
}

RP_API int rp_tower_compact(const int32_t* labels, const int32_t* n_valid, int capacity, const int64_t* negatives, int n_neg,
                            int neg_mode, int n_neg_rows, const int32_t* valid_idx, int seq_len, int ignore_index, int n_items,
                            const void* table, int d, int cap, int32_t* n_slots, int32_t* item_of_slot, int32_t* labels_out,
                            int64_t* negatives_out, void* rows_out, void* workspace, size_t workspace_bytes, void* stream_) {
  if (!labels || !n_valid || !negatives || !table || !n_slots || !item_of_slot || !labels_out || !negatives_out || !workspace)
    return RP_EINVAL;
  if (neg_mode != 0 && !valid_idx) return RP_EINVAL;
  if (capacity <= 0 || n_items <= 0 || n_neg <= 0 || d <= 0 || d % 8 || cap <= 0 || cap > n_items || seq_len <= 0 ||
      neg_mode < 0 || neg_mode > 2 || (neg_mode == 2 && n_neg_rows <= 0))
    return RP_ESHAPE;
  if (((uintptr_t)table | (uintptr_t)rows_out) & 15) return RP_EALIGN;
  if (workspace_bytes < rp_tower_compact_workspace(n_items)) return RP_EWORKSPACE;
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  int32_t* flag = reinterpret_cast<int32_t*>(workspace);
  int32_t* tile_sum = flag + n_items;
  CompactArgs a{labels, n_valid, capacity, negatives, n_neg, neg_mode, n_neg_rows, seq_len, valid_idx, ignore_index, n_items, cap};
  const long long entries = (long long)capacity + (neg_mode == 0 ? n_neg : neg_mode == 2 ? (long long)n_neg_rows * n_neg
                                                                                          : (long long)capacity * n_neg);
  RP_CUDA_CHECK(cudaMemsetAsync(flag, 0, (size_t)n_items * sizeof(int32_t), stream));
  mark_kernel<<<grid_for(entries), kThreads, 0, stream>>>(a, flag);
  RP_LAUNCH_CHECK();
  const int tiles = n_tiles(n_items);
  tile_count_kernel<<<tiles, kThreads, 0, stream>>>(flag, n_items, tile_sum);
  RP_LAUNCH_CHECK();
  tile_assign_kernel<<<tiles, kThreads, 0, stream>>>(flag, n_items, tile_sum, cap, item_of_slot, n_slots);
  RP_LAUNCH_CHECK();
  remap_kernel<<<grid_for(entries), kThreads, 0, stream>>>(a, flag, labels_out, negatives_out);
  RP_LAUNCH_CHECK();
  const int d8 = rows_out ? d / 8 : 1;
  gather_kernel<<<grid_for((long long)cap * d8), kThreads, 0, stream>>>(
      reinterpret_cast<const uint4*>(table), d8, cap, item_of_slot, n_slots, reinterpret_cast<uint4*>(rows_out));
  RP_LAUNCH_CHECK();
  return RP_OK;
}

RP_API int rp_tower_scatter_rows(const void* dx, const int32_t* item_of_slot, const int32_t* n_slots, int n_rows, int d,
                                 float* d_table, void* stream_) {
  if (!dx || !d_table || (item_of_slot && !n_slots)) return RP_EINVAL;
  if (n_rows < 0 || d <= 0 || d % 8) return RP_ESHAPE;
  if (((uintptr_t)dx | (uintptr_t)d_table) & 15) return RP_EALIGN;
  if (n_rows == 0) return RP_OK;
  scatter_kernel<<<grid_for((long long)n_rows * (d / 8)), kThreads, 0, reinterpret_cast<cudaStream_t>(stream_)>>>(
      reinterpret_cast<const uint4*>(dx), item_of_slot, n_slots, n_rows, d / 8, d_table);
  RP_LAUNCH_CHECK();
  return RP_OK;
}
