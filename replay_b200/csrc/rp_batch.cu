// rp_batch.cu - device-side batch construction (SURVEY.md §8 f.1): all user histories live in HBM as one CSR store
// (offsets + item ids); one launch cuts, left-pads, shifts and masks the windows of a whole batch.  Replaces the per-sample
// host path of the reference: TorchSequentialDataset.__getitem__ / _pad_sequence / _generate_padding_mask
// (replay/data/nn/torch_sequential_dataset.py:69-136), SasRecTrainingDataset.__getitem__
// (replay/models/nn/sequential/sasrec/dataset.py:104-126), Bert4RecUniformMasker.mask + Bert4RecTrainingDataset.__getitem__
// (replay/models/nn/sequential/bert4rec/dataset.py:71-92,163-177), _shift_features (bert4rec/dataset.py:322-351) and the
// default collate that stacks the samples; and the new path's torch-op version of the same thing: Array1DColumn.__getitem__
// (replay/data/nn/parquet/impl/array_1d_column.py:70-84, indexing.py:42-78) + NextTokenTransform
// (replay/nn/transform/next_token.py:65-96), ~10 small kernels there.
//
// HBM-bound integer work: per row one CSR offset pair + <= W item ids are read (coalesced along the window) and W x
// (8 + 1 [+ 8 + 1]) bytes are written; one CTA per batch row so the BERT masker's row-wide all()/any() fix-ups are block
// reductions.
//
// rp_build_batch_features adds the store's feature columns (one entry per event, aligned with the item ids) to the same
// launch: after the row's ids, every column's [L(, width)] slab of the row is written through the same window, offset and
// shift, with the column's own padding value.  Loads and stores run along the flattened (position, element) axis, so
// consecutive threads touch consecutive events' values.  Query lists (one list per history: ground-truth and train items
// of validation batches) ride in the same launch as [width] rows read by the row's history index.
#include "rp_b200.h"
#include "rp_host.h"
#include "rp_philox.cuh"

namespace rp {

enum { kSasrecTrain = 0, kPredict = 1, kBertTrain = 2, kBertPredict = 3 };

struct BatchArgs {
  const int64_t* offsets;
  const int32_t* items;
  const int32_t* seq_index;
  const int32_t* seq_offset;
  const int64_t* query_ids;
  const float* uniforms;
  int64_t* ids;
  uint8_t* pad_mask;
  int64_t* labels;
  uint8_t* aux_mask;
  int64_t* query_out;
  long long n_seq;
  int B, L, mode, pad_value;
  float mask_prob;
  unsigned long long seed, draw0;
};

// window position w of a W-wide left-padded window holding the n items [first, first+n) of the history
__device__ __forceinline__ int64_t window_item(const int32_t* __restrict__ items, long long first, int n, int W, int w,
                                               int pad_value) {
  const int k = w - (W - n);
  return k >= 0 ? (int64_t)items[first + k] : (int64_t)pad_value;
}

// one batch row: the ids, masks, labels and query id of row b (every thread of the CTA takes part)
__device__ __forceinline__ void build_row(const BatchArgs& a, const int b) {
  const int s = a.seq_index[b];
  const long long beg = a.offsets[s], end = a.offsets[s + 1];
  const int len = (int)(end - beg);
  const int shift = a.mode == kSasrecTrain ? 1 : 0;
  const int L = a.L, W = L + shift;
  int off = a.seq_offset ? a.seq_offset[b] : max(0, len - W);
  off = min(max(off, 0), len);
  const int n = min(len - off, W);  // items inside the window; the mask has exactly n trailing ones
  const long long first = beg + off;
  if (threadIdx.x == 0 && a.query_out) a.query_out[b] = a.query_ids ? a.query_ids[s] : (int64_t)s;

  int64_t* ids = a.ids + (size_t)b * L;
  uint8_t* pm = a.pad_mask + (size_t)b * L;

  if (a.mode == kSasrecTrain) {
    // inputs = window[:-1], labels = window[1:], masks likewise (sasrec/dataset.py:107-118)
    int64_t* lab = a.labels + (size_t)b * L;
    uint8_t* tm = a.aux_mask + (size_t)b * L;
    for (int p = threadIdx.x; p < L; p += blockDim.x) {
      ids[p] = window_item(a.items, first, n, W, p, a.pad_value);
      pm[p] = p >= W - n;
      lab[p] = window_item(a.items, first, n, W, p + 1, a.pad_value);
      tm[p] = p + 1 >= W - n;
    }
    return;
  }
  if (a.mode == kPredict) {
    for (int p = threadIdx.x; p < L; p += blockDim.x) {
      ids[p] = window_item(a.items, first, n, W, p, a.pad_value);
      pm[p] = p >= W - n;
    }
    return;
  }
  if (a.mode == kBertPredict) {
    // roll the window left by one, last slot = padding; token_mask = shifted pad mask, pad_mask = that with last = 1
    uint8_t* tk = a.aux_mask + (size_t)b * L;
    for (int p = threadIdx.x; p < L; p += blockDim.x) {
      const bool last = p == L - 1;
      ids[p] = last ? (int64_t)a.pad_value : window_item(a.items, first, n, W, p + 1, a.pad_value);
      const uint8_t t = last ? 0 : (uint8_t)(p + 1 >= W - n);
      tk[p] = t;
      pm[p] = last ? 1 : t;
    }
    return;
  }
  // kBertTrain: inputs = positive_labels = window; token_mask[p] = (u[p] * pad[p]) >= mask_prob, then the two corner-case
  // fix-ups of Bert4RecUniformMasker.mask (all kept -> mask the last token; none kept -> un-mask the one before last)
  int64_t* lab = a.labels + (size_t)b * L;
  uint8_t* tk = a.aux_mask + (size_t)b * L;
  int all_kept = 1, any_kept = 0;
  for (int p = threadIdx.x; p < L; p += blockDim.x) {
    const int64_t v = window_item(a.items, first, n, W, p, a.pad_value);
    const bool real = p >= W - n;
    ids[p] = v;
    lab[p] = v;
    pm[p] = real;
    float u;
    if (a.uniforms) {
      u = a.uniforms[(size_t)b * L + p];
    } else {
      // uniform in [0,1) with 24 random bits, like torch.rand(float32); one Philox block per 4 positions of one draw
      const uint4 r = philox4x32(a.seed, (a.draw0 + (unsigned long long)b) * (unsigned long long)((L + 3) / 4) + (p >> 2));
      const uint32_t w = (p & 3) == 0 ? r.x : (p & 3) == 1 ? r.y : (p & 3) == 2 ? r.z : r.w;
      u = (float)(w >> 8) * (1.0f / 16777216.0f);
    }
    const bool keep = (u * (real ? 1.f : 0.f)) >= a.mask_prob;
    tk[p] = keep;
    all_kept &= keep ? 1 : 0;
    any_kept |= keep ? 1 : 0;
  }
  all_kept = __syncthreads_and(all_kept);
  any_kept = __syncthreads_or(any_kept);
  if (threadIdx.x == 0) {
    if (all_kept) tk[L - 1] = 0;
    else if (!any_kept && L > 1) tk[L - 2] = 1;
  }
}

__global__ void __launch_bounds__(128) build_batch_kernel(const BatchArgs a) { build_row(a, blockIdx.x); }

struct ColumnArgs {
  rp_batch_column c[RP_BATCH_MAX_COLUMNS];
  int n;
};

template <typename T> __device__ __forceinline__ T pad_of(const rp_batch_column& c);
template <> __device__ __forceinline__ int64_t pad_of<int64_t>(const rp_batch_column& c) { return (int64_t)c.pad_int; }
template <> __device__ __forceinline__ float pad_of<float>(const rp_batch_column& c) { return (float)c.pad_float; }
template <> __device__ __forceinline__ double pad_of<double>(const rp_batch_column& c) { return c.pad_float; }

// the event (absolute store index) behind output position p of this row, or -1 for padding: the ids' rule of build_row
struct RowWindow {
  long long first;
  int n, W, L, skip;  // skip = 1: output p reads window position p + 1 and the last position is padding (BERT predict)
  __device__ __forceinline__ long long event(int p) const {
    if (skip && p == L - 1) return -1;
    const int k = p + skip - (W - n);
    return k >= 0 ? first + k : -1;
  }
};

// integer and float columns: [L, width] outputs, flattened so consecutive threads read consecutive values
template <typename In, typename Out>
__device__ __forceinline__ void copy_dense(const rp_batch_column& c, const RowWindow& w, size_t row) {
  const In* __restrict__ v = reinterpret_cast<const In*>(c.values);
  const int wd = c.width;
  Out* out = reinterpret_cast<Out*>(c.out) + row * (size_t)w.L * wd;
  const Out pad = pad_of<Out>(c);
  for (int i = threadIdx.x; i < w.L * wd; i += blockDim.x) {
    const int p = wd == 1 ? i : i / wd;
    const long long e = w.event(p);
    out[i] = e >= 0 ? (Out)v[e * wd + (i - p * wd)] : pad;
  }
}

// list columns: each event's last `width` entries, left-padded
template <typename In>
__device__ __forceinline__ void copy_list(const rp_batch_column& c, const RowWindow& w, size_t row) {
  const In* __restrict__ v = reinterpret_cast<const In*>(c.values);
  const int K = c.width;
  int64_t* out = reinterpret_cast<int64_t*>(c.out) + row * (size_t)w.L * K;
  for (int i = threadIdx.x; i < w.L * K; i += blockDim.x) {
    const int p = i / K, j = i - p * K;
    const long long e = w.event(p);
    int64_t x = (int64_t)c.pad_int;
    if (e >= 0) {
      const long long lo = c.list_offsets[e], hi = c.list_offsets[e + 1];
      const int m = (int)min(hi - lo, (long long)K);
      const int kk = j - (K - m);
      if (kk >= 0) x = (int64_t)v[hi - m + kk];
    }
    out[i] = x;
  }
}

// query lists: one list per history, cut by the row's history index alone; head = first entries right-padded (legacy),
// else last entries left-padded (new path)
template <typename In>
__device__ __forceinline__ void copy_query_list(const rp_batch_column& c, int s, size_t row, bool head) {
  const In* __restrict__ v = reinterpret_cast<const In*>(c.values);
  const int K = c.width;
  int64_t* out = reinterpret_cast<int64_t*>(c.out) + row * (size_t)K;
  const long long lo = c.list_offsets[s], hi = c.list_offsets[s + 1];
  const int m = (int)min(hi - lo, (long long)K);
  for (int j = threadIdx.x; j < K; j += blockDim.x) {
    int64_t x = (int64_t)c.pad_int;
    if (head) {
      if (j < m) x = (int64_t)v[lo + j];
    } else {
      const int kk = j - (K - m);
      if (kk >= 0) x = (int64_t)v[hi - m + kk];
    }
    out[j] = x;
  }
}

__global__ void __launch_bounds__(128) build_batch_features_kernel(const BatchArgs a, const ColumnArgs cols) {
  const int b = blockIdx.x;
  build_row(a, b);
  const int s = a.seq_index[b];
  const long long beg = a.offsets[s], end = a.offsets[s + 1];
  const int len = (int)(end - beg);
  const int shift = a.mode == kSasrecTrain ? 1 : 0;
  RowWindow w;
  w.L = a.L;
  w.W = a.L + shift;
  int off = a.seq_offset ? a.seq_offset[b] : max(0, len - w.W);
  off = min(max(off, 0), len);
  w.n = min(len - off, w.W);
  w.first = beg + off;
  w.skip = a.mode == kBertPredict ? 1 : 0;
  for (int ci = 0; ci < cols.n; ++ci) {
    const rp_batch_column& c = cols.c[ci];
    if (c.kind == RP_BATCH_COL_INT) {
      if (c.in_bytes == 4) copy_dense<int32_t, int64_t>(c, w, b);
      else copy_dense<int64_t, int64_t>(c, w, b);
    } else if (c.kind == RP_BATCH_COL_FLOAT) {
      if (c.in_bytes == 4) {
        if (c.out_bytes == 4) copy_dense<float, float>(c, w, b);
        else copy_dense<float, double>(c, w, b);
      } else {
        if (c.out_bytes == 4) copy_dense<double, float>(c, w, b);
        else copy_dense<double, double>(c, w, b);
      }
    } else if (c.kind == RP_BATCH_COL_LIST) {
      if (c.in_bytes == 4) copy_list<int32_t>(c, w, b);
      else copy_list<int64_t>(c, w, b);
    } else {
      const bool head = c.kind == RP_BATCH_COL_QUERY_LIST;
      if (c.in_bytes == 4) copy_query_list<int32_t>(c, s, b, head);
      else copy_query_list<int64_t>(c, s, b, head);
    }
  }
}

// validation and launch shared by both entry points; cols == nullptr (or no columns): the item-only kernel
static int launch_batch(const int64_t* offsets, const int32_t* items, long long n_seq, const int32_t* seq_index,
                        const int32_t* seq_offset, int B, int L, int mode, int pad_value, float mask_prob,
                        const float* uniforms, unsigned long long seed, unsigned long long draw0, const int64_t* query_ids,
                        int64_t* ids, uint8_t* pad_mask, int64_t* labels, uint8_t* aux_mask, int64_t* query_out,
                        const ColumnArgs* cols, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (!offsets || !items || !seq_index || !ids || !pad_mask || n_seq <= 0 || B < 0 || L <= 0) return RP_EINVAL;
  if (mode < kSasrecTrain || mode > kBertPredict) return RP_EINVAL;
  if ((mode == kSasrecTrain || mode == kBertTrain) && (!labels || !aux_mask)) return RP_EINVAL;
  if (mode == kBertPredict && !aux_mask) return RP_EINVAL;
  if (mode == kBertTrain && !(mask_prob >= 0.f)) return RP_EINVAL;
  if (B == 0) return RP_OK;
  BatchArgs a;
  a.offsets = offsets; a.items = items; a.seq_index = seq_index; a.seq_offset = seq_offset; a.query_ids = query_ids;
  a.uniforms = uniforms; a.ids = ids; a.pad_mask = pad_mask; a.labels = labels; a.aux_mask = aux_mask;
  a.query_out = query_out; a.n_seq = n_seq; a.B = B; a.L = L; a.mode = mode; a.pad_value = pad_value;
  a.mask_prob = mask_prob; a.seed = seed; a.draw0 = draw0;
  if (cols && cols->n > 0) build_batch_features_kernel<<<B, 128, 0, stream>>>(a, *cols);
  else build_batch_kernel<<<B, 128, 0, stream>>>(a);
  RP_LAUNCH_CHECK();
  return RP_OK;
}

}  // namespace rp

using namespace rp;

RP_API int rp_build_batch(const int64_t* offsets, const int32_t* items, long long n_seq, const int32_t* seq_index,
                          const int32_t* seq_offset, int B, int L, int mode, int pad_value, float mask_prob,
                          const float* uniforms, unsigned long long seed, unsigned long long draw0, const int64_t* query_ids,
                          int64_t* ids, uint8_t* pad_mask, int64_t* labels, uint8_t* aux_mask, int64_t* query_out,
                          void* stream_) {
  return launch_batch(offsets, items, n_seq, seq_index, seq_offset, B, L, mode, pad_value, mask_prob, uniforms, seed, draw0,
                      query_ids, ids, pad_mask, labels, aux_mask, query_out, nullptr, stream_);
}

RP_API int rp_build_batch_features(const int64_t* offsets, const int32_t* items, long long n_seq, const int32_t* seq_index,
                                   const int32_t* seq_offset, int B, int L, int mode, int pad_value, float mask_prob,
                                   const float* uniforms, unsigned long long seed, unsigned long long draw0,
                                   const int64_t* query_ids, int64_t* ids, uint8_t* pad_mask, int64_t* labels,
                                   uint8_t* aux_mask, int64_t* query_out, const rp_batch_column* cols, int n_cols,
                                   void* stream_) {
  if (n_cols < 0 || n_cols > RP_BATCH_MAX_COLUMNS || (n_cols > 0 && !cols)) return RP_EINVAL;
  ColumnArgs ca;
  ca.n = n_cols;
  for (int i = 0; i < n_cols; ++i) {
    const rp_batch_column& c = cols[i];
    if (!c.values || !c.out || c.width < 1) return RP_EINVAL;
    if ((c.in_bytes != 4 && c.in_bytes != 8) || (c.out_bytes != 4 && c.out_bytes != 8)) return RP_EINVAL;
    if (c.kind == RP_BATCH_COL_INT && (c.out_bytes != 8 || c.width != 1)) return RP_EINVAL;
    const bool lists = c.kind == RP_BATCH_COL_LIST || c.kind == RP_BATCH_COL_QUERY_LIST ||
                       c.kind == RP_BATCH_COL_QUERY_LIST_LAST;
    if (lists && (c.out_bytes != 8 || !c.list_offsets)) return RP_EINVAL;
    if (c.kind != RP_BATCH_COL_INT && c.kind != RP_BATCH_COL_FLOAT && !lists) return RP_EINVAL;
    ca.c[i] = c;
  }
  return launch_batch(offsets, items, n_seq, seq_index, seq_offset, B, L, mode, pad_value, mask_prob, uniforms, seed, draw0,
                      query_ids, ids, pad_mask, labels, aux_mask, query_out, &ca, stream_);
}
