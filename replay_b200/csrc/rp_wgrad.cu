// rp_wgrad.cu - ALL weight and bias gradients of one transformer block in one launch (+ one reduction launch).
//
//   dW_i[n_out_i, n_in_i] (+)= dY_i[T, n_out_i]^T . X_i[T, n_in_i]        db_i[n_out_i] (+)= sum_t dY_i[t, :]      i < n_pairs
//
// Replaces the autograd weight / bias gradients of the projections and FFN layers of a block
//   (replay/nn/sequential/sasrec/transformer.py:36-46,99-110 ; replay/nn/ffn.py:43-57 ;
//    replay/models/nn/sequential/sasrec/model.py:407-414,490-506 ; replay/models/nn/sequential/bert4rec/model.py:471-527)
// that round 1 ran as 5-6 split-K GEMM launches + as many reduction launches + a column-sum launch per block.
//
// The contraction runs over the tokens, so both operands are read IN PLACE as MN-major tiles (rows = 64 tokens of the
// row-major activation, TMA -> 128B-swizzled shared memory -> wgmma).  Work unit = one 128 x BN tile of one dW and one
// slab of the tokens; the grid is ~one CTA per SM (units x token splits).  The bias gradient rides on the tensor core too:
// one extra N = 16 MMA per k-step against a resident tile of ones gives the column sums of the dY tile that is already in
// shared memory (no extra pass over dY, no float atomics).  Every CTA stores its fp32 partial tile; `wgrad_reduce_kernel` adds
// the partials in a fixed order (deterministic) into the gradient buffers.
#include <string.h>

#include "rp_host.h"
#include "rp_sm90.cuh"

namespace rp {

static constexpr int kWgMaxPairs = 8;
static constexpr int kWgMaxUnits = 48;
static constexpr int kWgThreads = 256;   // warpgroup g: output rows [64 g, 64 g + 64) of the tile; thread 0 feeds the ring
static constexpr int kWgStages = 5;

struct WgradParams {
  CUtensorMap tmA[kWgMaxPairs];   // dY_i: [T rows, n_out_i cols], box [64 tokens x 64 features]
  CUtensorMap tmB[kWgMaxPairs];   // X_i : [T rows, n_in_i cols],  box [64 tokens x 64 features]
  int unit_pair[kWgMaxUnits], unit_m0[kWgMaxUnits], unit_n0[kWgMaxUnits];
  int n_units, splits, T;
  const int32_t* n_rows_dev;   // packed rows: the token count lives on the device (<= T, which sizes the maps), or null
  float* part;     // [n_units][splits][128 * BN]
  float* part_b;   // [n_units][splits][128]
};

template <int BN>
__global__ void __launch_bounds__(kWgThreads, 1) wgrad_group_kernel(const __grid_constant__ WgradParams p) {
  constexpr int A_BYTES = 2 * 8192;            // [64 tok x 128 out] as two [64 x 64] boxes
  constexpr int B_BYTES = (BN / 64) * 8192;    // [64 tok x BN in]
  constexpr int STAGE = A_BYTES + B_BYTES;
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sOnes = smem;                       // bf16 ones (8 KB): K-major B operand [16 x 64] of the bias MMA
  uint8_t* sRing = smem + 8192;
  __shared__ uint64_t bar_full[kWgStages], bar_empty[kWgStages];

  const int lane = threadIdx.x & 31;
  const int unit = blockIdx.x / p.splits, split = blockIdx.x % p.splits;
  const int pair = p.unit_pair[unit], m0 = p.unit_m0[unit], n0 = p.unit_n0[unit];
  const bool do_bias = (n0 == 0);              // exactly one column tile per dY row block carries the bias gradient
  const int T = p.n_rows_dev ? *p.n_rows_dev : p.T;
  const int chunks = (T + 63) / 64;
  const int c_begin = (int)(((long long)chunks * split) / p.splits);
  const int c_end = (int)(((long long)chunks * (split + 1)) / p.splits);
  const CUtensorMap* tmA = &p.tmA[pair];
  const CUtensorMap* tmB = &p.tmB[pair];

  if (threadIdx.x == 0) {
    for (int i = 0; i < kWgStages; ++i) {
      mbar_init(&bar_full[i], 1);
      mbar_init(&bar_empty[i], 8);
    }
    fence_barrier_init();
    tma_prefetch_desc(tmA);
    tma_prefetch_desc(tmB);
  }
  for (int i = threadIdx.x; i < 8192 / 4; i += kWgThreads) reinterpret_cast<uint32_t*>(sOnes)[i] = 0x3F803F80u;  // bf16 1.0 x 2
  fence_proxy_async();
  __syncthreads();
  const int n_it = c_end - c_begin;
  auto issue = [&](int it) {   // thread 0: token chunk c_begin + it -> stage it % kWgStages
    const uint32_t s = it % kWgStages;
    mbar_wait(&bar_empty[s], ((it / kWgStages) & 1) ^ 1);
    mbar_arrive_expect_tx(&bar_full[s], STAGE);
    uint8_t* sa = sRing + s * STAGE;
    uint8_t* sb = sa + A_BYTES;
    const int c = c_begin + it;
    tma_load_2d(sa, tmA, &bar_full[s], m0, c * 64);
    tma_load_2d(sa + 8192, tmA, &bar_full[s], m0 + 64, c * 64);
#pragma unroll
    for (int q = 0; q < BN / 64; ++q) tma_load_2d(sb + q * 8192, tmB, &bar_full[s], n0 + q * 64, c * 64);
  };
  if (threadIdx.x == 0)
    for (int it = 0; it < kWgStages && it < n_it; ++it) issue(it);

  const int wg = threadIdx.x >> 7, t = threadIdx.x & 127;
  float acc[BN / 2], accb[8];
  acc_zero(acc);   // (more splits than token chunks: the partial is zero)
  acc_zero(accb);
  const uint32_t ones = smem_u32(sOnes);
  for (int it = 0; it < n_it; ++it) {
    const uint32_t s = it % kWgStages, ph = (it / kWgStages) & 1;
    mbar_wait(&bar_full[s], ph);
    if (p.n_rows_dev && (c_begin + it) * 64 + 64 > T) {
      // the last chunk of a packed batch: its rows [T, ...) are stale (not zero-filled by TMA, possibly not even finite), so
      // they are cleared in every box of the stage before the MMAs read it
      const int r0 = T - (c_begin + it) * 64, per = (64 - r0) * 8;
      uint8_t* st = sRing + s * STAGE;
      for (int i = threadIdx.x; i < (STAGE / 8192) * per; i += kWgThreads)
        *reinterpret_cast<uint4*>(st + (i / per) * 8192 + (r0 + (i % per) / 8) * 128 + (i % 8) * 16) = make_uint4(0u, 0u, 0u, 0u);
      fence_proxy_async();
      __syncthreads();
    }
    const uint32_t a0 = smem_u32(sRing + s * STAGE) + wg * 8192, b0 = smem_u32(sRing + s * STAGE + A_BYTES);
    wg_fence();
#pragma unroll
    for (int ks = 0; ks < 4; ++ks) {  // 16 tokens per k-step = 16 rows x 128 B of every [64 x 64] box
      const uint64_t ad = desc_mn(a0 + ks * 2048, 8192);
      WgmmaSS<BN>::template run<1, 1>(acc, ad, desc_mn(b0 + ks * 2048, 8192), 1);
      if (do_bias) WgmmaSS<16>::template run<1, 0>(accb, ad, desc_k(ones + ks * 32), 1);
    }
    wg_commit();
    wg_wait<0>();
    wg_fence_acc(acc);
    wg_fence_acc(accb);
    __syncwarp();
    if (lane == 0) mbar_arrive(&bar_empty[s]);
    if (threadIdx.x == 0 && it + kWgStages < n_it) issue(it + kWgStages);
  }
  // ------------------------------------------------ partial tile: rows 64 wg + frag_row (+ 8), fp32
  const int ra = 64 * wg + frag_row(t), fc = frag_col(t);
  float* oa = p.part + ((size_t)(unit * p.splits + split) * 128 + ra) * BN;
  float* ob = oa + 8 * BN;
#pragma unroll
  for (int j = 0; j < BN / 8; ++j) {
    *reinterpret_cast<float2*>(oa + 8 * j + fc) = make_float2(acc[4 * j], acc[4 * j + 1]);
    *reinterpret_cast<float2*>(ob + 8 * j + fc) = make_float2(acc[4 * j + 2], acc[4 * j + 3]);
  }
  if (do_bias && fc == 0) {   // every column of the ones product holds the row's sum
    p.part_b[(size_t)(unit * p.splits + split) * 128 + ra] = accb[0];
    p.part_b[(size_t)(unit * p.splits + split) * 128 + ra + 8] = accb[2];
  }
}

struct WgradReduceParams {
  float* dW[kWgMaxPairs];
  float* db[kWgMaxPairs];
  long long ld_dw[kWgMaxPairs];
  int n_out[kWgMaxPairs], n_in[kWgMaxPairs];
  int unit_pair[kWgMaxUnits], unit_m0[kWgMaxUnits], unit_n0[kWgMaxUnits];
  int n_units, splits, bn, accumulate;
  const float* part;
  const float* part_b;
};

// grid = (n_units, blocks per unit); 256 threads = 32 float4 columns x 8 split groups (as reduce_splits_kernel in rp_gemm.cu):
// ~splits independent 16-byte loads per output column are in flight instead of one serial chain; fixed summation order.
__global__ void __launch_bounds__(256) wgrad_reduce_kernel(const __grid_constant__ WgradReduceParams p) {
  __shared__ float4 red[8][32];
  const int unit = blockIdx.x;
  const int pair = p.unit_pair[unit], m0 = p.unit_m0[unit], n0 = p.unit_n0[unit];
  const int col = threadIdx.x & 31, sg = threadIdx.x >> 5;
  const int n_elem = 128 * p.bn;  // elements of one partial tile
  const float* src = p.part + (size_t)unit * p.splits * n_elem;
  for (int i0 = blockIdx.y * 128; i0 < n_elem; i0 += gridDim.y * 128) {
    const int i = i0 + col * 4;
    float4 a = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int s = sg; s < p.splits; s += 8) {
      const float4 v = __ldg(reinterpret_cast<const float4*>(src + (size_t)s * n_elem + i));
      a.x += v.x; a.y += v.y; a.z += v.z; a.w += v.w;
    }
    red[sg][col] = a;
    __syncthreads();
    if (sg == 0) {
      const int r = i / p.bn, c = i % p.bn;
      if (m0 + r < p.n_out[pair] && n0 + c < p.n_in[pair]) {
        float* dst = p.dW[pair] + (size_t)(m0 + r) * p.ld_dw[pair] + n0 + c;
        float4 t = p.accumulate ? *reinterpret_cast<const float4*>(dst) : make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
        for (int g = 0; g < 8; ++g) {
          const float4 v = red[g][col];
          t.x += v.x; t.y += v.y; t.z += v.z; t.w += v.w;
        }
        *reinterpret_cast<float4*>(dst) = t;
      }
    }
    __syncthreads();
  }
  // bias gradient of this unit's 128 output rows (column tile 0 only)
  if (n0 == 0 && blockIdx.y == 0 && p.db[pair] != nullptr && threadIdx.x < 128) {
    const int r = threadIdx.x;
    if (m0 + r < p.n_out[pair]) {
      const float* sb = p.part_b + (size_t)unit * p.splits * 128 + r;
      float t = 0.f;
      for (int s = 0; s < p.splits; ++s) t += sb[(size_t)s * 128];
      float* dst = p.db[pair] + m0 + r;
      *dst = (p.accumulate ? *dst : 0.f) + t;
    }
  }
}

}  // namespace rp

using namespace rp;

struct rp_wgrad_pair {
  const void* dY; long long dy_ld; int n_out;   // bf16 [T, n_out] with row pitch dy_ld (elements)
  const void* X; long long x_ld; int n_in;      // bf16 [T, n_in]  with row pitch x_ld
  float* dW; long long dw_ld;                   // fp32 [n_out, n_in] with row pitch dw_ld
  float* db;                                    // fp32 [n_out] or NULL
};

static int wgrad_plan(const rp_wgrad_pair* pairs, int n_pairs, int* bn_out, int* n_units_out, int* splits_out,
                      int* up, int* um, int* un) {
  if (!pairs || n_pairs <= 0 || n_pairs > kWgMaxPairs) return RP_EINVAL;
  int bn = 128;
  for (int i = 0; i < n_pairs; ++i) {
    if (pairs[i].n_out <= 0 || pairs[i].n_in <= 0 || pairs[i].n_out % 64 || pairs[i].n_in % 64) return RP_ESHAPE;
    if (pairs[i].n_in == 64) bn = 64;
  }
  for (int i = 0; i < n_pairs; ++i)
    if (pairs[i].n_in % bn) return RP_ESHAPE;  // BN = 64 only when every n_in is a multiple of 64 (always) - kept for clarity
  int n_units = 0;
  for (int i = 0; i < n_pairs; ++i)
    for (int m0 = 0; m0 < pairs[i].n_out; m0 += 128)
      for (int n0 = 0; n0 < pairs[i].n_in; n0 += bn) {
        if (n_units >= kWgMaxUnits) return RP_ESHAPE;
        if (up) { up[n_units] = i; um[n_units] = m0; un[n_units] = n0; }
        ++n_units;
      }
  int splits = sm_count() / n_units;
  if (splits < 1) splits = 1;
  if (splits > 64) splits = 64;
  *bn_out = bn; *n_units_out = n_units; *splits_out = splits;
  return RP_OK;
}

// workspace for rp_wgrad_group with these output shapes (bytes)
RP_API size_t rp_wgrad_group_workspace(const rp_wgrad_pair* pairs, int n_pairs) {
  int bn, nu, sp;
  if (wgrad_plan(pairs, n_pairs, &bn, &nu, &sp, nullptr, nullptr, nullptr) != RP_OK) return 0;
  return (size_t)nu * sp * (128 * bn + 128) * sizeof(float);
}

static int wgrad_group(const rp_wgrad_pair* pairs, int n_pairs, int T, int accumulate, const int32_t* n_rows_dev,
                       void* workspace, size_t workspace_bytes, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (T <= 0 || !workspace) return RP_EINVAL;
  WgradParams p;
  WgradReduceParams r;
  memset(&p, 0, sizeof(p));
  memset(&r, 0, sizeof(r));
  int bn, nu, sp, rc;
  if ((rc = wgrad_plan(pairs, n_pairs, &bn, &nu, &sp, p.unit_pair, p.unit_m0, p.unit_n0)) != RP_OK) return rc;
  if (workspace_bytes < (size_t)nu * sp * (128 * bn + 128) * sizeof(float)) return RP_EWORKSPACE;
  for (int i = 0; i < n_pairs; ++i) {
    if (!pairs[i].dY || !pairs[i].X || !pairs[i].dW) return RP_EINVAL;
    if (pairs[i].dw_ld % 4 || (reinterpret_cast<uintptr_t>(pairs[i].dW) & 15)) return RP_EALIGN;
    if ((rc = make_tmap_bf16(&p.tmA[i], pairs[i].dY, T, pairs[i].n_out, pairs[i].dy_ld, 64)) != RP_OK) return rc;
    if ((rc = make_tmap_bf16(&p.tmB[i], pairs[i].X, T, pairs[i].n_in, pairs[i].x_ld, 64)) != RP_OK) return rc;
    r.dW[i] = pairs[i].dW; r.db[i] = pairs[i].db; r.ld_dw[i] = pairs[i].dw_ld;
    r.n_out[i] = pairs[i].n_out; r.n_in[i] = pairs[i].n_in;
  }
  p.n_units = nu; p.splits = sp; p.T = T; p.n_rows_dev = n_rows_dev;
  p.part = reinterpret_cast<float*>(workspace);
  p.part_b = p.part + (size_t)nu * sp * 128 * bn;
  memcpy(r.unit_pair, p.unit_pair, sizeof(p.unit_pair));
  memcpy(r.unit_m0, p.unit_m0, sizeof(p.unit_m0));
  memcpy(r.unit_n0, p.unit_n0, sizeof(p.unit_n0));
  r.n_units = nu; r.splits = sp; r.bn = bn; r.accumulate = accumulate;
  r.part = p.part; r.part_b = p.part_b;
  const int smem = 8192 + kWgStages * (2 * 8192 + (bn / 64) * 8192) + 1024;
  if (bn == 128) {
    RP_CUDA_CHECK(cudaFuncSetAttribute(wgrad_group_kernel<128>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    wgrad_group_kernel<128><<<nu * sp, kWgThreads, smem, stream>>>(p);
  } else {
    RP_CUDA_CHECK(cudaFuncSetAttribute(wgrad_group_kernel<64>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    wgrad_group_kernel<64><<<nu * sp, kWgThreads, smem, stream>>>(p);
  }
  RP_LAUNCH_CHECK();
  int by = (2 * sm_count() + nu - 1) / nu;
  const int max_by = (128 * bn) / 128;
  if (by > max_by) by = max_by;
  wgrad_reduce_kernel<<<dim3(nu, by), 256, 0, stream>>>(r);
  RP_LAUNCH_CHECK();
  return RP_OK;
}

// All pairs share the token count T.  accumulate != 0: dW / db += result, else they are overwritten.
RP_API int rp_wgrad_group(const rp_wgrad_pair* pairs, int n_pairs, int T, int accumulate, void* workspace,
                          size_t workspace_bytes, void* stream_) {
  return wgrad_group(pairs, n_pairs, T, accumulate, nullptr, workspace, workspace_bytes, stream_);
}

// Packed rows: the contraction covers the first *n_rows_dev of the T rows (T, the capacity, sizes the maps).
RP_API int rp_wgrad_group_rows(const rp_wgrad_pair* pairs, int n_pairs, int T, int accumulate, const int32_t* n_rows_dev,
                               void* workspace, size_t workspace_bytes, void* stream_) {
  if (!n_rows_dev) return RP_EINVAL;
  return wgrad_group(pairs, n_pairs, T, accumulate, n_rows_dev, workspace, workspace_bytes, stream_);
}
