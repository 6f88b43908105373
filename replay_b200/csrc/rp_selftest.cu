// rp_selftest.cu - single-CTA wgmma bring-up test: D[128,128] = A[128,128] * B[128,128]^T in the operand modes the
// production kernels rely on.  Exposed through the C ABI as rp_selftest_mma so a GPU test can pin the descriptor
// encodings (K-major / MN-major shared-memory operands, A operand from registers) against a plain matmul.
// rp_selftest_exp2 applies the two exp2 helpers of the CE passes (ex2_poly, ex2f) to an array, so they can be tested apart
// from the GEMMs around them.
#include "rp_host.h"
#include "rp_sm90.cuh"

namespace rp {

// mode bit 0: B is MN-major (global Bt[K,N])   bit 1: A from registers   bit 2: A is MN-major (global At[K,M])
// One warpgroup computes the two 64-row halves of D one after the other.
template <int MODE>
__global__ void __launch_bounds__(128, 1)
mma_selftest_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                    const __nv_bfloat16* __restrict__ Araw, float* __restrict__ D) {
  constexpr bool B_MN = (MODE & 1) != 0;
  constexpr bool A_REG = (MODE & 2) != 0;
  constexpr bool A_MN = (MODE & 4) != 0;
  constexpr int N = 128, K = 128;
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sA = smem;            // 32 KB
  uint8_t* sB = smem + 32768;    // 32 KB
  __shared__ uint64_t bar_full;
  const int t = threadIdx.x;

  if (t == 0) {
    mbar_init(&bar_full, 1);
    fence_barrier_init();
  }
  __syncthreads();
  if (t == 0) {
    mbar_arrive_expect_tx(&bar_full, 32768 + (A_REG ? 0 : 32768));
    if (!A_REG) {
      // two boxes of [128 rows x 64 cols]; for K-major these are the two K chunks, for MN-major the two M chunks
      tma_load_2d(sA, &tmA, &bar_full, 0, 0);
      tma_load_2d(sA + 16384, &tmA, &bar_full, 64, 0);
    }
    tma_load_2d(sB, &tmB, &bar_full, 0, 0);
    tma_load_2d(sB + 16384, &tmB, &bar_full, 64, 0);
  }
  mbar_wait(&bar_full, 0);
  const int fr = frag_row(t), fc = frag_col(t);
#pragma unroll 1
  for (int h = 0; h < 2; ++h) {
    float acc[N / 2];
    wg_fence();
#pragma unroll
    for (int ks = 0; ks < K / 16; ++ks) {
      const uint64_t bdesc = B_MN ? desc_mn(smem_u32(sB) + ks * 2048, 16384)
                                  : desc_k(smem_u32(sB) + (ks / 4) * 16384 + (ks % 4) * 32);
      if (A_REG) {
        // fragment of rows 64 h + fr (+ 8), columns 16 ks + fc (+ 1) and + 8
        const uint32_t* a0 = reinterpret_cast<const uint32_t*>(Araw + (size_t)(64 * h + fr) * K + 16 * ks + fc);
        const uint32_t* a8 = reinterpret_cast<const uint32_t*>(Araw + (size_t)(64 * h + fr + 8) * K + 16 * ks + fc);
        const uint32_t a[4] = {a0[0], a8[0], a0[4], a8[4]};
        WgmmaRS<N>::template run<B_MN>(acc, a, bdesc, ks > 0);
      } else {
        const uint64_t adesc = A_MN ? desc_mn(smem_u32(sA) + h * 16384 + ks * 2048, 16384)
                                    : desc_k(smem_u32(sA) + (ks / 4) * 16384 + h * 8192 + (ks % 4) * 32);
        WgmmaSS<N>::template run<A_MN, B_MN>(acc, adesc, bdesc, ks > 0);
      }
    }
    wg_commit();
    wg_wait<0>();
    wg_fence_acc(acc);
#pragma unroll
    for (int j = 0; j < N / 8; ++j) {
      float* d0 = D + (size_t)(64 * h + fr) * N + 8 * j + fc;
      float* d8 = D + (size_t)(64 * h + fr + 8) * N + 8 * j + fc;
      d0[0] = acc[4 * j]; d0[1] = acc[4 * j + 1];
      d8[0] = acc[4 * j + 2]; d8[1] = acc[4 * j + 3];
    }
  }
}

__global__ void exp2_selftest_kernel(const float* __restrict__ x, float* __restrict__ y_poly, float* __restrict__ y_mufu,
                                     long long n) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const float v = x[i];
    y_poly[i] = ex2_poly(v);
    y_mufu[i] = ex2f(v);
  }
}

// Probe (tools/probe_tma.py): how fast can ONE SM pull [box_rows x 64] bf16 boxes of a K-major [rows, d] table through TMA
// into a 6-stage ring when nothing consumes them?  Every CTA streams `tiles` row tiles (all d/64 chunks each), CTAs start
// at different tiles.  The ceiling this gives bounds the B-operand feed of score_topk / CE kernels (32 KB per 128x128 tile).
__global__ void __launch_bounds__(64, 1) tma_probe_kernel(const __grid_constant__ CUtensorMap tm, int n_row_tiles, int kch,
                                                          int tiles, int box_bytes, int same_tile) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  constexpr int NST = 6;
  __shared__ uint64_t bar_full[NST];
  if (threadIdx.x == 0) {
    for (int i = 0; i < NST; ++i) mbar_init(&bar_full[i], 1);
    fence_barrier_init();
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    uint32_t it = 0;
    for (int t = 0; t < tiles; ++t) {
      const int rt = same_tile ? (int)(blockIdx.x % n_row_tiles) : (int)((blockIdx.x * 7 + t) % n_row_tiles);
      for (int kc = 0; kc < kch; ++kc, ++it) {
        const uint32_t s = it % NST;
        if (it >= NST) mbar_wait(&bar_full[s], ((it / NST) - 1) & 1);  // the previous load into this slot has landed
        mbar_arrive_expect_tx(&bar_full[s], box_bytes);
        tma_load_2d(smem + s * 32768, &tm, &bar_full[s], kc * 64, rt * (box_bytes / 128));
      }
    }
    for (uint32_t k = (it > NST ? it - NST : 0); k < it; ++k) mbar_wait(&bar_full[k % NST], (k / NST) & 1);
  }
  __syncthreads();
}

// Probe (tools/probe_mma.py): issue rate of wgmma 64xNx16 bf16 for the operand forms the kernels use, with nothing else
// going on: one warpgroup issues `iters` groups of 8 k16 steps (K = 128) on fixed shared-memory / register operands
// (contents irrelevant) and the CTA reports elapsed SM cycles.  mode bit0: B MN-major, bit1: A from registers, bit2: A
// MN-major, bits 3-4: N = 128 / 256 / 64.
template <int N>
__device__ __forceinline__ float mma_probe_run(int mode, int iters, uint32_t a0, uint32_t b0) {
  const bool b_mn = mode & 1, a_reg = mode & 2, a_mn = mode & 4;
  float acc[N / 2];
  acc_zero(acc);
  const uint32_t areg[4] = {0x3c003c00u, 0x3c003c00u, 0x3c003c00u, 0x3c003c00u};
  for (int it = 0; it < iters; ++it) {
    wg_fence();
#pragma unroll
    for (int ks = 0; ks < 8; ++ks) {
      const uint64_t ad = a_mn ? desc_mn(a0 + ks * 2048, 16384) : desc_k(a0 + (ks >> 2) * 16384 + (ks & 3) * 32);
      const uint64_t bd = b_mn ? desc_mn(b0 + ks * 2048, 16384) : desc_k(b0 + (ks >> 2) * (N * 128) + (ks & 3) * 32);
      if (a_reg) {
        if (b_mn) WgmmaRS<N>::template run<1>(acc, areg, bd, 1);
        else WgmmaRS<N>::template run<0>(acc, areg, bd, 1);
      } else if (a_mn) {
        if (b_mn) WgmmaSS<N>::template run<1, 1>(acc, ad, bd, 1);
        else WgmmaSS<N>::template run<1, 0>(acc, ad, bd, 1);
      } else {
        if (b_mn) WgmmaSS<N>::template run<0, 1>(acc, ad, bd, 1);
        else WgmmaSS<N>::template run<0, 0>(acc, ad, bd, 1);
      }
    }
    wg_commit();
    wg_wait<1>();
  }
  wg_wait<0>();
  wg_fence_acc(acc);
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < N / 2; ++i) s += acc[i];
  return s;
}

__global__ void __launch_bounds__(128, 1) mma_probe_kernel(int mode, int iters, long long* cycles_out) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  for (int i = threadIdx.x; i < 98304 / 4; i += blockDim.x) reinterpret_cast<uint32_t*>(smem)[i] = 0x3c003c00u;
  fence_proxy_async();
  __syncthreads();
  const int nsel = (mode >> 3) & 3;
  const uint32_t a0 = smem_u32(smem), b0 = smem_u32(smem + 32768);
  const long long t0 = clock64();
  float s;
  if (nsel == 1) s = mma_probe_run<256>(mode, iters, a0, b0);
  else if (nsel == 2) s = mma_probe_run<64>(mode, iters, a0, b0);
  else s = mma_probe_run<128>(mode, iters, a0, b0);
  const long long t1 = clock64();
  // the accumulator sum feeds the result (0 or 1 extra cycle) so that the MMAs cannot be dropped
  if (threadIdx.x == 0) cycles_out[blockIdx.x] = t1 - t0 + (s == 1.2345f ? 1 : 0);
}

}  // namespace rp

RP_API int rp_selftest_mma_probe(int mode, int iters, int grid, long long* cycles_out, void* stream_) {
  using namespace rp;
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (mode < 0 || mode > 31 || iters <= 0 || grid <= 0 || !cycles_out) return RP_EINVAL;
  const int smem = 98304 + 1024;
  RP_CUDA_CHECK(cudaFuncSetAttribute(mma_probe_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  mma_probe_kernel<<<grid, 128, smem, stream>>>(mode, iters, cycles_out);
  RP_LAUNCH_CHECK();
  return RP_OK;
}

RP_API int rp_selftest_tma_probe(const void* table, long long rows, int d, int box_rows, int tiles, int same_tile, int grid,
                                 void* stream_) {
  using namespace rp;
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  CUtensorMap tm;
  int rc;
  if (!table || rows <= 0 || d % 64 || (box_rows != 64 && box_rows != 128 && box_rows != 256)) return RP_EINVAL;
  if ((rc = make_tmap_bf16(&tm, table, rows, d, d, box_rows)) != RP_OK) return rc;
  const int smem = 6 * 32768 + 1024;
  RP_CUDA_CHECK(cudaFuncSetAttribute(tma_probe_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  tma_probe_kernel<<<grid, 64, smem, stream>>>(tm, (int)(rows / box_rows), d / 64, tiles, box_rows * 128, same_tile);
  RP_LAUNCH_CHECK();
  return RP_OK;
}

RP_API int rp_selftest_exp2(const float* x, float* y_poly, float* y_mufu, long long n, void* stream_) {
  using namespace rp;
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (!x || !y_poly || !y_mufu || n < 0) return RP_EINVAL;
  if (n == 0) return RP_OK;
  const long long blocks = (n + 255) / 256;
  exp2_selftest_kernel<<<(int)(blocks < 4096 ? blocks : 4096), 256, 0, stream>>>(x, y_poly, y_mufu, n);
  RP_LAUNCH_CHECK();
  return RP_OK;
}

RP_API int rp_selftest_mma(int mode, const void* A, const void* B, float* D, void* stream_) {
  using namespace rp;
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  CUtensorMap tmA, tmB;
  int rc;
  // every operand is a [128,128] bf16 row-major array; what the rows mean depends on the mode
  if ((rc = make_tmap_bf16(&tmA, A, 128, 128, 128, 128)) != RP_OK) return rc;
  if ((rc = make_tmap_bf16(&tmB, B, 128, 128, 128, 128)) != RP_OK) return rc;
  const int smem = 65536 + 1024;
  const __nv_bfloat16* a = reinterpret_cast<const __nv_bfloat16*>(A);
#define RP_ST_CASE(m)                                                                                      \
  case m:                                                                                                  \
    RP_CUDA_CHECK(cudaFuncSetAttribute(mma_selftest_kernel<m>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem)); \
    mma_selftest_kernel<m><<<1, 128, smem, stream>>>(tmA, tmB, a, D);                                     \
    break;
  switch (mode) {
    RP_ST_CASE(0)
    RP_ST_CASE(1)
    RP_ST_CASE(2)
    RP_ST_CASE(3)
    RP_ST_CASE(4)
    RP_ST_CASE(5)
    default:
      return RP_EINVAL;
  }
#undef RP_ST_CASE
  RP_LAUNCH_CHECK();
  return RP_OK;
}
