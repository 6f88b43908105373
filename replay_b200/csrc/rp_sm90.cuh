// rp_sm90.cuh - thin inline-PTX layer for Hopper (sm_90a): mbarrier, TMA, wgmma.
// Hand-written for this project; no CUTLASS dependency.  Every kernel in csrc/ builds on these wrappers.
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "rp_wgmma.cuh"

namespace rp {

// ------------------------------------------------------------------------------------------------------------------
// misc
// ------------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ bool elect_one() {
  uint32_t pred;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "elect.sync _|p, 0xffffffff;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}\n"
      : "=r"(pred));
  return pred != 0;
}

// ------------------------------------------------------------------------------------------------------------------
// mbarrier
// ------------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
// make generic-proxy smem writes visible to the async proxy (TMA / wgmma reading smem)
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("{\n\t.reg .b64 st;\n\tmbarrier.arrive.shared::cta.b64 st, [%0];\n\t}" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("{\n\t.reg .b64 st;\n\tmbarrier.arrive.expect_tx.shared::cta.b64 st, [%0], %1;\n\t}" ::"r"(smem_u32(bar)),
               "r"(bytes)
               : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}\n"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  while (!mbar_try_wait(bar, parity)) {
  }
}
// shared-memory counter += 1 with acquire-release ordering (CTA scope); returns the previous value
__device__ __forceinline__ uint32_t smem_count_acq_rel(uint32_t* ctr) {
  uint32_t old;
  asm volatile("atom.acq_rel.cta.shared::cta.add.u32 %0, [%1], 1;" : "=r"(old) : "r"(smem_u32(ctr)) : "memory");
  return old;
}
// ------------------------------------------------------------------------------------------------------------------
// TMA (cp.async.bulk.tensor) - 2D tiled loads into shared memory, completion on an mbarrier
// ------------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* m) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
// x = innermost (contiguous) coordinate, y = row coordinate
__device__ __forceinline__ void tma_load_2d(void* smem_dst, const CUtensorMap* m, uint64_t* bar, int x, int y) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
      ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(x), "r"(y)
      : "memory");
}
// contiguous 1-D copy of `bytes` (a multiple of 16; both addresses 16-byte aligned), completion on an mbarrier like the tiles
__device__ __forceinline__ void bulk_load_1d(void* smem_dst, const void* gmem_src, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(gmem_src)), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}
// 3-D tile (x = column, y = position inside the sequence, z = sequence): see make_tmap_bf16_seq
__device__ __forceinline__ void tma_load_3d(void* smem_dst, const CUtensorMap* m, uint64_t* bar, int x, int y, int z) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
      ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(x), "r"(y), "r"(z)
      : "memory");
}
__device__ __forceinline__ void named_bar_sync(int id, int threads) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(threads) : "memory");
}
__device__ __forceinline__ void named_bar_arrive(int id, int threads) {
  asm volatile("bar.arrive %0, %1;" ::"r"(id), "r"(threads) : "memory");
}

// ------------------------------------------------------------------------------------------------------------------
// wgmma (warpgroup MMA): shared-memory descriptors, fences, and the accumulator <-> shared memory / A-operand helpers
// ------------------------------------------------------------------------------------------------------------------
// Shared-memory matrix descriptor, 128B swizzle (sm_90 layout type 1).  Tiles are written by TMA (or by st.shared in the
// same swizzle, sw128_off) with a 1024-byte aligned base.
//  K-major  tile: rows = M/N index, one row = 64 bf16 (128 B) of K, 8-row groups every 1024 B (SBO); k16 step = +32 B.
//  MN-major tile: rows = K index, one row = 64 bf16 (128 B) of M/N, 8-row groups every 1024 B (SBO), next 64-wide M/N
//                 chunk `lbo` bytes further; k16 step = +2048 B.
__device__ __forceinline__ uint64_t gmma_desc(uint32_t smem_addr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
  uint64_t d = 0;
  d |= (uint64_t)((smem_addr & 0x3FFFF) >> 4);
  d |= (uint64_t)((lbo_bytes >> 4) & 0x3FFF) << 16;
  d |= (uint64_t)((sbo_bytes >> 4) & 0x3FFF) << 32;
  d |= (uint64_t)1 << 62;  // SWIZZLE_128B
  return d;
}
__device__ __forceinline__ uint64_t desc_k(uint32_t smem_addr) { return gmma_desc(smem_addr, 16, 1024); }
__device__ __forceinline__ uint64_t desc_mn(uint32_t smem_addr, uint32_t lbo_bytes) { return gmma_desc(smem_addr, lbo_bytes, 1024); }

__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wg_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// keeps the compiler from moving accumulator reads / writes across an asynchronous wgmma
template <int R>
__device__ __forceinline__ void wg_fence_acc(float (&d)[R]) {
#pragma unroll
  for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}
template <int R>
__device__ __forceinline__ void acc_zero(float (&d)[R]) {
#pragma unroll
  for (int i = 0; i < R; ++i) d[i] = 0.f;
}
// Rows of the m64 x N accumulator fragment of warpgroup thread t (t = threadIdx.x % 128) in the warpgroup's 64 rows:
// frag_row(t) and frag_row(t) + 8; columns 8 j + frag_col(t) + {0, 1}.
__device__ __forceinline__ int frag_row(int t) { return 16 * (t >> 5) + ((t & 31) >> 2); }
__device__ __forceinline__ int frag_col(int t) { return 2 * (t & 3); }

// Store the m64 x N fragment as fp32 rows of a row-major shared-memory stage: element (r, c) of the warpgroup's tile at
// stage[(row0 + r) * pitch + col0 + c].  pitch = N + 4 words keeps the stores and the row-per-thread reads conflict-free.
template <int R>
__device__ __forceinline__ void acc_to_stage(const float (&d)[R], float* stage, int pitch, int row0, int col0) {
  const int t = threadIdx.x & 127;
  const int r = row0 + frag_row(t), c = col0 + frag_col(t);
#pragma unroll
  for (int j = 0; j < R / 4; ++j) {
    *reinterpret_cast<float2*>(stage + r * pitch + c + 8 * j) = make_float2(d[4 * j], d[4 * j + 1]);
    *reinterpret_cast<float2*>(stage + (r + 8) * pitch + c + 8 * j) = make_float2(d[4 * j + 2], d[4 * j + 3]);
  }
}
// 32 consecutive fp32 of one stage row (the per-thread chunk the row-wise epilogues work on)
__device__ __forceinline__ void stage_ld32(const float* src, uint32_t (&r)[32]) {
#pragma unroll
  for (int q = 0; q < 32; q += 4) {
    const float4 v = *reinterpret_cast<const float4*>(src + q);
    r[q] = __float_as_uint(v.x); r[q + 1] = __float_as_uint(v.y); r[q + 2] = __float_as_uint(v.z); r[q + 3] = __float_as_uint(v.w);
  }
}

// ------------------------------------------------------------------------------------------------------------------
// small math helpers
// ------------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ float ex2f(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
// 2^x on the FMA and integer pipes, for loops whose exponentials would otherwise queue on the special-function unit
// (MUFU.EX2 runs 16 lanes per clock per SM, FFMA 128).  Agrees with ex2f wherever the CE passes evaluate it: exactly +0 for
// -inf and every x < -126 (ex2f's flushed range), finite and normal on [-126, 127], relative error below 3e-6.
// x = j + f with j = round(x) from the magic-number add, f in [-1/2, 1/2].  Range reduction stays off F2I / FRND (they issue
// on the special-function unit as well).  2^f = 1 + f q(f), q a cubic relative-minimax fit; its constant term is exactly 1,
// so p >= 1 for f >= 0 and p < 1 for f < 0.  2^j is built in the exponent bits of t and the ftz multiply flushes every
// result below 2^-126 to zero, which is what .ftz does for ex2f.
__device__ __forceinline__ float ex2_poly(float x) {
  constexpr float kMagic = 12583039.f;            // 1.5 * 2^23 + 127: the low bits of t hold j + 127, the biased exponent
  x = fmaxf(x, -127.f);                           // -inf would turn f into NaN; 2^-127 flushes to 0 below
  const float t = __fadd_rn(x, kMagic);
  const float f = __fsub_rn(x, __fsub_rn(t, kMagic));
  float p = fmaf(0x1.3a02ccp-7f, f, 0x1.c9fc46p-5f);
  p = fmaf(p, f, 0x1.ec0378p-3f);
  p = fmaf(p, f, 0x1.62e12cp-1f);
  p = fmaf(p, f, 1.f);
  const float scale = __int_as_float(__float_as_int(t) << 23);   // 2^j, or 0 for j = -127
  float y;
  asm("mul.ftz.f32 %0, %1, %2;" : "=f"(y) : "f"(p), "f"(scale));
  return y;
}
__device__ __forceinline__ uint32_t pack_bf16(float lo, float hi) {
  __nv_bfloat162 v = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&v);
}
// byte offset of (row, 16-byte chunk) inside a [rows x 128 B] SWIZZLE_128B tile whose base is 1024 B aligned
__device__ __forceinline__ uint32_t sw128_off(uint32_t row, uint32_t chunk16) {
  return row * 128u + ((chunk16 ^ (row & 7u)) << 4);
}

// ------------------------------------------------------------------------------------------------------------------
// row fragments: the 64 rows x N columns of a warpgroup in the accumulator layout - element 4 j + 2 h + e of thread t is
// row frag_row(t) + 8 h, column 8 j + frag_col(t) + e.  The fused body kernels compute on this layout between their GEMMs;
// packed to bf16 (pk[2 j + h] = elements 4 j + 2 h, + 1) it is the register A operand of the next wgmma.
// ------------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ float quad_sum(float x) {  // the four threads of a quad hold the same two rows
  x += __shfl_xor_sync(0xffffffffu, x, 1);
  return x + __shfl_xor_sync(0xffffffffu, x, 2);
}
template <int R>
__device__ __forceinline__ void frag_pack(const float (&v)[R], uint32_t (&pk)[R / 2]) {
#pragma unroll
  for (int j = 0; j < R / 4; ++j) {
    pk[2 * j] = pack_bf16(v[4 * j], v[4 * j + 1]);
    pk[2 * j + 1] = pack_bf16(v[4 * j + 2], v[4 * j + 3]);
  }
}
// bf16 rows r_a and r_a + 8 (global row indices; rows >= n_rows read as zero) of a row-major array -> fragment
template <int R>
__device__ __forceinline__ void frag_load_bf16(const __nv_bfloat16* base, long long ld, int r_a, int n_rows, float (&v)[R]) {
  const int fc = frag_col(threadIdx.x & 127);
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int r = r_a + 8 * h;
    const __nv_bfloat16* row = base + (size_t)(r < n_rows ? r : 0) * ld + fc;
#pragma unroll
    for (int j = 0; j < R / 4; ++j) {
      const float2 f = r < n_rows ? __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(row + 8 * j)) : make_float2(0.f, 0.f);
      v[4 * j + 2 * h] = f.x;
      v[4 * j + 2 * h + 1] = f.y;
    }
  }
}
template <int P>
__device__ __forceinline__ void frag_store_bf16(const uint32_t (&pk)[P], __nv_bfloat16* base, long long ld, int r_a, int n_rows) {
  const int fc = frag_col(threadIdx.x & 127);
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int r = r_a + 8 * h;
    if (r >= n_rows) continue;
    __nv_bfloat16* row = base + (size_t)r * ld + fc;
#pragma unroll
    for (int j = 0; j < P / 2; ++j) *reinterpret_cast<uint32_t*>(row + 8 * j) = pk[2 * j + h];
  }
}
// rows r and r + 8 of a staged [128 x 64 KCH] bf16 tile (KCH SWIZZLE_128B chunks of 16 KB, as TMA wrote it) -> fragment
template <int R>
__device__ __forceinline__ void frag_load_tile(const uint8_t* tile, int r, float (&v)[R]) {
  const int fc = frag_col(threadIdx.x & 127);
#pragma unroll
  for (int h = 0; h < 2; ++h)
#pragma unroll
    for (int j = 0; j < R / 4; ++j) {
      const int c = 8 * j + fc;
      const uint32_t w = *reinterpret_cast<const uint32_t*>(tile + (c >> 6) * 16384 + sw128_off((uint32_t)(r + 8 * h), (uint32_t)((c & 63) >> 3)) + (c & 7) * 2);
      const float2 f = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&w));
      v[4 * j + 2 * h] = f.x;
      v[4 * j + 2 * h + 1] = f.y;
    }
}

// LayerNorm parameter gradients: per-column sums of this CTA's rows (fragment columns of every thread: cw / cb) -> one atomic per column and CTA
template <int R>
__device__ __forceinline__ void frag_colsum_commit(float (&cw)[R / 2], float (&cb)[R / 2], float* s_red /* [2][8][2R] */,
                                                   float* dln_w, float* dln_b, int n_threads) {
  constexpr int D = 2 * R;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, fc = frag_col(threadIdx.x & 127);
#pragma unroll
  for (int i = 0; i < R / 2; ++i)
#pragma unroll
    for (int o = 4; o <= 16; o <<= 1) {   // lanes with the same fragment column
      cw[i] += __shfl_xor_sync(0xffffffffu, cw[i], o);
      cb[i] += __shfl_xor_sync(0xffffffffu, cb[i], o);
    }
  if (lane < 4) {
#pragma unroll
    for (int j = 0; j < R / 4; ++j)
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        s_red[(0 * 8 + warp) * D + 8 * j + fc + e] = cw[2 * j + e];
        s_red[(1 * 8 + warp) * D + 8 * j + fc + e] = cb[2 * j + e];
      }
  }
  named_bar_sync(1, n_threads);
  for (int i = threadIdx.x; i < 2 * D; i += n_threads) {
    const int qty = i / D, col = i % D;
    float tot = 0.f;
#pragma unroll
    for (int w = 0; w < 8; ++w) tot += s_red[(qty * 8 + w) * D + col];
    atomicAdd((qty == 0 ? dln_w : dln_b) + col, tot);
  }
}

// GEMMs of a warpgroup's 64 rows against a resident weight W[N_out, K_in] (torch layout, bf16, in shared memory):
//   x . W^T  (contraction over W's input features): W K-major, chunk kc = [N rows x 64] at w0 + kc * w_chunk (default N * 128)
//   g . W    (contraction over W's output features): W read MN-major, box (kc, nc) = [64 x 64] at w0 + (kc * NC + nc) * 8192
// A operand from a staged K-major tile (a0 = the warpgroup's rows of chunk 0, chunks 16 KB apart) or from registers (pk).
template <int N, int KCH>
__device__ __forceinline__ void wg_gemm_ss_wt(float (&acc)[N / 2], uint32_t a0, uint32_t w0, uint32_t w_chunk = N * 128) {
  wg_fence();
#pragma unroll
  for (int kc = 0; kc < KCH; ++kc)
#pragma unroll
    for (int ks = 0; ks < 4; ++ks)
      WgmmaSS<N>::template run<0, 0>(acc, desc_k(a0 + kc * 16384 + ks * 32), desc_k(w0 + kc * w_chunk + ks * 32), (kc | ks) != 0);
  wg_commit();
  wg_wait<0>();
  wg_fence_acc(acc);
}
template <int N, int KCH>
__device__ __forceinline__ void wg_gemm_rs_wt(float (&acc)[N / 2], const uint32_t (&pk)[KCH * 16], uint32_t w0) {
  wg_fence();
#pragma unroll
  for (int kc = 0; kc < KCH; ++kc)
#pragma unroll
    for (int ks = 0; ks < 4; ++ks) {
      const int kk = 4 * kc + ks;
      const uint32_t a[4] = {pk[4 * kk], pk[4 * kk + 1], pk[4 * kk + 2], pk[4 * kk + 3]};
      WgmmaRS<N>::template run<0>(acc, a, desc_k(w0 + kc * (N * 128) + ks * 32), (kc | ks) != 0);
    }
  wg_commit();
  wg_wait<0>();
  wg_fence_acc(acc);
}
template <int N, int KCH>
__device__ __forceinline__ void wg_gemm_ss_w(float (&acc)[N / 2], uint32_t a0, uint32_t w0) {
  wg_fence();
#pragma unroll
  for (int kc = 0; kc < KCH; ++kc)
#pragma unroll
    for (int ks = 0; ks < 4; ++ks)
      WgmmaSS<N>::template run<0, 1>(acc, desc_k(a0 + kc * 16384 + ks * 32), desc_mn(w0 + kc * (N / 64) * 8192 + ks * 2048, 8192),
                                     (kc | ks) != 0);
  wg_commit();
  wg_wait<0>();
  wg_fence_acc(acc);
}
template <int N, int KCH>
__device__ __forceinline__ void wg_gemm_rs_w(float (&acc)[N / 2], const uint32_t (&pk)[KCH * 16], uint32_t w0) {
  wg_fence();
#pragma unroll
  for (int kc = 0; kc < KCH; ++kc)
#pragma unroll
    for (int ks = 0; ks < 4; ++ks) {
      const int kk = 4 * kc + ks;
      const uint32_t a[4] = {pk[4 * kk], pk[4 * kk + 1], pk[4 * kk + 2], pk[4 * kk + 3]};
      WgmmaRS<N>::template run<1>(acc, a, desc_mn(w0 + kc * (N / 64) * 8192 + ks * 2048, 8192), (kc | ks) != 0);
    }
  wg_commit();
  wg_wait<0>();
  wg_fence_acc(acc);
}

// ------------------------------------------------------------------------------------------------------------------
// padded feature layout ("feature slots")
// ------------------------------------------------------------------------------------------------------------------
// hd_valid > 0: PADDED feature layout (include/rp_b200.h "feature slots"): the row holds D/slot slots of `slot` = 64 (hd_valid
// <= 64) or 128 columns of which only the first hd_valid are real features; the padded columns are zero in every activation,
// weight and bias, the statistics run over the real features only and padded outputs / gradients stay zero.
__device__ __forceinline__ bool feat_valid(int col, int hd_valid) {
  return hd_valid <= 0 || (col & (hd_valid <= 64 ? 63 : 127)) < hd_valid;
}
__host__ __device__ __forceinline__ int feat_count(int D, int hd_valid) {
  return hd_valid <= 0 ? D : (D / (hd_valid <= 64 ? 64 : 128)) * hd_valid;
}


}  // namespace rp
