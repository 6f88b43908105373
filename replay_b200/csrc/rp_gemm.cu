// rp_gemm.cu - generic batched bf16 GEMM on wgmma with a fused epilogue; the workhorse of the transformer body.
//
//   C[m, n] = epilogue( alpha * sum_k A(m, k) * B(n, k) )            (per batch element)
//
// Operands may be K-major (stored [rows = M/N, cols = K]) or MN-major (stored [rows = K, cols = M/N]); both are fed to
// the tensor core straight from TMA-written 128B-swizzled shared memory (no transposes in HBM).  Replaces, on the body:
//   torch.nn.MultiheadAttention in/out projections, Conv1d(d,d,1)/Linear FFN layers and their autograd backward
//   (replay/nn/sequential/sasrec/transformer.py:36-46,99-106 ; replay/nn/ffn.py:43-57 ;
//    replay/models/nn/sequential/sasrec/model.py:407-414,490-506 ; replay/models/nn/sequential/bert4rec/model.py:471-527).
//
#include "rp_host.h"
#include "rp_philox.cuh"
#include "rp_sm90.cuh"

namespace rp {

struct GemmParams {
  int M, N, K;                 // per-batch problem size
  int inner;                   // batch index bz = outer * inner + in
  int a_r0, a_ro, a_ri;        // A row offset = a_r0 + outer*a_ro + in*a_ri   (rows of the stored 2-D array)
  int a_c0, a_co, a_ci;        // A col offset
  int b_r0, b_ro, b_ri, b_c0, b_co, b_ci;
  void* C;                     // output
  long long ldc, c_off0, c_oo, c_oi;   // element offsets: c_off0 + outer*c_oo + in*c_oi, row pitch ldc
  int out_mode;                // 0: bf16 store, 1: fp32 atomic add, 2: fp32 store, 3: fp32 store of the split-K partial at
                               //    C + ksplit * c_split_stride (reduced afterwards by rp_reduce_splits; no atomics)
  long long c_split_stride;
  float alpha;
  const float* bias;           // [N] or null
  int act;                     // 0 none, 1 relu, 2 gelu(erf), 3 exp2, 4 sigmoid (row_exp2_offset below)
  const __nv_bfloat16* residual;  // same geometry as C (bf16) or null
  const uint8_t* rowmask;      // multiply row m by (rowmask[rowmask_off0 + outer*rowmask_oo + m] != 0) or null
  long long rowmask_off0, rowmask_oo;   // row index base per batch: rowmask_off0 + outer*rowmask_oo
  float drop_p;                // dropout prob applied after act, before residual (0 = off)
  unsigned long long seed, drop_offset;
  const unsigned long long* seed_ptr;  // optional device counter added to seed (CUDA-graph replays get fresh masks)
  int split_k;                 // number of K splits (out_mode 1 / 3; alpha and rowmask are the only epilogue stages allowed)
  const __nv_bfloat16* gate;   // same geometry as C: x *= (gate != 0) ? gate_scale : 0   (ReLU+dropout backward) or null
  float gate_scale;
  __nv_bfloat16* C2;           // optional second output (bf16, geometry of C): the value after bias, before the activation
  int gate_mode;               // 0: gate != 0 ? gate_scale : 0 ;  1: gelu'(gate) * gate_scale (gate = saved pre-activation)
  float post_drop_p;           // second dropout applied AFTER the residual add (BERT4Rec block output), 0 = off
  unsigned long long post_drop_offset;
  const float* row_exp2_offset;  // act 3: x = exp2(x * log2(e) + row_exp2_offset[m])   (softmax numerators from stored lse)
                                 // act 4: x = sigmoid(x) * exp2(row_exp2_offset[m])   (BCE gradient / T_v, 0 past T_v)
  const int32_t* m_limit_dev;    // optional device scalar: rows m with m_limit_base + m >= *m_limit_dev are not computed
  int m_limit_base;
  const int32_t* k_limit_dev;    // optional device scalar: the contraction stops at *k_limit_dev - k_limit_base (whole 64-chunks)
  int k_limit_base;
};

// Epilogue of one [1 row x 32 columns] strip held in registers.
struct EpiRow {
  long long c_base;   // element offset of this output row in C
  long long drop_row; // row index of the activation dropout stream (rp_philox.cuh): element (drop_row, column)
  float rm;           // row-mask factor
  float exp_off;      // act 3: per-row exponent offset
  float keep_scale;
  uint32_t drop_thr;
  unsigned long long seed_eff;
};

// SIGMOID: the act 4 epilogue (BCE head at d = 512) is compiled only into its own instantiation, so it costs the other
// GEMMs no registers
template <bool SIGMOID>
__device__ __forceinline__ void gemm_epilogue_chunk(const GemmParams& p, const float* __restrict__ s_bias, const EpiRow& er,
                                                    const uint32_t (&raw)[32], int n0, int c) {
  const long long c_base = er.c_base;
  const float rm = er.rm, keep_scale = er.keep_scale;
  const uint32_t drop_thr = er.drop_thr;
  const unsigned long long seed_eff = er.seed_eff;
  float x[32];
#pragma unroll
      for (int q = 0; q < 32; ++q) x[q] = __uint_as_float(raw[q]) * p.alpha;
      if (p.bias) {
#pragma unroll
        for (int q = 0; q < 32; q += 4) {
          const float4 b4 = *reinterpret_cast<const float4*>(&s_bias[c + q]);
          x[q] += b4.x; x[q + 1] += b4.y; x[q + 2] += b4.z; x[q + 3] += b4.w;
        }
      }
      const bool full = (n0 + c + 32 <= p.N);
      if (p.C2) {
        __nv_bfloat16* o2 = p.C2 + c_base + n0 + c;
#pragma unroll
        for (int q = 0; q < 32; q += 2) {
          if (n0 + c + q + 1 < p.N) *reinterpret_cast<uint32_t*>(o2 + q) = pack_bf16(x[q], x[q + 1]);
          else if (n0 + c + q < p.N) o2[q] = __float2bfloat16(x[q]);   // odd N: the last column alone, not column N
        }
      }
      if (p.act == 1) {
#pragma unroll
        for (int q = 0; q < 32; ++q) x[q] = fmaxf(x[q], 0.f);
      } else if (p.act == 2) {
#pragma unroll
        for (int q = 0; q < 32; ++q) x[q] = 0.5f * x[q] * (1.f + erff(x[q] * 0.70710678118654752f));
      } else if (p.act == 3) {
#pragma unroll
        for (int q = 0; q < 32; ++q) x[q] = ex2f(fmaf(x[q], 1.4426950408889634f, er.exp_off));
      } else if (SIGMOID && p.act == 4) {  // sigmoid(x) * 2^offset: (1 or e) / (1 + e) with e = exp(-|x|); offset -inf gives exactly 0
        const float sc = ex2f(er.exp_off);
#pragma unroll
        for (int q = 0; q < 32; ++q) {
          const float e = ex2f(-fabsf(x[q]) * 1.4426950408889634f);
          x[q] = __fdividef(x[q] >= 0.f ? sc : e * sc, 1.f + e);
        }
      }
      if (p.drop_p > 0.f) {
        const uint32_t rk = drop_row_key(seed_eff, p.drop_offset, (unsigned long long)er.drop_row);
#pragma unroll
        for (int q = 0; q < 32; ++q)
          x[q] = drop_mix(rk, drop_col_key((uint32_t)(n0 + c + q))) >= drop_thr ? x[q] * keep_scale : 0.f;
      }
      if (p.gate) {
        const __nv_bfloat16* gp = p.gate + c_base + n0 + c;
        if (p.gate_mode == 0) {
#pragma unroll
          for (int q = 0; q < 32; ++q)
            if (n0 + c + q < p.N) x[q] = (__bfloat162float(gp[q]) != 0.f) ? x[q] * p.gate_scale : 0.f;
        } else {
#pragma unroll
          for (int q = 0; q < 32; ++q)
            if (n0 + c + q < p.N) {
              const float z = __bfloat162float(gp[q]);
              const float dg = 0.5f * (1.f + erff(z * 0.70710678118654752f)) + z * 0.3989422804014327f * __expf(-0.5f * z * z);
              x[q] *= dg * p.gate_scale;
            }
        }
      }
      if (p.residual) {
        const __nv_bfloat16* rp_ = p.residual + c_base + n0 + c;
        if (full) {
#pragma unroll
          for (int q = 0; q < 32; q += 8) {
            const uint4 rv = *reinterpret_cast<const uint4*>(rp_ + q);
            const __nv_bfloat162* r2 = reinterpret_cast<const __nv_bfloat162*>(&rv);
#pragma unroll
            for (int t = 0; t < 4; ++t) {
              const float2 f = __bfloat1622float2(r2[t]);
              x[q + 2 * t] += f.x;
              x[q + 2 * t + 1] += f.y;
            }
          }
        } else {
#pragma unroll
          for (int q = 0; q < 32; ++q)
            if (n0 + c + q < p.N) x[q] += __bfloat162float(rp_[q]);
        }
      }
      if (p.post_drop_p > 0.f) {
        const float ks2 = 1.f / (1.f - p.post_drop_p);
        const uint32_t thr2 = (uint32_t)(p.post_drop_p * 4294967296.0);
        const uint32_t rk = drop_row_key(p.seed + (p.seed_ptr ? *p.seed_ptr : 0ull), p.post_drop_offset, (unsigned long long)er.drop_row);
#pragma unroll
        for (int q = 0; q < 32; ++q)
          x[q] = drop_mix(rk, drop_col_key((uint32_t)(n0 + c + q))) >= thr2 ? x[q] * ks2 : 0.f;
      }
      if (p.rowmask) {
#pragma unroll
        for (int q = 0; q < 32; ++q) x[q] *= rm;
      }
      if (p.out_mode == 0) {
        __nv_bfloat16* o = reinterpret_cast<__nv_bfloat16*>(p.C) + c_base + n0 + c;
        if (full) {
#pragma unroll
          for (int q = 0; q < 32; q += 8) {
            uint4 w;
            w.x = pack_bf16(x[q], x[q + 1]);
            w.y = pack_bf16(x[q + 2], x[q + 3]);
            w.z = pack_bf16(x[q + 4], x[q + 5]);
            w.w = pack_bf16(x[q + 6], x[q + 7]);
            *reinterpret_cast<uint4*>(o + q) = w;
          }
        } else {
#pragma unroll
          for (int q = 0; q < 32; ++q)
            if (n0 + c + q < p.N) o[q] = __float2bfloat16(x[q]);
        }
      } else {
        float* o = reinterpret_cast<float*>(p.C) + c_base + n0 + c;
        if (p.out_mode == 1) {
#pragma unroll
          for (int q = 0; q < 32; ++q)
            if (n0 + c + q < p.N) atomicAdd(o + q, x[q]);
        } else if (p.out_mode == 4) {  // C += x, plain read-modify-write (every element has exactly one owner: split_k == 1)
          if (full && ((reinterpret_cast<uintptr_t>(o) & 15) == 0)) {
#pragma unroll
            for (int q = 0; q < 32; q += 4) {
              float4 v = *reinterpret_cast<float4*>(o + q);
              v.x += x[q]; v.y += x[q + 1]; v.z += x[q + 2]; v.w += x[q + 3];
              *reinterpret_cast<float4*>(o + q) = v;
            }
          } else {
#pragma unroll
            for (int q = 0; q < 32; ++q)
              if (n0 + c + q < p.N) o[q] += x[q];
          }
        } else if (full && ((reinterpret_cast<uintptr_t>(o) & 15) == 0)) {
#pragma unroll
          for (int q = 0; q < 32; q += 4) *reinterpret_cast<float4*>(o + q) = make_float4(x[q], x[q + 1], x[q + 2], x[q + 3]);
        } else {
#pragma unroll
          for (int q = 0; q < 32; ++q)
            if (n0 + c + q < p.N) o[q] = x[q];
        }
      }
}

// CTA = one 128 x BN output tile (x one K split).  Warpgroups 0 / 1: wgmma over rows [0, 64) / [64, 128) of the tile, then
// the epilogue (thread = output row, warpgroup = column half); warp 8: TMA producer.
static constexpr int kGemmThreads = 288;

template <int BN, bool A_MN, bool B_MN, int NSTAGE, bool SIGMOID = false>
__global__ void __launch_bounds__(kGemmThreads, 1)
gemm_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, const GemmParams p) {
  constexpr int A_BYTES = 128 * 128;       // [128 x 64] bf16
  constexpr int B_BYTES = BN * 128;        // [BN x 64] bf16
  constexpr int STAGE = A_BYTES + B_BYTES;
  constexpr int PITCH = BN + 4;            // fp32 accumulator stage, placed over the operand ring once the contraction ends
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  __shared__ uint64_t bar_full[NSTAGE], bar_empty[NSTAGE];
  __shared__ __align__(16) float s_bias[BN];

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  // one linear grid dimension (no 65535 limit on the row tiles of tall GEMMs): n tile fastest, then K split, then m tile -
  // CTAs launched side by side share their A rows in L2
  const int n_tiles = (p.N + BN - 1) / BN;
  const int n_tile = (int)(blockIdx.x % n_tiles);
  const int mk = (int)(blockIdx.x / n_tiles);
  const int m_tile = mk / p.split_k, ksplit = mk % p.split_k;
  const int bz = blockIdx.z, outer = bz / p.inner, in = bz % p.inner;
  const int m0 = m_tile * 128, n0 = n_tile * BN;
  if (p.m_limit_dev != nullptr && m0 + p.m_limit_base >= *p.m_limit_dev) return;  // whole tile beyond the dynamic row count
  int k_eff = p.K;
  if (p.k_limit_dev != nullptr) k_eff = max(0, min(p.K, *p.k_limit_dev - p.k_limit_base));
  const int k_chunks = (k_eff + 63) / 64;
  const int kc_begin = (int)(((long long)k_chunks * ksplit) / p.split_k);
  const int kc_end = (int)(((long long)k_chunks * (ksplit + 1)) / p.split_k);
  const int a_r = p.a_r0 + outer * p.a_ro + in * p.a_ri, a_c = p.a_c0 + outer * p.a_co + in * p.a_ci;
  const int b_r = p.b_r0 + outer * p.b_ro + in * p.b_ri, b_c = p.b_c0 + outer * p.b_co + in * p.b_ci;

  if (threadIdx.x == 0) {
    for (int i = 0; i < NSTAGE; ++i) {
      mbar_init(&bar_full[i], 1);
      mbar_init(&bar_empty[i], 8);
    }
    fence_barrier_init();
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
  }
  if (p.bias != nullptr && threadIdx.x < 256) {
    for (int i = threadIdx.x; i < BN; i += 256) s_bias[i] = (n0 + i < p.N) ? p.bias[n0 + i] : 0.f;
  }
  __syncthreads();

  if (warp == 8) {
    if (elect_one()) {
      for (int kc = kc_begin, it = 0; kc < kc_end; ++kc, ++it) {
        const uint32_t s = it % NSTAGE, ph = (it / NSTAGE) & 1;
        mbar_wait(&bar_empty[s], ph ^ 1);
        mbar_arrive_expect_tx(&bar_full[s], STAGE);
        uint8_t* sa = smem + s * STAGE;
        uint8_t* sb = sa + A_BYTES;
        if (A_MN) {  // stored [K rows, M cols]: two boxes of [64 k-rows x 64 m]
          tma_load_2d(sa, &tmA, &bar_full[s], a_c + m0, a_r + kc * 64);
          tma_load_2d(sa + 8192, &tmA, &bar_full[s], a_c + m0 + 64, a_r + kc * 64);
        } else {     // stored [M rows, K cols]: one box of [128 rows x 64 k]
          tma_load_2d(sa, &tmA, &bar_full[s], a_c + kc * 64, a_r + m0);
        }
        if (B_MN) {
#pragma unroll
          for (int c = 0; c < BN / 64; ++c)
            tma_load_2d(sb + c * 8192, &tmB, &bar_full[s], b_c + n0 + c * 64, b_r + kc * 64);
        } else {
          tma_load_2d(sb, &tmB, &bar_full[s], b_c + kc * 64, b_r + n0);
        }
      }
    }
    return;
  }
  // ------------------------------------------------ warpgroup wg: rows [64 wg, 64 wg + 64) of the tile
  const int wg = warp >> 2;
  float acc[BN / 2];
  acc_zero(acc);  // an empty contraction (dynamic K limit) leaves zeros
  for (int kc = kc_begin, it = 0; kc < kc_end; ++kc, ++it) {
    const uint32_t s = it % NSTAGE, ph = (it / NSTAGE) & 1;
    mbar_wait(&bar_full[s], ph);
    const uint32_t a0 = smem_u32(smem + s * STAGE) + wg * 8192, b0 = smem_u32(smem + s * STAGE + A_BYTES);
    wg_fence_acc(acc);
    wg_fence();
#pragma unroll
    for (int ks = 0; ks < 4; ++ks) {
      const uint64_t ad = A_MN ? desc_mn(a0 + ks * 2048, 8192) : desc_k(a0 + ks * 32);
      const uint64_t bd = B_MN ? desc_mn(b0 + ks * 2048, 8192) : desc_k(b0 + ks * 32);
      WgmmaSS<BN>::template run<A_MN, B_MN>(acc, ad, bd, 1);
    }
    wg_commit();
    wg_wait<0>();
    wg_fence_acc(acc);
    __syncwarp();
    if (lane == 0) mbar_arrive(&bar_empty[s]);
  }
  named_bar_sync(1, 256);  // both warpgroups are done reading the ring
  float* stage = reinterpret_cast<float*>(smem);
  acc_to_stage(acc, stage, PITCH, wg * 64, 0);
  named_bar_sync(1, 256);
  // ------------------------------------------------ epilogue: thread = output row, warpgroup = column half
  const int row = threadIdx.x & 127;
  const int m = m0 + row;
  const bool row_ok = m < p.M;
  const long long c_base = p.c_off0 + (long long)outer * p.c_oo + (long long)in * p.c_oi + (long long)m * p.ldc +
                           (p.out_mode == 3 ? (long long)ksplit * p.c_split_stride : 0ll);
  float rm = 1.f;
  if (p.rowmask && row_ok) rm = p.rowmask[p.rowmask_off0 + (long long)outer * p.rowmask_oo + m] ? 1.f : 0.f;
  EpiRow er;
  er.c_base = c_base;
  er.drop_row = (long long)bz * p.M + m;
  er.rm = rm;
  er.exp_off = ((p.act == 3 || (SIGMOID && p.act == 4)) && row_ok) ? p.row_exp2_offset[m] : 0.f;
  er.keep_scale = p.drop_p > 0.f ? 1.f / (1.f - p.drop_p) : 1.f;
  er.drop_thr = p.drop_p > 0.f ? (uint32_t)(p.drop_p * 4294967296.0) : 0u;
  er.seed_eff = p.seed + ((p.drop_p > 0.f && p.seed_ptr) ? *p.seed_ptr : 0ull);
  if (!row_ok) return;
#pragma unroll 1
  for (int c = wg * (BN / 2); c < (wg + 1) * (BN / 2); c += 32) {
    if (n0 + c >= p.N) break;
    uint32_t raw[32];
    stage_ld32(stage + row * PITCH + c, raw);
    gemm_epilogue_chunk<SIGMOID>(p, s_bias, er, raw, n0, c);
  }
}

template <int BN, bool A_MN, bool B_MN, int NSTAGE, bool SIGMOID = false>
static int launch_gemm_n(const CUtensorMap& tmA, const CUtensorMap& tmB, const GemmParams& p, int batch, cudaStream_t st) {
  const int ring = NSTAGE * (128 * 128 + BN * 128), stage = 128 * (BN + 4) * 4;
  const int smem = (ring > stage ? ring : stage) + 1024;
  auto kern = gemm_kernel<BN, A_MN, B_MN, NSTAGE, SIGMOID>;
  RP_CUDA_CHECK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  const long long ctas = (long long)((p.N + BN - 1) / BN) * ((p.M + 127) / 128) * p.split_k;
  if (ctas > 0x7fffffffll) return RP_ESHAPE;
  dim3 grid((unsigned)ctas, 1, batch);
  kern<<<grid, kGemmThreads, smem, st>>>(tmA, tmB, p);
  RP_LAUNCH_CHECK();
  return RP_OK;
}

// short-K problems (the body's d x d projections) use 2 stages so that several CTAs share an SM and their prologues,
// main loops and epilogues overlap; long-K problems (weight gradients) use a 4-deep ring.
template <int BN, bool A_MN, bool B_MN>
static int launch_gemm(const CUtensorMap& tmA, const CUtensorMap& tmB, const GemmParams& p, int batch, cudaStream_t st) {
  const int chunks_per_cta = ((p.K + 63) / 64 + p.split_k - 1) / p.split_k;
  if (chunks_per_cta <= 2) return launch_gemm_n<BN, A_MN, B_MN, 2>(tmA, tmB, p, batch, st);
  return launch_gemm_n<BN, A_MN, B_MN, 4>(tmA, tmB, p, batch, st);
}

}  // namespace rp

using namespace rp;

#include "rp_gemm_desc.h"

// every element offset of C's geometry (ldc, c_off0, c_oo, c_oi) is a multiple of `elems`
static bool c_geom_multiple(const rp_gemm_desc* g, long long elems) {
  return g->ldc % elems == 0 && g->c_off0 % elems == 0 && g->c_oo % elems == 0 && g->c_oi % elems == 0;
}

static bool aligned(const void* ptr, uintptr_t bytes) { return (reinterpret_cast<uintptr_t>(ptr) & (bytes - 1)) == 0; }

RP_API int rp_gemm(const rp_gemm_desc* g, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  // every argument check comes before the tensor maps are made, so it holds without a driver
  if (!g || !g->A || !g->B || !g->C) return RP_EINVAL;
  if (g->M <= 0 || g->N <= 0 || g->K <= 0 || g->batch <= 0 || g->inner <= 0) return RP_ESHAPE;
  if (g->split_k < 1 || (g->split_k > 1 && g->out_mode != 1 && g->out_mode != 3)) return RP_EINVAL;
  // each K split runs the epilogue on its partial sum: only the linear stages (alpha, rowmask) may be split
  if (g->split_k > 1 && (g->bias || g->act != 0 || g->residual || g->gate || g->C2 || g->drop_p > 0.f || g->post_drop_p > 0.f))
    return RP_EINVAL;
  // TMA boxes start at a 16-byte aligned column of the stored operands
  if ((g->a_c0 | g->a_co | g->a_ci | g->b_c0 | g->b_co | g->b_ci) & 7) return RP_EALIGN;
  if ((g->act == 3 || g->act == 4) && !g->row_exp2_offset) return RP_EINVAL;
  if (g->act == 4 && (g->a_mn || g->b_mn)) return RP_EINVAL;   // split_k > 1 with an act is rejected above
  if (g->out_mode == 4 && g->split_k != 1) return RP_EINVAL;
  // out_mode 0 stores 8 bf16 per 16-byte store, and the residual is read the same way at C's geometry; C2 is stored in
  // bf16 pairs
  if (g->out_mode == 0 && (!aligned(g->C, 16) || !c_geom_multiple(g, 8))) return RP_EALIGN;
  if (g->residual && (!aligned(g->residual, 16) || !c_geom_multiple(g, 8))) return RP_EALIGN;
  if (g->C2 && (!aligned(g->C2, 4) || !c_geom_multiple(g, 2))) return RP_EALIGN;
  GemmParams p;
  p.M = g->M; p.N = g->N; p.K = g->K; p.inner = g->inner;
  p.a_r0 = g->a_r0; p.a_ro = g->a_ro; p.a_ri = g->a_ri; p.a_c0 = g->a_c0; p.a_co = g->a_co; p.a_ci = g->a_ci;
  p.b_r0 = g->b_r0; p.b_ro = g->b_ro; p.b_ri = g->b_ri; p.b_c0 = g->b_c0; p.b_co = g->b_co; p.b_ci = g->b_ci;
  p.C = g->C; p.ldc = g->ldc; p.c_off0 = g->c_off0; p.c_oo = g->c_oo; p.c_oi = g->c_oi; p.out_mode = g->out_mode;
  p.alpha = g->alpha; p.bias = g->bias; p.act = g->act;
  p.residual = reinterpret_cast<const __nv_bfloat16*>(g->residual);
  p.rowmask = g->rowmask; p.rowmask_off0 = g->rowmask_off0; p.rowmask_oo = g->rowmask_oo;
  p.drop_p = g->drop_p; p.seed = g->seed; p.drop_offset = g->drop_offset; p.seed_ptr = g->seed_ptr; p.split_k = g->split_k;
  p.gate = reinterpret_cast<const __nv_bfloat16*>(g->gate); p.gate_scale = g->gate_scale;
  p.C2 = reinterpret_cast<__nv_bfloat16*>(g->C2); p.gate_mode = g->gate_mode; p.post_drop_p = g->post_drop_p;
  p.post_drop_offset = g->post_drop_offset;
  p.c_split_stride = g->c_split_stride;
  p.row_exp2_offset = g->row_exp2_offset;
  p.m_limit_dev = g->m_limit_dev; p.m_limit_base = g->m_limit_base;
  p.k_limit_dev = g->k_limit_dev; p.k_limit_base = g->k_limit_base;
  CUtensorMap tmA, tmB;
  int rc;
  // K-major operand: box [128 (or BN) rows x 64 cols]; MN-major operand: box [64 k-rows x 64 cols]
  const int bn = (g->N <= 64 && g->act != 4) ? 64 : 128;
  if ((rc = make_tmap_bf16(&tmA, g->A, g->a_rows, g->a_cols, g->lda, g->a_mn ? 64 : 128)) != RP_OK) return rc;
  if ((rc = make_tmap_bf16(&tmB, g->B, g->b_rows, g->b_cols, g->ldb, g->b_mn ? 64 : bn)) != RP_OK) return rc;
  if (g->act == 4)   // sigmoid epilogue: one instantiation, K-major operands and 128-column tiles (BCE logit chunks)
    return launch_gemm_n<128, false, false, 4, true>(tmA, tmB, p, g->batch, stream);
#define RP_GEMM_CASE(BN_, AMN_, BMN_) return launch_gemm<BN_, AMN_, BMN_>(tmA, tmB, p, g->batch, stream)
  if (bn == 64) {
    if (!g->a_mn && !g->b_mn) RP_GEMM_CASE(64, false, false);
    if (!g->a_mn && g->b_mn) RP_GEMM_CASE(64, false, true);
    if (g->a_mn && !g->b_mn) RP_GEMM_CASE(64, true, false);
    RP_GEMM_CASE(64, true, true);
  } else {
    if (!g->a_mn && !g->b_mn) RP_GEMM_CASE(128, false, false);
    if (!g->a_mn && g->b_mn) RP_GEMM_CASE(128, false, true);
    if (g->a_mn && !g->b_mn) RP_GEMM_CASE(128, true, false);
    RP_GEMM_CASE(128, true, true);
  }
#undef RP_GEMM_CASE
}

// dst[i] (+)= sum_s src[s * stride + i]   - second stage of the split-K weight-gradient GEMMs (out_mode 3).
// The sums are short (n = d*d elements) but deep (~100 splits): a block covers 32 float4 columns x 8 split groups so that
// ~100 independent 16-byte loads per column are in flight instead of one serial chain; fixed summation order (deterministic).
__global__ void __launch_bounds__(256) reduce_splits_kernel(const float* __restrict__ src, int n_splits, long long stride,
                                                            long long n, float* __restrict__ dst, int accumulate) {
  __shared__ float4 part[8][32];
  const int col = threadIdx.x & 31, sg = threadIdx.x >> 5;
  for (long long i0 = (long long)blockIdx.x * 128; i0 < n; i0 += (long long)gridDim.x * 128) {
    const long long i = i0 + col * 4;
    float4 a = make_float4(0.f, 0.f, 0.f, 0.f);
    if (i < n) {
      for (int s2 = sg; s2 < n_splits; s2 += 8) {
        const float4 v = __ldg(reinterpret_cast<const float4*>(src + (long long)s2 * stride + i));
        a.x += v.x; a.y += v.y; a.z += v.z; a.w += v.w;
      }
    }
    part[sg][col] = a;
    __syncthreads();
    if (sg == 0 && i < n) {
      float4 t = accumulate ? *reinterpret_cast<const float4*>(dst + i) : make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
      for (int g = 0; g < 8; ++g) {
        const float4 v = part[g][col];
        t.x += v.x; t.y += v.y; t.z += v.z; t.w += v.w;
      }
      *reinterpret_cast<float4*>(dst + i) = t;
    }
    __syncthreads();
  }
}

RP_API int rp_reduce_splits(const float* src, int n_splits, long long stride, long long n, float* dst, int accumulate,
                            void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (!src || !dst || n_splits <= 0 || n <= 0 || (n & 3) || (stride & 3)) return RP_EINVAL;
  long long blocks = (n + 127) / 128;
  if (blocks > rp::sm_count() * 8) blocks = rp::sm_count() * 8;
  reduce_splits_kernel<<<(int)blocks, 256, 0, stream>>>(src, n_splits, stride, n, dst, accumulate);
  RP_LAUNCH_CHECK();
  return RP_OK;
}
