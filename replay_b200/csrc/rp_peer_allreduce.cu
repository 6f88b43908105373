// rp_peer_allreduce.cu - sum-all-reduce of the flat fp32 gradient over NVLink peer memory, as ONE kernel that lives inside
// the captured training-step graph (between the backward kernels and Adam).
//
// Replaces  the bucketed gradient all-reduce Lightning's DDP runs under `loss.backward()` for the reference
//           (replay/nn/lightning/module.py:62-75 under Trainer(strategy="ddp"); SURVEY.md 2.1 / 8e)
// and an eager ncclAllReduce between two graph replays (launch gaps on both sides of it).
//
// Every rank holds the gradient in a buffer of the SAME symmetric allocation (torch.distributed._symmetric_memory does the
// cuMem export / import - plumbing); the kernel gets the W peer pointers by value.  Two-shot scheme:
//   start barrier   rank r tells every peer "my gradient is final" (one flag per (peer, r)), then waits for all W flags
//   reduce-scatter  rank r owns slice r: s = sum over p = 0..W-1 (fixed order) of g_p[i]   - P2P loads through NVLink
//   all-gather      ... and stores s into EVERY rank's buffer at i                         - P2P stores
//   end barrier     the last CTA to finish tells every peer "my slice is everywhere, and I have read all I needed", waits for
//                   the peers' flags and only then lets the kernel end (so the next kernel may read / overwrite the buffer)
// Each element is summed by exactly one rank in a fixed order and broadcast, so all replicas see bit-identical gradients.
// Flags carry a launch counter (epoch) that lives in device memory: nothing is reset between launches and the kernel is
// CUDA-graph capturable.  All CTAs spin on flags, so the grid never exceeds the number of SMs.
#include "rp_host.h"

namespace rp {

#ifndef RP_PEER_LD_VOLATILE
#define RP_PEER_LD_VOLATILE 0
#endif
static constexpr int kMaxPeers = 8;
struct PeerArgs {
  float* buf[kMaxPeers];        // the gradient buffer of every rank (this rank's own included), peer-mapped
  uint32_t* flags[kMaxPeers];   // [2][kMaxPeers] launch-counter flags of every rank: [0] = start barrier, [1] = end barrier
};

__device__ __forceinline__ void st_release_sys(uint32_t* p, uint32_t v) {
  asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ uint32_t ld_acquire_sys(const uint32_t* p) {
  uint32_t v;
  asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
// peer data must not come out of this SM's L1 (it may hold last step's lines): relaxed system-scope loads go to the owner
__device__ __forceinline__ float4 ld_sys_f4(const float* p) {
  float4 v;
#if RP_PEER_LD_VOLATILE
  asm volatile("ld.volatile.global.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(p) : "memory");
#else
  asm volatile("ld.relaxed.sys.global.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(p) : "memory");
#endif
  return v;
}
__device__ __forceinline__ float ld_sys_f1(const float* p) {
  float v;
  asm volatile("ld.relaxed.sys.global.f32 %0, [%1];" : "=f"(v) : "l"(p) : "memory");
  return v;
}

__device__ __forceinline__ unsigned long long global_ns() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}
// spin until *f has reached `epoch`; gives up after ~60 s (a peer process died: better a wrong gradient and a clean exit of
// this kernel than a GPU that spins until the box is reclaimed) and reports it through the state block
__device__ __forceinline__ void wait_flag(const uint32_t* f, uint32_t epoch, uint32_t* timed_out) {
  const unsigned long long t0 = global_ns();
  uint32_t polls = 0;
  while ((int32_t)(ld_acquire_sys(f) - epoch) < 0) {
    if ((++polls & 0xfffu) == 0 && global_ns() - t0 > 60000000000ull) {
      *timed_out = 1u;
      return;
    }
  }
}

__global__ void __launch_bounds__(512, 1)
peer_allreduce_kernel(const PeerArgs a, int rank, int world, long long n, uint32_t* __restrict__ epoch_dev,
                      uint32_t* __restrict__ done_ctas) {
  const uint32_t epoch = *reinterpret_cast<volatile uint32_t*>(epoch_dev) + 1;
  // ---- start barrier: this rank's backward kernels ended before this kernel began; publish that to the peers
  if (blockIdx.x == 0 && (int)threadIdx.x < world) {
    __threadfence_system();
    st_release_sys(a.flags[threadIdx.x] + 0 * kMaxPeers + rank, epoch);
  }
  if ((int)threadIdx.x < world) {
    wait_flag(a.flags[rank] + 0 * kMaxPeers + threadIdx.x, epoch, done_ctas + 1);
  }
  __syncthreads();
  // ---- this rank's slice [lo, hi), multiples of 4 floats (the last slice takes the tail)
  const long long n4 = n >> 2;
  const long long per = (n4 + world - 1) / world;
  const long long lo4 = per * rank < n4 ? per * rank : n4, hi4 = per * (rank + 1) < n4 ? per * (rank + 1) : n4;
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (long long i = lo4 + (long long)blockIdx.x * blockDim.x + threadIdx.x; i < hi4; i += stride * 2) {
    // two independent float4 columns per thread and iteration: W loads each in flight before the first add
    const long long i1 = i + stride;
    const bool two = i1 < hi4;
    float4 v0[kMaxPeers], v1[kMaxPeers];
#pragma unroll
    for (int p = 0; p < kMaxPeers; ++p)
      if (p < world) {
        v0[p] = ld_sys_f4(a.buf[p] + i * 4);
        if (two) v1[p] = ld_sys_f4(a.buf[p] + i1 * 4);
      }
    float4 s0 = v0[0], s1 = two ? v1[0] : make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
    for (int p = 1; p < kMaxPeers; ++p)
      if (p < world) {
        s0.x += v0[p].x; s0.y += v0[p].y; s0.z += v0[p].z; s0.w += v0[p].w;
        if (two) { s1.x += v1[p].x; s1.y += v1[p].y; s1.z += v1[p].z; s1.w += v1[p].w; }
      }
#pragma unroll
    for (int p = 0; p < kMaxPeers; ++p)
      if (p < world) {
        *reinterpret_cast<float4*>(a.buf[p] + i * 4) = s0;
        if (two) *reinterpret_cast<float4*>(a.buf[p] + i1 * 4) = s1;
      }
  }
  if (rank == world - 1 && blockIdx.x == 0) {   // the n % 4 tail
    for (long long i = (n4 << 2) + threadIdx.x; i < n; i += blockDim.x) {
      float s = 0.f;
      for (int p = 0; p < world; ++p) s += ld_sys_f1(a.buf[p] + i);
      for (int p = 0; p < world; ++p) a.buf[p][i] = s;
    }
  }
  // ---- end barrier, run by the last CTA of this rank to get here
  __shared__ bool last;
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence_system();   // this CTA's peer stores are on their way before the counter says so
    last = atomicAdd(done_ctas, 1u) == gridDim.x - 1;
  }
  __syncthreads();
  if (!last) return;
  if ((int)threadIdx.x < world) {
    __threadfence_system();
    st_release_sys(a.flags[threadIdx.x] + 1 * kMaxPeers + rank, epoch);
    wait_flag(a.flags[rank] + 1 * kMaxPeers + threadIdx.x, epoch, done_ctas + 1);
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    *done_ctas = 0;
    *epoch_dev = epoch;
    __threadfence();
  }
}

}  // namespace rp

using namespace rp;

// flags / counters of one rank: uint32 [2 * 8] flags + epoch + done counter + timed-out marker (non-zero: a peer never answered), zeroed once by the caller (rp_peer_allreduce_state_bytes)
RP_API size_t rp_peer_allreduce_state_bytes(void) { return (2 * kMaxPeers + 3) * sizeof(uint32_t); }

// bufs[w] / states[w]: device pointers of rank w's gradient buffer / state block as mapped into THIS process (symmetric
// memory), w = 0..world-1; n fp32 elements, 16-byte aligned buffers.  Every rank must launch it once per step.
RP_API int rp_peer_allreduce(void* const* bufs, void* const* states, int rank, int world, long long n, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (!bufs || !states) return RP_EINVAL;
  if (world < 2 || world > kMaxPeers || rank < 0 || rank >= world || n <= 0) return RP_ESHAPE;
  PeerArgs a;
  for (int w = 0; w < kMaxPeers; ++w) {
    a.buf[w] = w < world ? reinterpret_cast<float*>(bufs[w]) : nullptr;
    a.flags[w] = w < world ? reinterpret_cast<uint32_t*>(states[w]) : nullptr;
    if (w < world && (!bufs[w] || !states[w])) return RP_EINVAL;
    if (w < world && (reinterpret_cast<uintptr_t>(bufs[w]) & 15) != 0) return RP_EALIGN;
  }
  uint32_t* mine = reinterpret_cast<uint32_t*>(states[rank]);
  // enough CTAs to keep the NVLink ports busy, never more than the SMs (every CTA spins on the start flags)
  long long want = ((n >> 2) / world + 1023) / 1024;
  int grid = (int)(want < 1 ? 1 : (want > sm_count() ? sm_count() : want));
  peer_allreduce_kernel<<<grid, 512, 0, stream>>>(a, rank, world, n, mine + 2 * kMaxPeers, mine + 2 * kMaxPeers + 1);
  RP_LAUNCH_CHECK();
  return RP_OK;
}
