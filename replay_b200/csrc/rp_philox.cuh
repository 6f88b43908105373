// rp_philox.cuh - counter-based RNGs: the forward and the backward regenerate the same dropout mask from
// (seed, site offset, row, column) instead of storing it (drop_row_key / drop_col_key / drop_mix below); Philox4x32-10 stays
// where a reference-grade stream matters (the BERT4Rec token masker).
#pragma once
#include <stdint.h>

namespace rp {

__host__ __device__ __forceinline__ uint4 philox4x32(unsigned long long seed, unsigned long long ctr) {
  const uint32_t M0 = 0xD2511F53u, M1 = 0xCD9E8D57u, W0 = 0x9E3779B9u, W1 = 0xBB67AE85u;
  uint32_t c0 = (uint32_t)ctr, c1 = (uint32_t)(ctr >> 32), c2 = 0u, c3 = 0u;
  uint32_t k0 = (uint32_t)seed, k1 = (uint32_t)(seed >> 32);
#pragma unroll
  for (int r = 0; r < 10; ++r) {
#ifdef __CUDA_ARCH__
    const uint32_t hi0 = __umulhi(M0, c0), lo0 = M0 * c0;
    const uint32_t hi1 = __umulhi(M1, c2), lo1 = M1 * c2;
#else
    const unsigned long long p0 = (unsigned long long)M0 * c0, p1 = (unsigned long long)M1 * c2;
    const uint32_t hi0 = (uint32_t)(p0 >> 32), lo0 = (uint32_t)p0, hi1 = (uint32_t)(p1 >> 32), lo1 = (uint32_t)p1;
#endif
    const uint32_t n0 = hi1 ^ c1 ^ k0, n1 = lo1, n2 = hi0 ^ c3 ^ k1, n3 = lo0;
    c0 = n0; c1 = n1; c2 = n2; c3 = n3;
    k0 += W0; k1 += W1;
  }
  return make_uint4(c0, c1, c2, c3);
}

__host__ __device__ __forceinline__ uint32_t fmix32(uint32_t h) {  // murmur3 finaliser: full avalanche in 5 steps
  h ^= h >> 16;
  h *= 0x85EBCA6Bu;
  h ^= h >> 13;
  h *= 0xC2B2AE35u;
  h ^= h >> 16;
  return h;
}

// Dropout draws.  The attention forward walks the [query, key] matrix by query rows, the fused backward by key rows, the
// activation kernels by token rows - so the mask must be computable per element in any order - and it is a large integer
// cost of those kernels (a full hash finaliser per element would dominate them): a row key and a column key are hashed
// once each and mixed cheaply per element.  The draw for element (row r, column j) of a site is
//   drop_mix(drop_row_key(seed, site offset, r), drop_col_key(j))
// (attention probabilities: r = (batch*head)*Lp + query, j = key; activations [T, d]: r = token row, j = feature column)
// with the two well-mixed 32-bit keys computed once per row / per key (shared-memory tables) and a two-multiply mix per
// element; keep <=> draw >= p * 2^32.  (4096 x 256 grid at p = 0.2: mean 0.7995, row / column correlations at the
// sampling-noise floor, no 2x2 interaction.)
__host__ __device__ __forceinline__ uint32_t drop_row_key(unsigned long long seed, unsigned long long off, unsigned long long row) {
  const uint32_t s = fmix32((uint32_t)seed ^ ((uint32_t)(seed >> 32) * 0x85EBCA77u) ^ ((uint32_t)(off >> 32) * 0xC2B2AE3Du) ^
                            ((uint32_t)off * 0x27D4EB2Fu));
  return fmix32(s + (uint32_t)row * 0x9E3779B1u + (uint32_t)(row >> 32) * 0x165667B1u);
}
__host__ __device__ __forceinline__ uint32_t drop_col_key(uint32_t j) { return fmix32(j * 0x9E3779B1u + 0x27D4EB2Fu); }
__host__ __device__ __forceinline__ uint32_t drop_mix(uint32_t row_key, uint32_t col_key) {
  uint32_t x = (row_key ^ col_key) * 0x9E3779B1u;
  x ^= x >> 15;
  return x * 0x85EBCA77u;
}

}  // namespace rp
