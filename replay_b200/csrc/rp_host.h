// rp_host.h - host-side helpers shared by the C-ABI entry points: error codes, TMA tensor-map construction.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

// C-ABI return convention (include/rp_b200.h): 0 ok, <0 argument/shape/alignment error, >0 cudaError_t
#define RP_API extern "C" __attribute__((visibility("default")))

#define RP_OK 0
#define RP_EINVAL (-1)
#define RP_ESHAPE (-2)
#define RP_EALIGN (-3)
#define RP_EDRIVER (-4)
#define RP_EWORKSPACE (-5)

#define RP_MAX_POSITIVES 32   // include/rp_b200.h: most positive slots per position of a multi-positive batch

#define RP_CUDA_CHECK(expr)                  \
  do {                                       \
    cudaError_t _e = (expr);                 \
    if (_e != cudaSuccess) return (int)_e;   \
  } while (0)

#define RP_LAUNCH_CHECK()                    \
  do {                                       \
    cudaError_t _e = cudaGetLastError();     \
    if (_e != cudaSuccess) return (int)_e;   \
  } while (0)

namespace rp {

typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

PFN_encodeTiled get_encode_tiled();

// 2-D bf16 row-major tensor [rows, cols] (cols contiguous, row pitch `ld` elements); box = [box_rows, 64 cols] with
// SWIZZLE_128B (64 bf16 = 128 B inner extent).  Out-of-bounds elements are filled with zeros.
// Returns 0 on success, RP_E* otherwise.
int make_tmap_bf16(CUtensorMap* out, const void* base, uint64_t rows, uint64_t cols, uint64_t ld, uint32_t box_rows,
                   uint32_t box_cols = 64);

// 3-D view [n_seq][seq_len][cols] of the same kind of array (row b * seq_len + l of the 2-D array): box = [1, box_rows, 64 cols].
// Rows l >= seq_len of a box are OUT OF BOUNDS: loads fill them with zeros, stores drop them - a 128-row box never touches
// the next sequence (padded-sequence attention, L not a multiple of 128).
int make_tmap_bf16_seq(CUtensorMap* out, const void* base, uint64_t n_seq, uint64_t seq_len, uint64_t cols, uint64_t ld,
                       uint32_t box_rows, uint32_t box_cols = 64);

int sm_count();

}  // namespace rp
