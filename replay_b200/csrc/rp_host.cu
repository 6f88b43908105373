// rp_host.cu - tensor-map construction through the driver entry point (no link-time libcuda dependency), device info.
#include <mutex>

#include "rp_host.h"

namespace rp {

PFN_encodeTiled get_encode_tiled() {
  static PFN_encodeTiled fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<PFN_encodeTiled>(p);
  });
  return fn;
}

int make_tmap_bf16(CUtensorMap* out, const void* base, uint64_t rows, uint64_t cols, uint64_t ld, uint32_t box_rows,
                   uint32_t box_cols) {
  PFN_encodeTiled enc = get_encode_tiled();
  if (!enc) return RP_EDRIVER;
  if ((reinterpret_cast<uintptr_t>(base) & 15) != 0 || ((ld * 2) & 15) != 0) return RP_EALIGN;
  if (box_rows == 0 || box_rows > 256 || box_cols * 2 > 128) return RP_ESHAPE;
  cuuint64_t gdim[2] = {cols, rows};
  cuuint64_t gstride[1] = {ld * 2};
  cuuint32_t box[2] = {box_cols, box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = enc(out, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(base), gdim, gstride, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS ? RP_OK : RP_EDRIVER;
}

int make_tmap_bf16_seq(CUtensorMap* out, const void* base, uint64_t n_seq, uint64_t seq_len, uint64_t cols, uint64_t ld,
                       uint32_t box_rows, uint32_t box_cols) {
  PFN_encodeTiled enc = get_encode_tiled();
  if (!enc) return RP_EDRIVER;
  if ((reinterpret_cast<uintptr_t>(base) & 15) != 0 || ((ld * 2) & 15) != 0) return RP_EALIGN;
  if (box_rows == 0 || box_rows > 256 || box_cols * 2 > 128) return RP_ESHAPE;
  cuuint64_t gdim[3] = {cols, seq_len, n_seq};
  cuuint64_t gstride[2] = {ld * 2, seq_len * ld * 2};
  cuuint32_t box[3] = {box_cols, box_rows, 1};
  cuuint32_t estr[3] = {1, 1, 1};
  CUresult r = enc(out, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, const_cast<void*>(base), gdim, gstride, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS ? RP_OK : RP_EDRIVER;
}

int sm_count() {
  static int n = 0;
  if (n == 0) {
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
    if (n <= 0) n = 132;   // the query failed: assume an H100 SXM
  }
  return n;
}

}  // namespace rp
