// rp_gemm_desc.h - flat C view of the GEMM parameter block shared by the C-ABI entry point (rp_gemm.cu) and the kernels
// host code that sequences GEMMs internally (the CE, sampled and SCE heads).  Field-for-field the public `rp_gemm_desc` of
// include/rp_b200.h (tests/test_api_cpu.py checks the ctypes mirror against the header).
#pragma once
#include <stdint.h>
#include <string.h>

struct rp_gemm_desc {
  const void* A; long long a_rows, a_cols, lda; int a_mn;
  const void* B; long long b_rows, b_cols, ldb; int b_mn;
  int M, N, K, batch, inner;
  int a_r0, a_ro, a_ri, a_c0, a_co, a_ci;
  int b_r0, b_ro, b_ri, b_c0, b_co, b_ci;
  void* C; long long ldc, c_off0, c_oo, c_oi; int out_mode;
  float alpha; const float* bias; int act;
  const void* residual; const uint8_t* rowmask; long long rowmask_off0, rowmask_oo;
  float drop_p; unsigned long long seed, drop_offset; const unsigned long long* seed_ptr;
  int split_k;
  const void* gate; float gate_scale;
  void* C2; int gate_mode; float post_drop_p; unsigned long long post_drop_offset;
  long long c_split_stride;
  const float* row_exp2_offset;
  const int32_t* m_limit_dev; int m_limit_base;
  const int32_t* k_limit_dev; int k_limit_base;
};

// a plain single GEMM: every field zero except batch = inner = 1, alpha = 1, split_k = 1
inline rp_gemm_desc rp_gemm_default() {
  rp_gemm_desc g;
  memset(&g, 0, sizeof(g));
  g.batch = 1; g.inner = 1; g.alpha = 1.f; g.split_k = 1;
  return g;
}

extern "C" int rp_gemm(const rp_gemm_desc* g, void* stream);
