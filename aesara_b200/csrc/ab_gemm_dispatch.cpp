// ab_gemm_dispatch.cpp — ab_gemm / ab_gemm_workspace_bytes entry points.
//
// float32: wgmma tensor-core tiles fed by TMA (ab_gemm_tc.cu) when
// the operands can be described by TMA tensor maps (unit stride along one dim,
// 16-byte aligned pitches); float64 and everything else: the CUDA-core tiled
// kernel (ab_gemm_simt.cu).  Reference: aesara/tensor/blas.py:518-869.
#include "ab_common.h"

namespace ab {
template <typename T>
int gemm_simt(long long M, long long N, long long K, double alpha, const void* A, long long a_rs,
              long long a_cs, const void* B, long long b_rs, long long b_cs, double beta, void* C,
              long long c_rs, long long c_cs, cudaStream_t st);

// returns AB_ERR_UNSUPPORTED (without touching last_error semantics) when the
// problem does not fit the tensor-core kernel's constraints
int gemm_tc_f32(int precision, long long M, long long N, long long K, float alpha,
                     const float* A, long long a_rs, long long a_cs, const float* B,
                     long long b_rs, long long b_cs, float beta, float* C, long long c_rs,
                     long long c_cs, void* workspace, size_t workspace_bytes, cudaStream_t st,
                     bool* handled);
size_t gemm_tc_workspace(int precision, long long M, long long N, long long K,
                              long long a_rs, long long a_cs, long long b_rs, long long b_cs);
}  // namespace ab

using namespace ab;

extern "C" int ab_gemm_workspace_bytes(int dtype, int precision, int64_t m, int64_t n, int64_t k,
                                       int64_t a_rs, int64_t a_cs, int64_t b_rs, int64_t b_cs,
                                       size_t* bytes) {
  if (!bytes) return fail(AB_ERR_INVALID, "null out pointer");
  *bytes = 0;
  if (dtype == AB_F32) *bytes = gemm_tc_workspace(precision, m, n, k, a_rs, a_cs, b_rs, b_cs);
  return AB_OK;
}

extern "C" int ab_gemm(int dtype, int precision, int64_t m, int64_t n, int64_t k, double alpha,
                       const void* A, int64_t a_rs, int64_t a_cs, const void* B, int64_t b_rs,
                       int64_t b_cs, double beta, void* C, int64_t c_rs, int64_t c_cs,
                       void* workspace, size_t workspace_bytes, void* stream) {
  if (m < 0 || n < 0 || k < 0) return fail(AB_ERR_SHAPE, "negative dimension in gemm");
  cudaStream_t st = as_stream(stream);
  if (dtype == AB_F64)
    return gemm_simt<double>(m, n, k, alpha, A, a_rs, a_cs, B, b_rs, b_cs, beta, C, c_rs, c_cs, st);
  if (dtype != AB_F32)
    return fail(AB_ERR_UNSUPPORTED, "Gemm supports float32/float64 only (blas.py:613-629)");
  bool handled = false;
  int rc = gemm_tc_f32(precision, m, n, k, (float)alpha, static_cast<const float*>(A), a_rs,
                            a_cs, static_cast<const float*>(B), b_rs, b_cs, (float)beta,
                            static_cast<float*>(C), c_rs, c_cs, workspace, workspace_bytes, st,
                            &handled);
  if (handled) return rc;
  return gemm_simt<float>(m, n, k, alpha, A, a_rs, a_cs, B, b_rs, b_cs, beta, C, c_rs, c_cs, st);
}
