// ab_gemm_simt.cu — C <- beta*C + alpha*A@B on the FP32/FP64 CUDA-core pipes.
//
// This is the float64 path of Gemm/Dot22 (aesara/tensor/blas.py:872/:1659 accept
// float32 and float64 only, :613-629; the tensor-core path is float32 only) and the path for
// problems too small or too oddly strided for the TMA-fed tensor-core kernel in
// ab_gemm_tc.cu.  Classic shared-memory tiling: 64x64 output tile per CTA,
// K stepped by 16, each of the 256 threads owns a 4x4 register micro-tile.
// Arbitrary element strides for A, B, C (the eight transposed/strided cases of
// blas.py:765-776 need no copies here).
#include <algorithm>

#include "ab_common.h"

using namespace ab;

namespace {

constexpr int BM = 64, BN = 64, BK = 16, TM = 4, TN = 4;

template <typename T>
__global__ void __launch_bounds__(256)
gemm_simt_kernel(long long M, long long N, long long K, T alpha, const T* __restrict__ A,
                 long long a_rs, long long a_cs, const T* __restrict__ B, long long b_rs,
                 long long b_cs, T beta, T* __restrict__ C, long long c_rs, long long c_cs) {
  __shared__ T As[BK][BM + 1];
  __shared__ T Bs[BK][BN + 1];
  const int tid = threadIdx.x;
  const int tx = tid % 16, ty = tid / 16;
  const long long m0 = (long long)blockIdx.y * BM, n0 = (long long)blockIdx.x * BN;
  T acc[TM][TN];
#pragma unroll
  for (int i = 0; i < TM; ++i)
#pragma unroll
    for (int j = 0; j < TN; ++j) acc[i][j] = 0;

  // loader mapping: make the thread index run along the unit-stride dim when there is one
  const bool a_kfast = (a_cs == 1) || (a_rs != 1 && std::abs((double)a_cs) < std::abs((double)a_rs));
  const bool b_nfast = (b_cs == 1) || (b_rs != 1 && std::abs((double)b_cs) < std::abs((double)b_rs));

  for (long long k0 = 0; k0 < K; k0 += BK) {
#pragma unroll
    for (int r = 0; r < (BM * BK) / 256; ++r) {
      const int e = tid + r * 256;
      int mm, kk;
      if (a_kfast) { kk = e % BK; mm = e / BK; } else { mm = e % BM; kk = e / BM; }
      const long long gm = m0 + mm, gk = k0 + kk;
      As[kk][mm] = (gm < M && gk < K) ? A[gm * a_rs + gk * a_cs] : T(0);
    }
#pragma unroll
    for (int r = 0; r < (BN * BK) / 256; ++r) {
      const int e = tid + r * 256;
      int nn, kk;
      if (b_nfast) { nn = e % BN; kk = e / BN; } else { kk = e % BK; nn = e / BK; }
      const long long gn = n0 + nn, gk = k0 + kk;
      Bs[kk][nn] = (gn < N && gk < K) ? B[gk * b_rs + gn * b_cs] : T(0);
    }
    __syncthreads();
#pragma unroll
    for (int kk = 0; kk < BK; ++kk) {
      T a[TM], b[TN];
#pragma unroll
      for (int i = 0; i < TM; ++i) a[i] = As[kk][ty * TM + i];
#pragma unroll
      for (int j = 0; j < TN; ++j) b[j] = Bs[kk][tx * TN + j];
#pragma unroll
      for (int i = 0; i < TM; ++i)
#pragma unroll
        for (int j = 0; j < TN; ++j) acc[i][j] += a[i] * b[j];
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < TM; ++i) {
    const long long gm = m0 + ty * TM + i;
    if (gm >= M) continue;
#pragma unroll
    for (int j = 0; j < TN; ++j) {
      const long long gn = n0 + tx * TN + j;
      if (gn >= N) continue;
      T* c = C + gm * c_rs + gn * c_cs;
      T r = alpha * acc[i][j];
      if (beta != T(0)) r += beta * (*c);
      *c = r;
    }
  }
}

template <typename T>
__global__ void scale2d_kernel(long long M, long long N, T beta, T* C, long long c_rs, long long c_cs) {
  const long long j = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long i = blockIdx.y;
  if (j < N && i < M) {
    T* c = C + i * c_rs + j * c_cs;
    *c = beta == T(0) ? T(0) : beta * (*c);
  }
}

}  // namespace

namespace ab {

template <typename T>
int gemm_simt(long long M, long long N, long long K, double alpha, const void* A, long long a_rs,
              long long a_cs, const void* B, long long b_rs, long long b_cs, double beta, void* C,
              long long c_rs, long long c_cs, cudaStream_t st) {
  if (M == 0 || N == 0) return AB_OK;
  if (M > 65535LL * BM) return fail(AB_ERR_UNSUPPORTED, "gemm: M too large for the SIMT path");
  if (K == 0) {
    dim3 grid((unsigned)((N + 255) / 256), (unsigned)M);
    scale2d_kernel<T><<<grid, 256, 0, st>>>(M, N, (T)beta, static_cast<T*>(C), c_rs, c_cs);
    g_launches++;
    AB_CUDA(cudaGetLastError());
    return AB_OK;
  }
  dim3 grid((unsigned)((N + BN - 1) / BN), (unsigned)((M + BM - 1) / BM));
  gemm_simt_kernel<T><<<grid, 256, 0, st>>>(M, N, K, (T)alpha, static_cast<const T*>(A), a_rs, a_cs,
                                           static_cast<const T*>(B), b_rs, b_cs, (T)beta,
                                           static_cast<T*>(C), c_rs, c_cs);
  g_launches++;
  AB_CUDA(cudaGetLastError());
  return AB_OK;
}

template int gemm_simt<float>(long long, long long, long long, double, const void*, long long,
                              long long, const void*, long long, long long, double, void*,
                              long long, long long, cudaStream_t);
template int gemm_simt<double>(long long, long long, long long, double, const void*, long long,
                               long long, const void*, long long, long long, double, void*,
                               long long, long long, cudaStream_t);

}  // namespace ab
