// ab_blas_l2.cu — Gemv and Ger: the HBM-bound members of the BLAS family.
//
// Reference: aesara/tensor/blas.py:231 (Gemv.perform :279-318), blas_c.py:369-577
// (gemv_c_code: sgemv_/dgemv_ "N"/"T" chosen by the contiguity of A, beta==0
// means y is uninitialised and must not be read, :418-430) and blas.py:330 /
// blas_c.py:45-357 (Ger).  A matrix-vector product moves m*n*s bytes for 2*m*n
// flops, so these are streaming kernels (coalesced 128-bit loads, fp32/fp64 FMA),
// not tensor-core work.
//
//   row pattern   (a_cs == 1): one warp per row, lanes stride the row with
//                 16-byte loads, x staged in shared memory, shuffle-tree sum;
//   column pattern (a_rs == 1): thread per 16-byte group of outputs, the
//                 reduction (over columns of A) split across blockIdx.y with
//                 partials in `workspace`, summed by a second small kernel;
//   generic       any other strides: thread per output, scalar loads.
#include <algorithm>

#include "ab_common.h"

using namespace ab;

namespace {

constexpr int kThreads = 256;

template <typename T> struct Vec;
template <> struct Vec<float> { typedef float4 type; static constexpr int N = 4; };
template <> struct Vec<double> { typedef double2 type; static constexpr int N = 2; };

template <typename T>
__device__ __forceinline__ T warp_sum(T v) {
#pragma unroll
  for (int m = 16; m >= 1; m >>= 1) v += __shfl_xor_sync(0xffffffffu, v, m);
  return v;
}

// ---- row pattern ----------------------------------------------------------------
template <typename T, bool VEC>
__global__ void __launch_bounds__(kThreads)
gemv_rows_kernel(long long m, long long n, T alpha, const T* __restrict__ A, long long a_rs,
                 const T* __restrict__ x, long long x_s, T beta, T* __restrict__ y,
                 long long y_s, int x_in_smem) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  T* xs = reinterpret_cast<T*>(smem_raw);
  if (x_in_smem) {
    for (long long j = threadIdx.x; j < n; j += kThreads) xs[j] = x[j * x_s];
    __syncthreads();
  }
  const int lane = threadIdx.x & 31;
  const long long warp = (long long)blockIdx.x * (kThreads / 32) + (threadIdx.x >> 5);
  const long long nwarps = (long long)gridDim.x * (kThreads / 32);
  typedef typename Vec<T>::type V;
  constexpr int NV = Vec<T>::N;
  for (long long i = warp; i < m; i += nwarps) {
    const T* row = A + i * a_rs;
    T acc0 = 0, acc1 = 0;
    if (VEC) {
      const V* rv = reinterpret_cast<const V*>(row);
      const long long nvec = n / NV;
      long long v = lane;
      for (; v + 32 < nvec; v += 64) {
        const V a0 = __ldcs(rv + v);
        const V a1 = __ldcs(rv + v + 32);
        const T* e0 = reinterpret_cast<const T*>(&a0);
        const T* e1 = reinterpret_cast<const T*>(&a1);
#pragma unroll
        for (int e = 0; e < NV; ++e) {
          const long long j0 = v * NV + e, j1 = (v + 32) * NV + e;
          acc0 += e0[e] * (x_in_smem ? xs[j0] : __ldg(x + j0 * x_s));
          acc1 += e1[e] * (x_in_smem ? xs[j1] : __ldg(x + j1 * x_s));
        }
      }
      for (; v < nvec; v += 32) {
        const V a0 = __ldcs(rv + v);
        const T* e0 = reinterpret_cast<const T*>(&a0);
#pragma unroll
        for (int e = 0; e < NV; ++e) {
          const long long j0 = v * NV + e;
          acc0 += e0[e] * (x_in_smem ? xs[j0] : __ldg(x + j0 * x_s));
        }
      }
    } else {
      for (long long j = lane; j < n; j += 32)
        acc0 += __ldcs(row + j) * (x_in_smem ? xs[j] : __ldg(x + j * x_s));
    }
    T acc = warp_sum(acc0 + acc1);
    if (lane == 0) {
      T r = alpha * acc;
      if (beta != T(0)) r += beta * y[i * y_s];
      y[i * y_s] = r;
    }
  }
}

// ---- column pattern --------------------------------------------------------------
// A[i + j*a_cs]; thread (tx) owns NV consecutive outputs i, blockDim.y rows of
// threads and gridDim.y CTAs split the j range; partial[s][i] in workspace.
template <typename T, bool VEC>
__global__ void __launch_bounds__(kThreads)
gemv_cols_kernel(long long m, long long n, const T* __restrict__ A, long long a_cs,
                 const T* __restrict__ x, long long x_s, T* __restrict__ partial,
                 long long slice) {
  typedef typename Vec<T>::type V;
  constexpr int NV = VEC ? Vec<T>::N : 1;
  const long long i0 = ((long long)blockIdx.x * blockDim.x + threadIdx.x) * NV;
  const long long s = blockIdx.y;
  const long long j_begin = s * slice;
  const long long j_end = min(j_begin + slice, n);
  T acc[4][NV];
#pragma unroll
  for (int u = 0; u < 4; ++u)
#pragma unroll
    for (int e = 0; e < NV; ++e) acc[u][e] = 0;
  if (i0 < m) {
    const T* col = A + i0;
    long long j = j_begin + threadIdx.y;
    const long long step = blockDim.y;
    for (; j + 3 * step < j_end; j += 4 * step) {
      T xv[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) xv[u] = __ldg(x + (j + u * step) * x_s);
      if (VEC) {
        V a[4];
#pragma unroll
        for (int u = 0; u < 4; ++u) a[u] = __ldcs(reinterpret_cast<const V*>(col + (j + u * step) * a_cs));
#pragma unroll
        for (int u = 0; u < 4; ++u) {
          const T* e0 = reinterpret_cast<const T*>(&a[u]);
#pragma unroll
          for (int e = 0; e < NV; ++e) acc[u][e] += e0[e] * xv[u];
        }
      } else {
#pragma unroll
        for (int u = 0; u < 4; ++u) acc[u][0] += __ldcs(col + (j + u * step) * a_cs) * xv[u];
      }
    }
    for (; j < j_end; j += step) {
      const T xv = __ldg(x + j * x_s);
      if (VEC) {
        const V a = __ldcs(reinterpret_cast<const V*>(col + j * a_cs));
        const T* e0 = reinterpret_cast<const T*>(&a);
#pragma unroll
        for (int e = 0; e < NV; ++e) acc[0][e] += e0[e] * xv;
      } else {
        acc[0][0] += __ldcs(col + j * a_cs) * xv;
      }
    }
  }
  // combine the blockDim.y partial rows through shared memory
  extern __shared__ __align__(16) unsigned char smem_raw[];
  T* sm = reinterpret_cast<T*>(smem_raw);  // [blockDim.y][blockDim.x * NV]
  const int width = blockDim.x * NV;
#pragma unroll
  for (int e = 0; e < NV; ++e)
    sm[threadIdx.y * width + threadIdx.x * NV + e] =
        (acc[0][e] + acc[1][e]) + (acc[2][e] + acc[3][e]);
  __syncthreads();
  if (threadIdx.y == 0 && i0 < m) {
#pragma unroll
    for (int e = 0; e < NV; ++e) {
      T t = 0;
      for (int r = 0; r < (int)blockDim.y; ++r) t += sm[r * width + threadIdx.x * NV + e];
      if (i0 + e < m) partial[s * m + i0 + e] = t;
    }
  }
}

template <typename T>
__global__ void __launch_bounds__(kThreads)
gemv_finish_kernel(long long m, long long split, const T* __restrict__ partial, T alpha, T beta,
                   T* __restrict__ y, long long y_s) {
  const long long i = (long long)blockIdx.x * kThreads + threadIdx.x;
  if (i >= m) return;
  T acc = 0;
  for (long long s = 0; s < split; ++s) acc += partial[s * m + i];
  T r = alpha * acc;
  if (beta != T(0)) r += beta * y[i * y_s];
  y[i * y_s] = r;
}

// ---- generic ----------------------------------------------------------------------
template <typename T>
__global__ void __launch_bounds__(kThreads)
gemv_generic_kernel(long long m, long long n, T alpha, const T* __restrict__ A, long long a_rs,
                    long long a_cs, const T* __restrict__ x, long long x_s, T beta,
                    T* __restrict__ y, long long y_s) {
  const long long i = (long long)blockIdx.x * kThreads + threadIdx.x;
  if (i >= m) return;
  T acc = 0;
  for (long long j = 0; j < n; ++j) acc += A[i * a_rs + j * a_cs] * x[j * x_s];
  T r = alpha * acc;
  if (beta != T(0)) r += beta * y[i * y_s];
  y[i * y_s] = r;
}

// y <- beta*y when the product is empty (n == 0)
template <typename T>
__global__ void scale_kernel(long long m, T beta, T* y, long long y_s) {
  const long long i = (long long)blockIdx.x * kThreads + threadIdx.x;
  if (i < m) y[i * y_s] = beta == T(0) ? T(0) : beta * y[i * y_s];
}

// ---- Ger ---------------------------------------------------------------------------
template <typename T>
__global__ void __launch_bounds__(kThreads)
ger_kernel(long long m, long long n, T alpha, const T* __restrict__ x, long long x_s,
           const T* __restrict__ y, long long y_s, T* __restrict__ A, long long a_rs,
           long long a_cs) {
  // inner index j runs along the smaller-stride dim of A (chosen by the host)
  const long long j = (long long)blockIdx.x * kThreads + threadIdx.x;
  if (j >= n) return;
  const T yj = alpha * y[j * y_s];
  for (long long i = blockIdx.y; i < m; i += gridDim.y) {
    T* a = A + i * a_rs + j * a_cs;
    *a = *a + x[i * x_s] * yj;
  }
}

int sm_count() {
  static int n = 0;
  if (!n) {
    int dev = 0;
    cudaGetDevice(&dev);
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0)
      n = 132;
  }
  return n;
}

struct ColsPlan { int bx, by; long long gx, split, slice; bool vec; };

template <typename T>
ColsPlan cols_plan(long long m, long long n, const void* A, long long a_cs) {
  ColsPlan p;
  constexpr int NV = Vec<T>::N;
  p.vec = (m % NV == 0) && (a_cs % NV == 0) && (reinterpret_cast<uintptr_t>(A) % 16 == 0);
  const long long groups = p.vec ? m / NV : m;
  int bx = 32;
  while (bx < kThreads && bx < groups) bx <<= 1;
  p.bx = bx;
  p.by = kThreads / bx;
  p.gx = (groups + bx - 1) / bx;
  const long long target = (long long)sm_count() * 8;
  long long split = std::max<long long>(1, target / p.gx);
  split = std::min<long long>(split, std::max<long long>(1, n / (4LL * p.by)));
  split = std::min<long long>(split, 65535);
  p.slice = (n + split - 1) / split;
  p.split = p.slice > 0 ? (n + p.slice - 1) / p.slice : 1;
  return p;
}

template <typename T>
int gemv_impl(long long m, long long n, double alpha_d, const void* Av, long long a_rs,
              long long a_cs, const void* xv, long long x_s, double beta_d, void* yv,
              long long y_s, void* workspace, size_t workspace_bytes, cudaStream_t st) {
  const T* A = static_cast<const T*>(Av);
  const T* x = static_cast<const T*>(xv);
  T* y = static_cast<T*>(yv);
  const T alpha = (T)alpha_d, beta = (T)beta_d;
  if (m == 0) return AB_OK;
  if (n == 0) {
    scale_kernel<T><<<(unsigned)((m + kThreads - 1) / kThreads), kThreads, 0, st>>>(m, beta, y, y_s);
    g_launches++;
    AB_CUDA(cudaGetLastError());
    return AB_OK;
  }
  constexpr int NV = Vec<T>::N;
  if (a_cs == 1 || m == 1) {
    const long long rs = (m == 1) ? 0 : a_rs;
    if (a_cs != 1) {  // a single strided row: treat through the generic kernel
      gemv_generic_kernel<T><<<1, kThreads, 0, st>>>(m, n, alpha, A, rs, a_cs, x, x_s, beta, y, y_s);
      g_launches++;
      AB_CUDA(cudaGetLastError());
      return AB_OK;
    }
    const bool vec = (n % NV == 0) && (rs % NV == 0) && (reinterpret_cast<uintptr_t>(A) % 16 == 0);
    const size_t xbytes = (size_t)n * sizeof(T);
    const int x_in_smem = xbytes <= 40 * 1024;
    const long long warps_needed = m;
    long long blocks = (warps_needed + (kThreads / 32) - 1) / (kThreads / 32);
    blocks = std::max<long long>(1, std::min<long long>(blocks, (long long)sm_count() * 8));
    const size_t smem = x_in_smem ? xbytes : 0;
    if (vec)
      gemv_rows_kernel<T, true><<<(unsigned)blocks, kThreads, smem, st>>>(m, n, alpha, A, rs, x, x_s, beta, y, y_s, x_in_smem);
    else
      gemv_rows_kernel<T, false><<<(unsigned)blocks, kThreads, smem, st>>>(m, n, alpha, A, rs, x, x_s, beta, y, y_s, x_in_smem);
    g_launches++;
    AB_CUDA(cudaGetLastError());
    return AB_OK;
  }
  if (a_rs == 1) {
    ColsPlan p = cols_plan<T>(m, n, A, a_cs);
    const size_t need = (size_t)p.split * (size_t)m * sizeof(T);
    if (!workspace || workspace_bytes < need)
      return fail(AB_ERR_INVALID, "Gemv workspace too small: need %zu bytes, have %zu", need,
                  workspace_bytes);
    T* partial = static_cast<T*>(workspace);
    dim3 grid((unsigned)p.gx, (unsigned)p.split), block(p.bx, p.by);
    const size_t smem = (size_t)p.by * p.bx * (p.vec ? NV : 1) * sizeof(T);
    if (p.vec)
      gemv_cols_kernel<T, true><<<grid, block, smem, st>>>(m, n, A, a_cs, x, x_s, partial, p.slice);
    else
      gemv_cols_kernel<T, false><<<grid, block, smem, st>>>(m, n, A, a_cs, x, x_s, partial, p.slice);
    g_launches++;
    AB_CUDA(cudaGetLastError());
    gemv_finish_kernel<T><<<(unsigned)((m + kThreads - 1) / kThreads), kThreads, 0, st>>>(m, p.split, partial, alpha, beta, y, y_s);
    g_launches++;
    AB_CUDA(cudaGetLastError());
    return AB_OK;
  }
  gemv_generic_kernel<T><<<(unsigned)((m + kThreads - 1) / kThreads), kThreads, 0, st>>>(m, n, alpha, A, a_rs, a_cs, x, x_s, beta, y, y_s);
  g_launches++;
  AB_CUDA(cudaGetLastError());
  return AB_OK;
}

template <typename T>
int ger_impl(long long m, long long n, double alpha, const void* x, long long x_s, const void* y,
             long long y_s, void* A, long long a_rs, long long a_cs, cudaStream_t st) {
  if (m == 0 || n == 0) return AB_OK;
  // make the thread index run along the dim of A with the smaller |stride|
  const bool swap = std::llabs(a_rs) < std::llabs(a_cs);
  const long long mm = swap ? n : m, nn = swap ? m : n;
  const void* xx = swap ? y : x;
  const void* yy = swap ? x : y;
  const long long xs = swap ? y_s : x_s, ys = swap ? x_s : y_s;
  const long long rs = swap ? a_cs : a_rs, cs = swap ? a_rs : a_cs;
  dim3 grid((unsigned)((nn + kThreads - 1) / kThreads),
            (unsigned)std::max<long long>(1, std::min<long long>(mm, 4096)));
  ger_kernel<T><<<grid, kThreads, 0, st>>>(mm, nn, (T)alpha, static_cast<const T*>(xx), xs,
                                           static_cast<const T*>(yy), ys, static_cast<T*>(A), rs, cs);
  g_launches++;
  AB_CUDA(cudaGetLastError());
  return AB_OK;
}

}  // namespace

extern "C" int ab_gemv_workspace_bytes(int dtype, int64_t m, int64_t n, int64_t a_rs,
                                       int64_t a_cs, size_t* bytes) {
  if (!bytes) return fail(AB_ERR_INVALID, "null out pointer");
  *bytes = 0;
  if (m > 0 && n > 0 && a_cs != 1 && a_rs == 1 && m != 1) {
    // worst case over alignment-dependent plans
    const size_t es = dtype == AB_F64 ? 8 : 4;
    const long long target = (long long)sm_count() * 8;
    *bytes = (size_t)std::min<long long>(65535, std::max<long long>(1, target)) * (size_t)m * es;
  }
  return AB_OK;
}

extern "C" int ab_gemv(int dtype, int64_t m, int64_t n, double alpha, const void* A, int64_t a_rs,
                       int64_t a_cs, const void* x, int64_t x_s, double beta, void* y,
                       int64_t y_s, void* workspace, size_t workspace_bytes, void* stream) {
  if (m < 0 || n < 0) return fail(AB_ERR_SHAPE, "negative dimension in gemv");
  if (dtype == AB_F32)
    return gemv_impl<float>(m, n, alpha, A, a_rs, a_cs, x, x_s, beta, y, y_s, workspace,
                            workspace_bytes, as_stream(stream));
  if (dtype == AB_F64)
    return gemv_impl<double>(m, n, alpha, A, a_rs, a_cs, x, x_s, beta, y, y_s, workspace,
                             workspace_bytes, as_stream(stream));
  return fail(AB_ERR_UNSUPPORTED, "Gemv supports float32/float64 only (blas.py:613-629)");
}

extern "C" int ab_ger(int dtype, int64_t m, int64_t n, double alpha, const void* x, int64_t x_s,
                      const void* y, int64_t y_s, void* A, int64_t a_rs, int64_t a_cs,
                      void* stream) {
  if (m < 0 || n < 0) return fail(AB_ERR_SHAPE, "negative dimension in ger");
  if (dtype == AB_F32) return ger_impl<float>(m, n, alpha, x, x_s, y, y_s, A, a_rs, a_cs, as_stream(stream));
  if (dtype == AB_F64) return ger_impl<double>(m, n, alpha, x, x_s, y, y_s, A, a_rs, a_cs, as_stream(stream));
  return fail(AB_ERR_UNSUPPORTED, "Ger supports float32/float64 only");
}
