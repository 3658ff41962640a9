// ab_linalg.cu — Cholesky factorisation and triangular solves (aesara/tensor/slinalg.py:
// Cholesky, SolveTriangular, CholeskySolve, Solve(assume_a="pos")), float32 and float64.
//
// Both run blocked with NB x NB diagonal blocks, the whole loop inside one C-ABI call:
//   ab_cholesky  right-looking: per panel, one CTA factors the diagonal block in shared
//                memory (potrf_diag_kernel), the panel below it is solved against that block
//                (trsm_diag_kernel on the transposed panel), and the trailing matrix takes the
//                rank-NB update C -= L21 L21^T on the project's GEMMs (rank_update).
//   ab_trsm      the same for op(A) X = B: every (lower, trans) case is a forward substitution
//                with a lower-triangular T read through strides -- trans swaps A's strides, an
//                upper T is reversed by negative strides (rows and columns of T, rows of X) --
//                so no operand is copied.  Per block of NB rows: trsm_diag_kernel solves the
//                block, then the rows below take X_rest -= T_rest,blk X_blk.  A vector right-hand
//                side takes trsv_diag_kernel / trsv_update_kernel instead: a matrix-vector
//                update is bandwidth-bound, and a GEMM with N = 1 would waste its tile.
//
// Float32 updates always use the fp32-faithful 3xTF32 product, whatever product policy the
// caller runs its Dot/Gemm nodes with: the error of a factorisation grows with the condition
// number of the matrix, so a bf16 or single-TF32 update (2^-8 / 2^-11 relative operand error)
// makes the factor of a matrix with condition 1e4 useless.  The tensor-core GEMM reads its
// operands from packed planes but stores C directly with 128-bit stores, which needs a
// row-contiguous C with 16-byte aligned rows; where C's pitch does not allow that (float32
// with n % 4 != 0) the update runs on the CUDA-core kernel.  ab_linalg_update_count tells the
// two apart.
//
// Errors cannot be raised from a kernel.  They are written to a device status word that the
// caller owns (initialised by ab_linalg_status_reset): the smallest of kind << 56 | index wins,
// so a non-finite input (kind 1, the reference's ValueError, checked first) beats a pivot
// failure (kind 2, not positive definite) or a zero diagonal (kind 3, singular).  The diagonal
// kernels of later panels read the word and exit, so the panel loop never waits on the host;
// ab_linalg_status_check reads it once (one synchronisation) and maps it to a status code.
#include <algorithm>
#include <cmath>

#include "ab_common.h"

using namespace ab;

namespace ab {
template <typename T>
int gemm_simt(long long M, long long N, long long K, double alpha, const void* A, long long a_rs,
              long long a_cs, const void* B, long long b_rs, long long b_cs, double beta, void* C,
              long long c_rs, long long c_cs, cudaStream_t st);
int gemm_tc_f32(int precision, long long M, long long N, long long K, float alpha, const float* A,
                long long a_rs, long long a_cs, const float* B, long long b_rs, long long b_cs,
                float beta, float* C, long long c_rs, long long c_cs, void* workspace,
                size_t workspace_bytes, cudaStream_t st, bool* handled);
size_t gemm_tc_workspace(int precision, long long M, long long N, long long K, long long a_rs,
                         long long a_cs, long long b_rs, long long b_cs);
}  // namespace ab

namespace {

// Diagonal block size.  The rank-NB updates carry 2*NB flops per element of C they read and
// write, so a larger NB moves them away from the bandwidth bound; the diagonal factorisation
// (one CTA) and the block solves grow with NB^2 and run on few SMs.
constexpr int NB = 128;
constexpr int kFactorThreads = 512;
constexpr int kThreads = 256;
constexpr unsigned long long kOk = ~0ull;
enum { KIND_NONFINITE = 1, KIND_NOT_PD = 2, KIND_SINGULAR = 3 };

__device__ __forceinline__ unsigned long long code(int kind, int operand, long long index) {
  return ((unsigned long long)kind << 56) | ((unsigned long long)operand << 48) |
         ((unsigned long long)index & ((1ull << 48) - 1));
}

// columns of the block solve a CTA takes, one per thread (float / double: shared memory)
template <typename T> struct SolveCols { static constexpr int N = 128; };
template <> struct SolveCols<double> { static constexpr int N = 64; };

std::atomic<uint64_t> g_updates[2];

int sm_count() {
  static int n = 0;
  if (!n) {
    int dev = 0;
    cudaGetDevice(&dev);
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) n = 132;
  }
  return n;
}

unsigned grid_for(long long work) {
  return (unsigned)std::max<long long>(1, std::min<long long>((work + kThreads - 1) / kThreads, (long long)sm_count() * 16));
}

// ---------------------------------------------------------------- checks and copies
template <typename T>
__global__ void __launch_bounds__(kThreads)
check_finite_kernel(const T* __restrict__ a, long long rows, long long cols, long long rs, long long cs,
                    int operand, unsigned long long* status) {
  const long long total = rows * cols;
  for (long long e = (long long)blockIdx.x * kThreads + threadIdx.x; e < total; e += (long long)gridDim.x * kThreads) {
    const long long r = e / cols, c = e - r * cols;
    if (!isfinite(a[r * rs + c * cs])) atomicMin(status, code(KIND_NONFINITE, operand, e));
  }
}

template <typename T>
__global__ void __launch_bounds__(kThreads)
zero_diagonal_kernel(const T* __restrict__ a, long long n, long long ds, unsigned long long* status) {
  for (long long i = (long long)blockIdx.x * kThreads + threadIdx.x; i < n; i += (long long)gridDim.x * kThreads)
    if (a[i * ds] == T(0)) atomicMin(status, code(KIND_SINGULAR, 0, i));
}

// out (C-contiguous rows x cols) <- the triangle of a that is kept, 0 elsewhere: keep = -1
// r >= c (lower), 1 r <= c (upper), 0 everything.  a == nullptr: only the zeros are written.
template <typename T>
__global__ void __launch_bounds__(kThreads)
copy_kernel(const T* __restrict__ a, long long rs, long long cs, T* __restrict__ out, long long rows,
            long long cols, int keep) {
  const long long total = rows * cols;
  for (long long e = (long long)blockIdx.x * kThreads + threadIdx.x; e < total; e += (long long)gridDim.x * kThreads) {
    const long long r = e / cols, c = e - r * cols;
    const bool in = keep == 0 || (keep < 0 ? r >= c : r <= c);
    if (in) {
      if (a) out[e] = a[r * rs + c * cs];
    } else {
      out[e] = T(0);
    }
  }
}

// on_error="nan": the whole factor is NaN when a pivot failed
template <typename T>
__global__ void __launch_bounds__(kThreads)
nan_fill_kernel(T* __restrict__ out, long long total, const unsigned long long* status) {
  if ((*status >> 56) != KIND_NOT_PD) return;
  for (long long e = (long long)blockIdx.x * kThreads + threadIdx.x; e < total; e += (long long)gridDim.x * kThreads)
    out[e] = T(NAN);
}

// ---------------------------------------------------------------- diagonal blocks
// Factor the b x b diagonal block W[k0.., k0..] (lower triangle read and written, element
// strides wr, wc) in shared memory, unblocked right-looking like LAPACK potf2: a pivot that is
// not > 0 (NaN included) stops the factorisation with index k0 + j.
template <typename T>
__global__ void __launch_bounds__(kFactorThreads)
potrf_diag_kernel(T* __restrict__ W, long long wr, long long wc, long long k0, int b,
                  unsigned long long* status) {
  if (*status != kOk) return;
  extern __shared__ __align__(16) unsigned char smem_raw[];
  T* A = reinterpret_cast<T*>(smem_raw);
  constexpr int ld = NB + 1;
  __shared__ bool failed;
  T* base = W + k0 * (wr + wc);
  const bool c_fast = wc == 1;
  for (int e = threadIdx.x; e < b * b; e += kFactorThreads) {
    const int i = c_fast ? e / b : e % b, k = c_fast ? e % b : e / b;
    if (k <= i) A[i * ld + k] = base[i * wr + k * wc];
  }
  if (threadIdx.x == 0) failed = false;
  __syncthreads();
  for (int j = 0; j < b; ++j) {
    if (threadIdx.x == 0) {
      const T d = A[j * ld + j];
      if (!(d > T(0))) {
        failed = true;
        atomicMin(status, code(KIND_NOT_PD, 0, k0 + j));
      } else {
        A[j * ld + j] = sqrt(d);
      }
    }
    __syncthreads();
    if (failed) return;
    const T inv = T(1) / A[j * ld + j];
    for (int i = j + 1 + threadIdx.x; i < b; i += kFactorThreads) A[i * ld + j] *= inv;
    __syncthreads();
    const int m = b - j - 1;
    for (int e = threadIdx.x; e < m * m; e += kFactorThreads) {
      const int i = j + 1 + e / m, k = j + 1 + e % m;
      if (k <= i) A[i * ld + k] -= A[i * ld + j] * A[k * ld + j];
    }
    __syncthreads();
  }
  for (int e = threadIdx.x; e < b * b; e += kFactorThreads) {
    const int i = c_fast ? e / b : e % b, k = c_fast ? e % b : e / b;
    if (k <= i) base[i * wr + k * wc] = A[i * ld + k];
  }
}

// Solve L X = X for the b x ncols block X (element strides xr, xc) with the lower-triangular
// b x b block L (strides lr, lc; unit: its diagonal is taken as 1 and not read).  Each thread
// owns one column of X in shared memory and runs the substitution down it; L is read from
// shared memory by every thread at the same address (a broadcast).
template <typename T>
__global__ void __launch_bounds__(SolveCols<T>::N)
trsm_diag_kernel(const T* __restrict__ L, long long lr, long long lc, int b, int unit, T* __restrict__ X,
                 long long xr, long long xc, long long ncols, const unsigned long long* status) {
  if (*status != kOk) return;
  constexpr int CW = SolveCols<T>::N, ld = NB + 1;
  extern __shared__ __align__(16) unsigned char smem_raw[];
  T* Ls = reinterpret_cast<T*>(smem_raw);
  T* Xs = Ls + NB * ld;
  const long long c0 = (long long)blockIdx.x * CW;
  const int w = ncols - c0 < CW ? (int)(ncols - c0) : CW;
  const bool l_fast = llabs(lc) == 1;
  for (int e = threadIdx.x; e < b * b; e += CW) {
    const int i = l_fast ? e / b : e % b, k = l_fast ? e % b : e / b;
    if (k <= i) Ls[i * ld + k] = L[i * lr + k * lc];
  }
  T* Xb = X + c0 * xc;
  const bool x_cfast = llabs(xc) <= llabs(xr);  // threads along the contiguous dim of X
  for (int e = threadIdx.x; e < b * CW; e += CW) {
    const int i = x_cfast ? e / CW : e % b, c = x_cfast ? e % CW : e / b;
    if (c < w) Xs[i * CW + c] = Xb[i * xr + c * xc];
  }
  __syncthreads();
  const int c = threadIdx.x;
  if (c < w) {
    for (int i = 0; i < b; ++i) {
      // four partial sums: the dot product is a chain of dependent FMAs otherwise
      T s0 = Xs[i * CW + c], s1 = 0, s2 = 0, s3 = 0;
      const T* li = Ls + i * ld;
      int k = 0;
      for (; k + 4 <= i; k += 4) {
        s0 -= li[k] * Xs[k * CW + c];
        s1 -= li[k + 1] * Xs[(k + 1) * CW + c];
        s2 -= li[k + 2] * Xs[(k + 2) * CW + c];
        s3 -= li[k + 3] * Xs[(k + 3) * CW + c];
      }
      for (; k < i; ++k) s0 -= li[k] * Xs[k * CW + c];
      const T s = (s0 + s1) + (s2 + s3);
      Xs[i * CW + c] = unit ? s : s / li[i];
    }
  }
  __syncthreads();
  for (int e = threadIdx.x; e < b * CW; e += CW) {
    const int i = x_cfast ? e / CW : e % b, c2 = x_cfast ? e % CW : e / b;
    if (c2 < w) Xb[i * xr + c2 * xc] = Xs[i * CW + c2];
  }
}

// The vector case of trsm_diag_kernel: one CTA, threads over the rows of the block.
template <typename T>
__global__ void __launch_bounds__(NB)
trsv_diag_kernel(const T* __restrict__ L, long long lr, long long lc, int b, int unit, T* __restrict__ x,
                 long long xs, const unsigned long long* status) {
  if (*status != kOk) return;
  __shared__ T xv[NB];
  const int i = threadIdx.x;
  if (i < b) xv[i] = x[i * xs];
  __syncthreads();
  const T* li = L + (long long)i * lr;  // row i of the block; its diagonal is li[i * lc]
#pragma unroll 1
  for (int j = 0; j < b; ++j) {
    if (i == j && !unit) xv[j] /= li[j * lc];
    __syncthreads();
    if (i > j && i < b) xv[i] -= li[j * lc] * xv[j];
  }
  __syncthreads();
  if (i < b) x[i * xs] = xv[i];
}

// y[r] -= sum_k A[r][k] x[k] for r < m, k < b: a warp per row when A's rows are contiguous,
// else a thread per row (contiguous down the columns, or no unit stride at all).
template <typename T>
__global__ void __launch_bounds__(kThreads)
trsv_update_kernel(const T* __restrict__ A, long long ar, long long ac, long long m, int b,
                   const T* __restrict__ x, long long xs, T* __restrict__ y, long long ys,
                   const unsigned long long* status) {
  if (*status != kOk) return;
  __shared__ T xv[NB];
  for (int k = threadIdx.x; k < b; k += kThreads) xv[k] = x[k * xs];
  __syncthreads();
  if (llabs(ac) == 1) {
    const int lane = threadIdx.x & 31;
    for (long long r = ((long long)blockIdx.x * kThreads + threadIdx.x) >> 5; r < m;
         r += ((long long)gridDim.x * kThreads) >> 5) {
      T s = 0;
      for (int k = lane; k < b; k += 32) s += A[r * ar + k * ac] * xv[k];
#pragma unroll
      for (int o = 16; o; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
      if (lane == 0) y[r * ys] -= s;
    }
  } else {
    for (long long r = (long long)blockIdx.x * kThreads + threadIdx.x; r < m; r += (long long)gridDim.x * kThreads) {
      T s = 0;
      for (int k = 0; k < b; ++k) s += A[r * ar + k * ac] * xv[k];
      y[r * ys] -= s;
    }
  }
}

// ---------------------------------------------------------------- host side
template <typename T>
size_t diag_smem() { return (size_t)NB * (NB + 1) * sizeof(T); }
template <typename T>
size_t solve_smem() { return (size_t)NB * (NB + 1) * sizeof(T) + (size_t)NB * SolveCols<T>::N * sizeof(T); }

template <typename T>
int set_smem_limits() {
  static int rc = -1;
  if (rc < 0) {
    rc = cudaFuncSetAttribute(potrf_diag_kernel<T>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)diag_smem<T>()) ||
         cudaFuncSetAttribute(trsm_diag_kernel<T>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)solve_smem<T>());
  }
  if (rc) return fail(AB_ERR_CUDA, "cannot set the shared-memory limit of the linear-algebra kernels");
  return AB_OK;
}

// C[M,N] -= A[M,K] @ B[K,N]: the 3xTF32 tensor-core GEMM for float32 when C's rows are
// contiguous and 16-byte aligned and the problem is large enough for its tiles, else the
// CUDA-core kernel (float64 always)
template <typename T>
int rank_update(long long M, long long N, long long K, const T* A, long long a_rs, long long a_cs, const T* B,
                long long b_rs, long long b_cs, T* C, long long c_rs, long long c_cs, void* ws, size_t ws_bytes,
                cudaStream_t st) {
  if (M == 0 || N == 0 || K == 0) return AB_OK;
  if (sizeof(T) == 4 && c_cs == 1 && c_rs % 4 == 0 && reinterpret_cast<uintptr_t>(C) % 16 == 0) {
    bool handled = false;
    const int rc = gemm_tc_f32(0, M, N, K, -1.0f, reinterpret_cast<const float*>(A), a_rs, a_cs,
                               reinterpret_cast<const float*>(B), b_rs, b_cs, 1.0f, reinterpret_cast<float*>(C),
                               c_rs, c_cs, ws, ws_bytes, st, &handled);
    if (handled) {
      g_updates[1]++;
      return rc;
    }
  }
  g_updates[0]++;
  return gemm_simt<T>(M, N, K, -1.0, A, a_rs, a_cs, B, b_rs, b_cs, 1.0, C, c_rs, c_cs, st);
}

template <typename T>
int check_finite(const T* a, long long rows, long long cols, long long rs, long long cs, int operand,
                 unsigned long long* status, cudaStream_t st) {
  if (rows * cols == 0) return AB_OK;
  check_finite_kernel<T><<<grid_for(rows * cols), kThreads, 0, st>>>(a, rows, cols, rs, cs, operand, status);
  g_launches++;
  AB_CUDA(cudaGetLastError());
  return AB_OK;
}

template <typename T>
int copy(const T* a, long long rs, long long cs, T* out, long long rows, long long cols, int keep, cudaStream_t st) {
  if (rows * cols == 0) return AB_OK;
  copy_kernel<T><<<grid_for(rows * cols), kThreads, 0, st>>>(a, rs, cs, out, rows, cols, keep);
  g_launches++;
  AB_CUDA(cudaGetLastError());
  return AB_OK;
}

template <typename T>
int cholesky(long long n, const T* a, long long a_rs, long long a_cs, int lower, int nan_on_error, int check,
             T* out, unsigned long long* status, void* ws, size_t ws_bytes, cudaStream_t st) {
  int rc;
  if ((rc = set_smem_limits<T>())) return rc;
  if (check && (rc = check_finite<T>(a, n, n, a_rs, a_cs, 0, status, st))) return rc;
  const int keep = lower ? -1 : 1;
  if ((rc = copy<T>(a, a_rs, a_cs, out, n, n, keep, st))) return rc;
  // W is the lower factor being built: out itself for lower, out read transposed for upper
  // (out[r][c] = U[r][c] = L[c][r]), so the upper factor needs no final transpose
  const long long wr = lower ? n : 1, wc = lower ? 1 : n;
  for (long long k0 = 0; k0 < n; k0 += NB) {
    const int b = (int)std::min<long long>(NB, n - k0);
    potrf_diag_kernel<T><<<1, kFactorThreads, diag_smem<T>(), st>>>(out, wr, wc, k0, b, status);
    g_launches++;
    AB_CUDA(cudaGetLastError());
    const long long m = n - k0 - b;
    if (m == 0) break;
    // L21 = A21 L11^-T, i.e. L11 (L21)^T = (A21)^T: the panel read transposed
    T* l21 = out + (k0 + b) * wr + k0 * wc;
    const unsigned grid = (unsigned)((m + SolveCols<T>::N - 1) / SolveCols<T>::N);
    trsm_diag_kernel<T><<<grid, SolveCols<T>::N, solve_smem<T>(), st>>>(out + k0 * (wr + wc), wr, wc, b, 0, l21, wc,
                                                                       wr, m, status);
    g_launches++;
    AB_CUDA(cudaGetLastError());
    // A22 -= L21 L21^T over the whole square (the product is symmetric, so the row-major view
    // of the trailing block is updated correctly whichever way W is stored); what lands in
    // the strict upper triangle of W is cleared at the end
    if ((rc = rank_update<T>(m, m, b, l21, wr, wc, l21, wc, wr, out + (k0 + b) * (n + 1), n, 1, ws, ws_bytes, st)))
      return rc;
  }
  if ((rc = copy<T>(nullptr, 0, 0, out, n, n, keep, st))) return rc;
  if (nan_on_error) {
    nan_fill_kernel<T><<<grid_for(n * n), kThreads, 0, st>>>(out, n * n, status);
    g_launches++;
    AB_CUDA(cudaGetLastError());
  }
  return AB_OK;
}

template <typename T>
int trsm(long long n, long long nrhs, const T* a, long long a_rs, long long a_cs, int lower, int trans, int unit,
         const T* b, long long b_rs, long long b_cs, T* x, int check_finite_, int check_singular,
         unsigned long long* status, void* ws, size_t ws_bytes, cudaStream_t st) {
  int rc;
  if ((rc = set_smem_limits<T>())) return rc;
  if (check_finite_) {
    if ((rc = check_finite<T>(a, n, n, a_rs, a_cs, 0, status, st))) return rc;
    if ((rc = check_finite<T>(b, n, nrhs, b_rs, b_cs, 1, status, st))) return rc;
  }
  if (check_singular && !unit && n > 0) {
    zero_diagonal_kernel<T><<<grid_for(n), kThreads, 0, st>>>(a, n, a_rs + a_cs, status);
    g_launches++;
    AB_CUDA(cudaGetLastError());
  }
  if (n == 0 || nrhs == 0) return AB_OK;
  if (b != x || b_rs != nrhs || (nrhs > 1 && b_cs != 1))
    if ((rc = copy<T>(b, b_rs, b_cs, x, n, nrhs, 0, st))) return rc;
  // T = op(A) through strides; an upper T is walked from its last row/column backwards
  long long tr = trans ? a_cs : a_rs, tc = trans ? a_rs : a_cs;
  const T* t = a;
  long long xr = nrhs;
  T* xx = x;
  if (lower == (trans != 0)) {  // op(A) is upper triangular
    t = a + (n - 1) * (tr + tc);
    tr = -tr;
    tc = -tc;
    xx = x + (n - 1) * nrhs;
    xr = -nrhs;
  }
  for (long long r0 = 0; r0 < n; r0 += NB) {
    const int bs = (int)std::min<long long>(NB, n - r0);
    const T* tb = t + r0 * (tr + tc);
    T* xb = xx + r0 * xr;
    const long long m = n - r0 - bs;
    if (nrhs == 1) {
      trsv_diag_kernel<T><<<1, NB, 0, st>>>(tb, tr, tc, bs, unit, xb, xr, status);
      g_launches++;
      AB_CUDA(cudaGetLastError());
      if (m > 0) {
        trsv_update_kernel<T><<<grid_for(32 * m), kThreads, 0, st>>>(t + (r0 + bs) * tr + r0 * tc, tr, tc, m, bs, xb,
                                                                   xr, xb + bs * xr, xr, status);
        g_launches++;
        AB_CUDA(cudaGetLastError());
      }
      continue;
    }
    const unsigned grid = (unsigned)((nrhs + SolveCols<T>::N - 1) / SolveCols<T>::N);
    trsm_diag_kernel<T><<<grid, SolveCols<T>::N, solve_smem<T>(), st>>>(tb, tr, tc, bs, unit, xb, xr, 1, nrhs,
                                                                       status);
    g_launches++;
    AB_CUDA(cudaGetLastError());
    if (m > 0 && (rc = rank_update<T>(m, nrhs, bs, t + (r0 + bs) * tr + r0 * tc, tr, tc, xb, xr, 1, xb + bs * xr, xr,
                                      1, ws, ws_bytes, st)))
      return rc;
  }
  return AB_OK;
}

template <typename T>
size_t update_workspace(long long M, long long N, long long a_rs, long long a_cs, long long b_rs, long long b_cs) {
  if (sizeof(T) != 4 || M <= 0 || N <= 0) return 0;
  return gemm_tc_workspace(0, M, N, NB, a_rs, a_cs, b_rs, b_cs);
}

}  // namespace

extern "C" int ab_linalg_status_reset(void* status, void* stream) {
  if (!status) return fail(AB_ERR_INVALID, "null status word");
  AB_CUDA(cudaMemsetAsync(status, 0xff, sizeof(unsigned long long), as_stream(stream)));
  return AB_OK;
}

extern "C" int ab_linalg_status_check(const void* status, void* stream) {
  if (!status) return fail(AB_ERR_INVALID, "null status word");
  cudaStream_t st = as_stream(stream);
  cudaStreamCaptureStatus cap = cudaStreamCaptureStatusNone;
  AB_CUDA(cudaStreamIsCapturing(st, &cap));
  if (cap != cudaStreamCaptureStatusNone)
    return fail(AB_ERR_UNSUPPORTED, "the linear-algebra error check reads a device status word, which a CUDA "
                                    "graph cannot capture");
  unsigned long long host = kOk;
  AB_CUDA(cudaMemcpyAsync(&host, status, sizeof(host), cudaMemcpyDeviceToHost, st));
  AB_CUDA(cudaStreamSynchronize(st));
  if (host == kOk) return AB_OK;
  const int kind = (int)(host >> 56), operand = (int)((host >> 48) & 0xff);
  const long long index = (long long)(host & ((1ull << 48) - 1));
  if (kind == KIND_NONFINITE)
    return fail(AB_ERR_INVALID, "array must not contain infs or NaNs (%s, flat index %lld)", operand ? "b" : "a",
                index);
  if (kind == KIND_NOT_PD)
    return fail(AB_ERR_LINALG, "%lld-th leading minor of the array is not positive definite", index + 1);
  return fail(AB_ERR_LINALG, "singular matrix: resolution failed at diagonal %lld", index);
}

extern "C" uint64_t ab_linalg_update_count(int tensor_core) {
  return g_updates[tensor_core ? 1 : 0].load(std::memory_order_relaxed);
}

extern "C" int ab_cholesky_workspace_bytes(int dtype, int64_t n, size_t* bytes) {
  if (!bytes) return fail(AB_ERR_INVALID, "null out pointer");
  *bytes = dtype == AB_F32 ? update_workspace<float>(n - NB, n - NB, n, 1, 1, n) : 0;
  return AB_OK;
}

extern "C" int ab_cholesky(int dtype, int64_t n, const void* a, int64_t a_rs, int64_t a_cs, int lower,
                           int nan_on_error, int check_finite, void* out, void* status, void* workspace,
                           size_t workspace_bytes, void* stream) {
  if (n < 0) return fail(AB_ERR_SHAPE, "negative dimension in cholesky");
  if (n == 0) return AB_OK;
  if (!a || !out || !status) return fail(AB_ERR_INVALID, "null pointer in cholesky");
  auto* s = static_cast<unsigned long long*>(status);
  cudaStream_t st = as_stream(stream);
  if (dtype == AB_F32)
    return cholesky<float>(n, static_cast<const float*>(a), a_rs, a_cs, lower, nan_on_error, check_finite,
                           static_cast<float*>(out), s, workspace, workspace_bytes, st);
  if (dtype == AB_F64)
    return cholesky<double>(n, static_cast<const double*>(a), a_rs, a_cs, lower, nan_on_error, check_finite,
                            static_cast<double*>(out), s, workspace, workspace_bytes, st);
  return fail(AB_ERR_UNSUPPORTED, "cholesky: float32 / float64 only, got dtype code %d", dtype);
}

extern "C" int ab_trsm_workspace_bytes(int dtype, int64_t n, int64_t nrhs, size_t* bytes) {
  if (!bytes) return fail(AB_ERR_INVALID, "null out pointer");
  *bytes = dtype == AB_F32 && nrhs > 1 ? update_workspace<float>(n - NB, nrhs, n, 1, nrhs, 1) : 0;
  return AB_OK;
}

extern "C" int ab_trsm(int dtype, int64_t n, int64_t nrhs, const void* a, int64_t a_rs, int64_t a_cs, int lower,
                       int trans, int unit_diagonal, const void* b, int64_t b_rs, int64_t b_cs, void* x,
                       int check_finite, int check_singular, void* status, void* workspace, size_t workspace_bytes,
                       void* stream) {
  if (n < 0 || nrhs < 0) return fail(AB_ERR_SHAPE, "negative dimension in trsm");
  if (!status || (n > 0 && (!a || (nrhs > 0 && (!b || !x))))) return fail(AB_ERR_INVALID, "null pointer in trsm");
  auto* s = static_cast<unsigned long long*>(status);
  cudaStream_t st = as_stream(stream);
  if (dtype == AB_F32)
    return trsm<float>(n, nrhs, static_cast<const float*>(a), a_rs, a_cs, lower, trans, unit_diagonal,
                       static_cast<const float*>(b), b_rs, b_cs, static_cast<float*>(x), check_finite,
                       check_singular, s, workspace, workspace_bytes, st);
  if (dtype == AB_F64)
    return trsm<double>(n, nrhs, static_cast<const double*>(a), a_rs, a_cs, lower, trans, unit_diagonal,
                        static_cast<const double*>(b), b_rs, b_cs, static_cast<double*>(x), check_finite,
                        check_singular, s, workspace, workspace_bytes, st);
  return fail(AB_ERR_UNSUPPORTED, "trsm: float32 / float64 only, got dtype code %d", dtype);
}
