// ab_indexing.cu — AdvancedSubtensor1 / AdvancedIncSubtensor1 (SURVEY.md §8f N3: the
// embedding-lookup gather and its scatter-add gradient).
//
// Reference: aesara/tensor/subtensor.py:1925 (AdvancedSubtensor1.perform :1953-1990:
// x.take(i, axis=0), negative indices wrap, out-of-range -> IndexError) and :2128
// (AdvancedIncSubtensor1.perform: np.add.at(x, idx, y) — duplicates accumulate — or
// x[idx] = y with set_instead_of_inc).
//
// Byte/integer work, HBM-bound: rows of `inner` contiguous elements are moved with the
// widest aligned vector; x is viewed as [n_rows, inner], idx as int64[n_idx].
// Out-of-range indices cannot raise from a kernel: they set a device flag that the host
// reads after the launch (the reference's IndexError).  Scatter-add uses atomicAdd, so
// for floating point the order in which duplicates are summed is not fixed (integer
// results are exact; float results agree to rounding).
#include <algorithm>

#include "ab_common.h"

using namespace ab;

namespace {

constexpr int kThreads = 256;

template <typename IDX>
__device__ __forceinline__ long long wrap_index(IDX raw, long long n_rows, int* err) {
  long long i = (long long)raw;
  if (i < 0) i += n_rows;
  if (i < 0 || i >= n_rows) {
    *err = 1;
    return -1;
  }
  return i;
}

// gather: out[r, :] = x[idx[r], :], element size es bytes, rows of `row_bytes`
template <typename V, typename IDX>
__global__ void __launch_bounds__(kThreads)
gather_rows_kernel(const V* __restrict__ x, long long x_row_stride_v, const IDX* __restrict__ idx,
                   long long idx_stride, V* __restrict__ out, long long n_idx, long long n_rows,
                   long long row_v, int* err) {
  const long long total = n_idx * row_v;
  for (long long t = (long long)blockIdx.x * kThreads + threadIdx.x; t < total;
       t += (long long)gridDim.x * kThreads) {
    const long long r = t / row_v, c = t - r * row_v;
    const long long src = wrap_index(idx[r * idx_stride], n_rows, err);
    if (src >= 0) out[r * row_v + c] = x[src * x_row_stride_v + c];
  }
}

template <typename T, typename IDX, bool SET>
__global__ void __launch_bounds__(kThreads)
scatter_rows_kernel(T* __restrict__ x, long long x_row_stride, const IDX* __restrict__ idx,
                    long long idx_stride, const T* __restrict__ y, long long y_row_stride,
                    long long y_col_stride, long long n_idx, long long n_rows, long long inner,
                    int* err) {
  const long long total = n_idx * inner;
  for (long long t = (long long)blockIdx.x * kThreads + threadIdx.x; t < total;
       t += (long long)gridDim.x * kThreads) {
    const long long r = t / inner, c = t - r * inner;
    const long long dst = wrap_index(idx[r * idx_stride], n_rows, err);
    if (dst < 0) continue;
    const T v = y[r * y_row_stride + c * y_col_stride];
    if (SET) x[dst * x_row_stride + c] = v;
    else atomicAdd(&x[dst * x_row_stride + c], v);
  }
}

// integer types without a native atomicAdd overload go through CAS on the containing word
template <typename T>
__device__ __forceinline__ void atomic_add_small(T* addr, T v) {
  unsigned int* base = reinterpret_cast<unsigned int*>(reinterpret_cast<uintptr_t>(addr) & ~(uintptr_t)3);
  const unsigned shift = (unsigned)((reinterpret_cast<uintptr_t>(addr) & 3) * 8);
  const unsigned mask = (sizeof(T) == 1 ? 0xFFu : 0xFFFFu) << shift;
  unsigned int old = *base, assumed;
  do {
    assumed = old;
    const T cur = (T)((assumed & mask) >> shift);
    const unsigned nv = (assumed & ~mask) | ((((unsigned)(T)(cur + v)) << shift) & mask);
    old = atomicCAS(base, assumed, nv);
  } while (old != assumed);
}

template <typename T, typename IDX, bool SET>
__global__ void __launch_bounds__(kThreads)
scatter_rows_small_kernel(T* __restrict__ x, long long x_row_stride, const IDX* __restrict__ idx,
                          long long idx_stride, const T* __restrict__ y, long long y_row_stride,
                          long long y_col_stride, long long n_idx, long long n_rows,
                          long long inner, int* err) {
  const long long total = n_idx * inner;
  for (long long t = (long long)blockIdx.x * kThreads + threadIdx.x; t < total;
       t += (long long)gridDim.x * kThreads) {
    const long long r = t / inner, c = t - r * inner;
    const long long dst = wrap_index(idx[r * idx_stride], n_rows, err);
    if (dst < 0) continue;
    const T v = y[r * y_row_stride + c * y_col_stride];
    if (SET) x[dst * x_row_stride + c] = v;
    else atomic_add_small<T>(&x[dst * x_row_stride + c], v);
  }
}

__global__ void clear_flag_kernel(int* f) { *f = 0; }

unsigned grid_for(long long total) {
  long long b = (total + kThreads - 1) / kThreads;
  return (unsigned)std::max<long long>(1, std::min<long long>(b, 132LL * 32));
}

template <typename IDX>
int gather_impl(int itemsize, const void* x, long long x_row_stride, const void* idx,
                long long idx_stride, void* out, long long n_idx, long long n_rows,
                long long inner, int* err, cudaStream_t st) {
  if (n_idx == 0 || inner == 0) return AB_OK;
  const long long row_bytes = inner * itemsize;
  const long long stride_bytes = x_row_stride * itemsize;
  const uintptr_t a = reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(out);
  const IDX* ip = static_cast<const IDX*>(idx);
#define AB_GATHER(V)                                                                         \
  gather_rows_kernel<V, IDX><<<grid_for(n_idx*(row_bytes / (long long)sizeof(V))), kThreads, 0, st>>>( \
      static_cast<const V*>(x), stride_bytes / (long long)sizeof(V), ip, idx_stride,        \
      static_cast<V*>(out), n_idx, n_rows, row_bytes / (long long)sizeof(V), err)
  if (row_bytes % 16 == 0 && stride_bytes % 16 == 0 && a % 16 == 0) AB_GATHER(uint4);
  else if (row_bytes % 8 == 0 && stride_bytes % 8 == 0 && a % 8 == 0) AB_GATHER(uint2);
  else if (row_bytes % 4 == 0 && stride_bytes % 4 == 0 && a % 4 == 0) AB_GATHER(unsigned int);
  else if (row_bytes % 2 == 0 && stride_bytes % 2 == 0 && a % 2 == 0) AB_GATHER(unsigned short);
  else AB_GATHER(unsigned char);
#undef AB_GATHER
  g_launches++;
  AB_CUDA(cudaGetLastError());
  return AB_OK;
}

template <typename T, typename IDX, bool SMALL>
int scatter_impl(bool set, void* x, long long x_row_stride, const void* idx, long long idx_stride,
                 const void* y, long long y_rs, long long y_cs, long long n_idx, long long n_rows,
                 long long inner, int* err, cudaStream_t st) {
  if (n_idx == 0 || inner == 0) return AB_OK;
  const unsigned grid = grid_for(n_idx * inner);
  T* xp = static_cast<T*>(x);
  const T* yp = static_cast<const T*>(y);
  const IDX* ip = static_cast<const IDX*>(idx);
  if constexpr (SMALL) {
    if (set) scatter_rows_small_kernel<T, IDX, true><<<grid, kThreads, 0, st>>>(xp, x_row_stride, ip, idx_stride, yp, y_rs, y_cs, n_idx, n_rows, inner, err);
    else scatter_rows_small_kernel<T, IDX, false><<<grid, kThreads, 0, st>>>(xp, x_row_stride, ip, idx_stride, yp, y_rs, y_cs, n_idx, n_rows, inner, err);
  } else {
    if (set) scatter_rows_kernel<T, IDX, true><<<grid, kThreads, 0, st>>>(xp, x_row_stride, ip, idx_stride, yp, y_rs, y_cs, n_idx, n_rows, inner, err);
    else scatter_rows_kernel<T, IDX, false><<<grid, kThreads, 0, st>>>(xp, x_row_stride, ip, idx_stride, yp, y_rs, y_cs, n_idx, n_rows, inner, err);
  }
  g_launches++;
  AB_CUDA(cudaGetLastError());
  return AB_OK;
}

int* error_flag() {
  static int* flag = nullptr;
  if (!flag) {
    if (cudaMalloc(&flag, sizeof(int)) != cudaSuccess) return nullptr;
    cudaMemset(flag, 0, sizeof(int));
  }
  return flag;
}

int read_and_clear_flag(int* flag, cudaStream_t st, const char* what) {
  int host = 0;
  AB_CUDA(cudaMemcpyAsync(&host, flag, sizeof(int), cudaMemcpyDeviceToHost, st));
  AB_CUDA(cudaStreamSynchronize(st));
  if (host) {
    clear_flag_kernel<<<1, 1, 0, st>>>(flag);
    return fail(AB_ERR_SHAPE, "index out of bounds in %s", what);
  }
  return AB_OK;
}

}  // namespace

// x: [n_rows, inner] with row stride x_row_stride (elements, inner contiguous);
// idx: int32/int64 vector; out: C-contiguous [n_idx, inner].  check != 0 synchronises the
// stream and returns AB_ERR_SHAPE if any index was out of range.
extern "C" int ab_take_rows(int itemsize, int idx_dtype, const void* x, int64_t x_row_stride,
                            int64_t n_rows, int64_t inner, const void* idx, int64_t idx_stride,
                            int64_t n_idx, void* out, int check, void* stream) {
  cudaStream_t st = as_stream(stream);
  int* flag = error_flag();
  if (!flag) return fail(AB_ERR_CUDA, "cannot allocate the index-error flag");
  int rc;
  if (idx_dtype == AB_I64) rc = gather_impl<long long>(itemsize, x, x_row_stride, idx, idx_stride, out, n_idx, n_rows, inner, flag, st);
  else if (idx_dtype == AB_I32) rc = gather_impl<int>(itemsize, x, x_row_stride, idx, idx_stride, out, n_idx, n_rows, inner, flag, st);
  else if (idx_dtype == AB_I16) rc = gather_impl<short>(itemsize, x, x_row_stride, idx, idx_stride, out, n_idx, n_rows, inner, flag, st);
  else if (idx_dtype == AB_I8) rc = gather_impl<signed char>(itemsize, x, x_row_stride, idx, idx_stride, out, n_idx, n_rows, inner, flag, st);
  else if (idx_dtype == AB_U8) rc = gather_impl<unsigned char>(itemsize, x, x_row_stride, idx, idx_stride, out, n_idx, n_rows, inner, flag, st);
  else if (idx_dtype == AB_U16) rc = gather_impl<unsigned short>(itemsize, x, x_row_stride, idx, idx_stride, out, n_idx, n_rows, inner, flag, st);
  else if (idx_dtype == AB_U32) rc = gather_impl<unsigned int>(itemsize, x, x_row_stride, idx, idx_stride, out, n_idx, n_rows, inner, flag, st);
  else return fail(AB_ERR_UNSUPPORTED, "index dtype code %d", idx_dtype);
  if (rc) return rc;
  return check ? read_and_clear_flag(flag, st, "AdvancedSubtensor1") : AB_OK;
}

// x[idx[r], :] (+)= y[r, :]   (y may broadcast: strides 0)
extern "C" int ab_scatter_rows(int dtype, int idx_dtype, int set_instead_of_inc, void* x,
                               int64_t x_row_stride, int64_t n_rows, int64_t inner,
                               const void* idx, int64_t idx_stride, int64_t n_idx, const void* y,
                               int64_t y_row_stride, int64_t y_col_stride, int check,
                               void* stream) {
  cudaStream_t st = as_stream(stream);
  int* flag = error_flag();
  if (!flag) return fail(AB_ERR_CUDA, "cannot allocate the index-error flag");
  const bool set = set_instead_of_inc != 0;
  int rc = AB_ERR_UNSUPPORTED;
#define AB_SC(T, SMALL)                                                                          \
  (idx_dtype == AB_I64 ? scatter_impl<T, long long, SMALL>(set, x, x_row_stride, idx, idx_stride, y, y_row_stride, y_col_stride, n_idx, n_rows, inner, flag, st) \
   : idx_dtype == AB_I32 ? scatter_impl<T, int, SMALL>(set, x, x_row_stride, idx, idx_stride, y, y_row_stride, y_col_stride, n_idx, n_rows, inner, flag, st)    \
                         : fail(AB_ERR_UNSUPPORTED, "index dtype code %d (int32/int64 supported)", idx_dtype))
  switch (dtype) {
    case AB_F32: rc = AB_SC(float, false); break;
    case AB_F64: rc = AB_SC(double, false); break;
    case AB_I32: rc = AB_SC(int, false); break;
    case AB_U32: rc = AB_SC(unsigned int, false); break;
    case AB_I64: rc = AB_SC(unsigned long long, false); break;  // two's complement add
    case AB_U64: rc = AB_SC(unsigned long long, false); break;
    case AB_I16: case AB_U16: rc = AB_SC(unsigned short, true); break;
    case AB_I8: case AB_U8: rc = AB_SC(unsigned char, true); break;
    default: return fail(AB_ERR_UNSUPPORTED, "AdvancedIncSubtensor1: dtype code %d", dtype);
  }
#undef AB_SC
  if (rc) return rc;
  return check ? read_and_clear_flag(flag, st, "AdvancedIncSubtensor1") : AB_OK;
}


// ---- several index vectors -> one flat row index (AdvancedSubtensor, subtensor.py:2577) ----
// flat[r] = ravel(idx_0[r], ..., idx_{k-1}[r]) over dims d_0..d_{k-1}; negative indices wrap,
// an out-of-range index sets the error flag (flat = 0 keeps the following gather in bounds).
namespace {
struct RavelParams {
  const long long* idx[4];
  long long stride[4];   // element strides (0 = a length-1 index vector broadcast over r)
  long long dims[4];
  int k;
  long long n;
};
__global__ void __launch_bounds__(256)
ravel_index_kernel(const __grid_constant__ RavelParams p, long long* __restrict__ out, int* flag) {
  const long long r = (long long)blockIdx.x * 256 + threadIdx.x;
  if (r >= p.n) return;
  long long flat = 0;
  bool ok = true;
  for (int j = 0; j < p.k; ++j) {
    long long v = p.idx[j][r * p.stride[j]];
    if (v < 0) v += p.dims[j];
    ok = ok && v >= 0 && v < p.dims[j];
    flat = flat * p.dims[j] + v;
  }
  if (!ok) { *flag = 1; flat = 0; }
  out[r] = flat;
}
template <typename T>
__global__ void __launch_bounds__(256)
arange_kernel(T start, T step, long long n, T* __restrict__ out) {
  const long long i = (long long)blockIdx.x * 256 + threadIdx.x;
  if (i < n) out[i] = (T)(start + (T)i * step);
}
}  // namespace

extern "C" int ab_ravel_index(int k, const void* const* idx, const int64_t* idx_stride,
                              const int64_t* dims, int64_t n, void* out, int check, void* stream) {
  if (k < 1 || k > 4) return fail(AB_ERR_UNSUPPORTED, "ab_ravel_index takes 1..4 index vectors, got %d", k);
  if (n <= 0) return AB_OK;
  cudaStream_t st = as_stream(stream);
  int* flag = error_flag();
  if (!flag) return fail(AB_ERR_CUDA, "cannot allocate the index-error flag");
  RavelParams p{};
  p.k = k;
  p.n = n;
  for (int j = 0; j < k; ++j) {
    p.idx[j] = static_cast<const long long*>(idx[j]);
    p.stride[j] = idx_stride[j];
    p.dims[j] = dims[j];
  }
  ravel_index_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(p, static_cast<long long*>(out), flag);
  g_launches++;
  AB_CUDA(cudaGetLastError());
  return check ? read_and_clear_flag(flag, st, "AdvancedSubtensor") : AB_OK;
}

// ARange (tensor/basic.py:3011): out[i] = start + i * step, evaluated in the output dtype
extern "C" int ab_arange(int dtype, double start, double step, int64_t start_i, int64_t step_i,
                         int64_t n, void* out, void* stream) {
  if (n <= 0) return AB_OK;
  cudaStream_t st = as_stream(stream);
  const unsigned blocks = (unsigned)((n + 255) / 256);
  switch (dtype) {
    case AB_F32: arange_kernel<float><<<blocks, 256, 0, st>>>((float)start, (float)step, n, static_cast<float*>(out)); break;
    case AB_F64: arange_kernel<double><<<blocks, 256, 0, st>>>(start, step, n, static_cast<double*>(out)); break;
    case AB_I64: arange_kernel<long long><<<blocks, 256, 0, st>>>(start_i, step_i, n, static_cast<long long*>(out)); break;
    case AB_I32: arange_kernel<int><<<blocks, 256, 0, st>>>((int)start_i, (int)step_i, n, static_cast<int*>(out)); break;
    case AB_I16: arange_kernel<short><<<blocks, 256, 0, st>>>((short)start_i, (short)step_i, n, static_cast<short*>(out)); break;
    case AB_I8: arange_kernel<signed char><<<blocks, 256, 0, st>>>((signed char)start_i, (signed char)step_i, n, static_cast<signed char*>(out)); break;
    case AB_U8: arange_kernel<unsigned char><<<blocks, 256, 0, st>>>((unsigned char)start_i, (unsigned char)step_i, n, static_cast<unsigned char*>(out)); break;
    default: return fail(AB_ERR_UNSUPPORTED, "ARange: dtype code %d", dtype);
  }
  g_launches++;
  AB_CUDA(cudaGetLastError());
  return AB_OK;
}


// ---- CumOp (cumsum / cumprod along one axis; aesara/tensor/extra_ops.py:253) --------------
// x viewed as [outer, L, inner] (C-contiguous).  inner > 1: one thread per (outer, inner)
// line, consecutive threads on consecutive `inner` (coalesced), sequential over L.
// inner == 1: one CTA per line — chunks of 256 x 8 elements, thread-local scan, warp-shuffle
// scan of the thread totals, carry from chunk to chunk.  Output dtype = input dtype (the
// reference's C implementation, extra_ops.py:325-375, accumulates in that type too).
namespace {
template <typename T, bool MUL>
__device__ __forceinline__ T cum_op(T a, T b) { return MUL ? (T)(a * b) : (T)(a + b); }

template <typename T, bool MUL>
__global__ void __launch_bounds__(256)
cum_lines_kernel(const T* __restrict__ x, T* __restrict__ out, long long outer, long long L, long long inner) {
  const long long t = (long long)blockIdx.x * 256 + threadIdx.x;
  if (t >= outer * inner) return;
  const long long o = t / inner, i = t - o * inner;
  const T* p = x + o * L * inner + i;
  T* q = out + o * L * inner + i;
  T acc = MUL ? (T)1 : (T)0;
  for (long long l = 0; l < L; ++l) {
    acc = cum_op<T, MUL>(acc, p[l * inner]);
    q[l * inner] = acc;
  }
}

template <typename T, bool MUL>
__global__ void __launch_bounds__(256)
cum_block_kernel(const T* __restrict__ x, T* __restrict__ out, long long L) {
  constexpr int ITEMS = 8;
  __shared__ T warp_tot[8];
  __shared__ T carry_s;
  const T ident = MUL ? (T)1 : (T)0;
  const T* p = x + (long long)blockIdx.x * L;
  T* q = out + (long long)blockIdx.x * L;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (threadIdx.x == 0) carry_s = ident;
  __syncthreads();
  for (long long base = 0; base < L; base += 256 * ITEMS) {
    T v[ITEMS];
    const long long s0 = base + (long long)threadIdx.x * ITEMS;
    T run = ident;
#pragma unroll
    for (int k = 0; k < ITEMS; ++k) {
      const T e = (s0 + k < L) ? p[s0 + k] : ident;
      run = cum_op<T, MUL>(run, e);
      v[k] = run;
    }
    // inclusive scan of the thread totals inside the warp
    T incl = run;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const T up = __shfl_up_sync(0xffffffffu, incl, d);
      if (lane >= d) incl = cum_op<T, MUL>(up, incl);
    }
    if (lane == 31) warp_tot[warp] = incl;
    __syncthreads();
    T prefix = carry_s;                       // everything before this chunk
    for (int w = 0; w < warp; ++w) prefix = cum_op<T, MUL>(prefix, warp_tot[w]);
    T excl = __shfl_up_sync(0xffffffffu, incl, 1);
    if (lane == 0) excl = ident;
    prefix = cum_op<T, MUL>(prefix, excl);     // everything before this thread's items
#pragma unroll
    for (int k = 0; k < ITEMS; ++k)
      if (s0 + k < L) q[s0 + k] = cum_op<T, MUL>(prefix, v[k]);
    __syncthreads();
    if (threadIdx.x == 255) carry_s = cum_op<T, MUL>(prefix, run);
    __syncthreads();
  }
}

template <typename T>
int cum_dispatch(bool mul, const void* x, void* out, long long outer, long long L, long long inner,
                 cudaStream_t st) {
  const T* xi = static_cast<const T*>(x);
  T* oo = static_cast<T*>(out);
  if (inner == 1) {
    if (mul) cum_block_kernel<T, true><<<(unsigned)outer, 256, 0, st>>>(xi, oo, L);
    else cum_block_kernel<T, false><<<(unsigned)outer, 256, 0, st>>>(xi, oo, L);
  } else {
    const unsigned blocks = (unsigned)((outer * inner + 255) / 256);
    if (mul) cum_lines_kernel<T, true><<<blocks, 256, 0, st>>>(xi, oo, outer, L, inner);
    else cum_lines_kernel<T, false><<<blocks, 256, 0, st>>>(xi, oo, outer, L, inner);
  }
  g_launches++;
  AB_CUDA(cudaGetLastError());
  return AB_OK;
}
}  // namespace

extern "C" int ab_cumulative(int dtype, int mul, const void* x, void* out, int64_t outer, int64_t len,
                             int64_t inner, void* stream) {
  if (outer <= 0 || len <= 0 || inner <= 0) return AB_OK;
  if (outer > 0x7fffffffLL) return fail(AB_ERR_UNSUPPORTED, "CumOp over more than 2^31 lines");
  cudaStream_t st = as_stream(stream);
  switch (dtype) {
    case AB_F32: return cum_dispatch<float>(mul != 0, x, out, outer, len, inner, st);
    case AB_F64: return cum_dispatch<double>(mul != 0, x, out, outer, len, inner, st);
    case AB_I64: return cum_dispatch<long long>(mul != 0, x, out, outer, len, inner, st);
    case AB_I32: return cum_dispatch<int>(mul != 0, x, out, outer, len, inner, st);
    case AB_I16: return cum_dispatch<short>(mul != 0, x, out, outer, len, inner, st);
    case AB_I8: return cum_dispatch<signed char>(mul != 0, x, out, outer, len, inner, st);
    case AB_U8: return cum_dispatch<unsigned char>(mul != 0, x, out, outer, len, inner, st);
    case AB_U16: return cum_dispatch<unsigned short>(mul != 0, x, out, outer, len, inner, st);
    case AB_U32: return cum_dispatch<unsigned int>(mul != 0, x, out, outer, len, inner, st);
    case AB_U64: return cum_dispatch<unsigned long long>(mul != 0, x, out, outer, len, inner, st);
    default: return fail(AB_ERR_UNSUPPORTED, "CumOp: dtype code %d", dtype);
  }
}
