// ab_random.cu — draws of RandomVariable nodes (aesara/tensor/random/basic.py: UniformRV,
// NormalRV, BernoulliRV and BinomialRV with n = 1) from a counter-based Philox stream.
//
// The stream (README "Random draws"; oracle/random_np.py restates it in NumPy):
//   32-bit word w[i] is word i % 4 of Philox4x32-10 (Salmon et al., SC'11, Random123
//   constants) at counter (b_lo, b_hi, 0, 0), b = i / 4, under the 64-bit key (k_lo, k_hi)
//   the host drew from the node's Generator.  Element j (C order of the output) uses only its
//   own words, so a value depends on (key, j, the parameters at j) and never on the launch.
//     uniform f32   u = (w[j] >> 8) * 2^-24,                   low + (high - low) * u
//     uniform f64   u = ((w[2j+1] << 32 | w[2j]) >> 11) * 2^-53, same affine step
//     normal        Box-Muller on pair m -> elements 2m, 2m+1: f32 from words 2m, 2m+1, f64
//                   from words 4m..4m+3 (two 53-bit integers); u1 = (int + 1) * 2^-k in (0, 1],
//                   u2 = int * 2^-k in [0, 1); r = sqrt(-2 log u1), z = r cos(2 pi u2),
//                   r sin(2 pi u2); loc + scale * z
//     bernoulli     int64((w[j] >> 8) * 2^-24 < p), compared in float64
//   Every affine step rounds each operation on its own (no FMA contraction), so a NumPy port
//   reproduces uniform and Bernoulli draws bit for bit.
//
// One Philox block (4 words) makes 4 elements (f32 uniform, f32 normal, Bernoulli) or 2 (f64):
// a thread computes a block in registers and writes its elements with 128-bit stores.  The
// parameters are read through broadcast strides over the dims the Elemwise launcher's collapse
// leaves (one dim for scalars and full-shape contiguous parameters).  An invalid parameter
// (scale < 0, p outside [0, 1] or NaN) cannot raise from a kernel: it sets a device flag that
// the launcher reads after the launch when asked to, like the index checks of ab_indexing.cu.
#include <algorithm>

#include "ab_common.h"

using namespace ab;

namespace {

constexpr int kThreads = 256;
enum { DIST_UNIFORM = 0, DIST_NORMAL = 1, DIST_BERNOULLI = 2 };

struct RngParams {
  long long n;       // elements
  long long blocks;  // Philox blocks
  int nd;            // dims of the parameter index space (>= 1)
  int n_params;
  int vec;           // out is 16-byte aligned: whole blocks are written with 128-bit stores
  unsigned k0, k1;
  long long shape[AB_MAX_DIMS];
  const void* p[2];
  long long st[2][AB_MAX_DIMS];
  int* err;          // NULL: parameters are not checked
};

__device__ __forceinline__ uint4 philox4x32_10(unsigned c0, unsigned c1, unsigned k0, unsigned k1) {
  const unsigned M0 = 0xD2511F53u, M1 = 0xCD9E8D57u, W0 = 0x9E3779B9u, W1 = 0xBB67AE85u;
  unsigned c2 = 0u, c3 = 0u;
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    const unsigned hi0 = __umulhi(M0, c0), lo0 = M0 * c0;
    const unsigned hi1 = __umulhi(M1, c2), lo1 = M1 * c2;
    c0 = hi1 ^ c1 ^ k0;
    c1 = lo1;
    c2 = hi0 ^ c3 ^ k1;
    c3 = lo0;
    k0 += W0;
    k1 += W1;
  }
  return make_uint4(c0, c1, c2, c3);
}

// element offset of parameter k at output element j
__device__ __forceinline__ long long param_offset(const RngParams& P, int k, long long j) {
  if (P.nd == 1) return j * P.st[k][0];
  long long off = 0;
  for (int d = P.nd - 1; d >= 0; --d) {
    const long long s = P.shape[d], q = j / s;
    off += (j - q * s) * P.st[k][d];
    j = q;
  }
  return off;
}

template <typename T>
__device__ __forceinline__ T param(const RngParams& P, int k, long long j) {
  return static_cast<const T*>(P.p[k])[param_offset(P, k, j)];
}

__device__ __forceinline__ float affine(float a, float b, float u) { return __fadd_rn(a, __fmul_rn(b, u)); }
__device__ __forceinline__ double affine(double a, double b, double u) { return __dadd_rn(a, __dmul_rn(b, u)); }
__device__ __forceinline__ float diff(float a, float b) { return __fsub_rn(a, b); }
__device__ __forceinline__ double diff(double a, double b) { return __dsub_rn(a, b); }

__device__ __forceinline__ float unit24(unsigned w) { return (float)(w >> 8) * 0x1p-24f; }
__device__ __forceinline__ unsigned long long bits53(unsigned lo, unsigned hi) {
  return (((unsigned long long)hi << 32) | lo) >> 11;
}

__device__ __forceinline__ void box_muller(unsigned a, unsigned b, float* z0, float* z1) {
  const float u1 = (float)((a >> 8) + 1u) * 0x1p-24f, u2 = (float)(b >> 8) * 0x1p-24f;
  const float r = sqrtf(-2.0f * logf(u1));
  float s, c;
  sincospif(2.0f * u2, &s, &c);
  *z0 = r * c;
  *z1 = r * s;
}

__device__ __forceinline__ void box_muller(uint4 w, double* z0, double* z1) {
  const double u1 = (double)(bits53(w.x, w.y) + 1ull) * 0x1p-53, u2 = (double)bits53(w.z, w.w) * 0x1p-53;
  const double r = sqrt(-2.0 * log(u1));
  double s, c;
  sincospi(2.0 * u2, &s, &c);
  *z0 = r * c;
  *z1 = r * s;
}

// the E = 4 (f32, Bernoulli) or 2 (f64) raw values of one block, before the parameters
template <int DIST, typename T>
struct Block;

template <> struct Block<DIST_UNIFORM, float> {
  static constexpr int E = 4;
  __device__ static void raw(uint4 w, float* v) { v[0] = unit24(w.x); v[1] = unit24(w.y); v[2] = unit24(w.z); v[3] = unit24(w.w); }
};
template <> struct Block<DIST_UNIFORM, double> {
  static constexpr int E = 2;
  __device__ static void raw(uint4 w, double* v) {
    v[0] = (double)bits53(w.x, w.y) * 0x1p-53;
    v[1] = (double)bits53(w.z, w.w) * 0x1p-53;
  }
};
template <> struct Block<DIST_NORMAL, float> {
  static constexpr int E = 4;
  __device__ static void raw(uint4 w, float* v) { box_muller(w.x, w.y, &v[0], &v[1]); box_muller(w.z, w.w, &v[2], &v[3]); }
};
template <> struct Block<DIST_NORMAL, double> {
  static constexpr int E = 2;
  __device__ static void raw(uint4 w, double* v) { box_muller(w, &v[0], &v[1]); }
};
template <> struct Block<DIST_BERNOULLI, long long> {
  static constexpr int E = 4;
  __device__ static void raw(uint4 w, float* v) { v[0] = unit24(w.x); v[1] = unit24(w.y); v[2] = unit24(w.z); v[3] = unit24(w.w); }
};

// the parameters of one element (Bernoulli: p in a)
template <typename PT>
struct Par {
  PT a, b;
};

template <int DIST, typename PT>
__device__ __forceinline__ Par<PT> load_par(const RngParams& P, long long j) {
  Par<PT> q;
  q.a = param<PT>(P, 0, j);
  q.b = DIST == DIST_BERNOULLI ? q.a : param<PT>(P, 1, j);
  if (P.err) {
    if (DIST == DIST_NORMAL && q.b < (PT)0) *P.err = 1;
    if (DIST == DIST_BERNOULLI && !(q.a >= (PT)0 && q.a <= (PT)1)) *P.err = 1;
  }
  return q;
}

// parameters applied to raw value v
template <int DIST, typename T, typename PT, typename R>
__device__ __forceinline__ T finish(Par<PT> q, R v) {
  if constexpr (DIST == DIST_UNIFORM) return affine(q.a, diff(q.b, q.a), v);
  else if constexpr (DIST == DIST_NORMAL) return affine(q.a, q.b, v);
  else return (long long)((double)v < q.a);
}

template <typename T, int E>
__device__ __forceinline__ void store_block(T* out, const T* v) {
  if constexpr (sizeof(T) * E == 16) {
    if constexpr (sizeof(T) == 4)
      *reinterpret_cast<float4*>(out) = make_float4(v[0], v[1], v[2], v[3]);
    else
      *reinterpret_cast<double2*>(out) = make_double2(v[0], v[1]);
  } else {  // 4 x int64
    reinterpret_cast<longlong2*>(out)[0] = make_longlong2(v[0], v[1]);
    reinterpret_cast<longlong2*>(out)[1] = make_longlong2(v[2], v[3]);
  }
}

// SCALAR: every parameter has stride 0, so it is read once per thread
template <int DIST, typename T, bool SCALAR>
__global__ void __launch_bounds__(kThreads) random_kernel(const __grid_constant__ RngParams P, T* __restrict__ out) {
  using B = Block<DIST, T>;
  constexpr int E = B::E;
  using R = std::conditional_t<DIST == DIST_BERNOULLI, float, T>;
  using PT = std::conditional_t<DIST == DIST_BERNOULLI, double, T>;
  Par<PT> q0 = {};
  if (SCALAR) q0 = load_par<DIST, PT>(P, 0);
  for (long long b = (long long)blockIdx.x * kThreads + threadIdx.x; b < P.blocks;
       b += (long long)gridDim.x * kThreads) {
    R raw[E];
    B::raw(philox4x32_10((unsigned)b, (unsigned)(b >> 32), P.k0, P.k1), raw);
    const long long j0 = b * E;
    T v[E];
#pragma unroll
    for (int e = 0; e < E; ++e) {
      // the elements past the end of the last block are computed but not stored: they read
      // the parameters of the last element
      const Par<PT> q = SCALAR ? q0 : load_par<DIST, PT>(P, j0 + e < P.n ? j0 + e : P.n - 1);
      v[e] = finish<DIST, T>(q, raw[e]);
    }
    if constexpr (sizeof(T) * E == 32) {
      // 32 bytes per thread: two 128-bit stores, each covering 512 contiguous bytes of the warp
      // (store k holds lanes 16k..16k+15; lane l writes half l & 1 of lane 16k + l / 2) when
      // every lane of the warp has a whole block, so no store leaves a 32-byte sector half written
      const int lane = threadIdx.x & 31;
      if (P.vec && (b - lane + 32) * E <= P.n) {
#pragma unroll
        for (int k = 0; k < 2; ++k) {
          const int src = 16 * k + (lane >> 1);
          const T a0 = __shfl_sync(0xffffffffu, v[0], src), a1 = __shfl_sync(0xffffffffu, v[1], src);
          const T c0 = __shfl_sync(0xffffffffu, v[2], src), c1 = __shfl_sync(0xffffffffu, v[3], src);
          const T pair[2] = {lane & 1 ? c0 : a0, lane & 1 ? c1 : a1};
          const long long base = (b - lane + 16 * k + (lane >> 1)) * E + 2 * (lane & 1);
          *reinterpret_cast<longlong2*>(out + base) = make_longlong2(pair[0], pair[1]);
        }
        continue;
      }
    }
    if (P.vec && j0 + E <= P.n) {
      store_block<T, E>(out + j0, v);
    } else {
#pragma unroll
      for (int e = 0; e < E; ++e)
        if (j0 + e < P.n) out[j0 + e] = v[e];
    }
  }
}

int* error_flag() {
  static int* flag = nullptr;
  if (!flag) {
    if (cudaMalloc(&flag, sizeof(int)) != cudaSuccess) return nullptr;
    cudaMemset(flag, 0, sizeof(int));
  }
  return flag;
}

__global__ void clear_flag_kernel(int* f) { *f = 0; }

int sm_count() {
  static int n = 0;
  if (!n) {
    int dev = 0;
    cudaGetDevice(&dev);
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) n = 132;
  }
  return n;
}

template <int DIST, typename T>
int launch(const RngParams& P, void* out, cudaStream_t st) {
  long long grid = (P.blocks + kThreads - 1) / kThreads;
  grid = std::max<long long>(1, std::min<long long>(grid, (long long)sm_count() * 16));
  bool scalar = P.nd == 1;
  for (int k = 0; k < P.n_params; ++k) scalar = scalar && P.st[k][0] == 0;
  if (scalar) random_kernel<DIST, T, true><<<(unsigned)grid, kThreads, 0, st>>>(P, static_cast<T*>(out));
  else random_kernel<DIST, T, false><<<(unsigned)grid, kThreads, 0, st>>>(P, static_cast<T*>(out));
  g_launches++;
  AB_CUDA(cudaGetLastError());
  return AB_OK;
}

}  // namespace

extern "C" int ab_random(int dist, int dtype, uint64_t key, int ndim, const int64_t* shape, int n_params,
                         const void* const* params, const int64_t* param_strides, void* out, int check,
                         void* stream) {
  if (ndim < 0 || ndim > AB_MAX_RAW_DIMS) return fail(AB_ERR_INVALID, "bad ndim %d", ndim);
  const int want = dist == DIST_BERNOULLI ? 1 : 2;
  if (dist < DIST_UNIFORM || dist > DIST_BERNOULLI) return fail(AB_ERR_UNSUPPORTED, "random: distribution code %d", dist);
  if (n_params != want) return fail(AB_ERR_INVALID, "random: distribution %d takes %d parameters, got %d", dist, want, n_params);
  if (dist == DIST_BERNOULLI ? dtype != AB_I64 : (dtype != AB_F32 && dtype != AB_F64))
    return fail(AB_ERR_UNSUPPORTED, "random: distribution %d does not draw dtype code %d", dist, dtype);
  long long total = 1;
  for (int d = 0; d < ndim; ++d) {
    if (shape[d] < 0) return fail(AB_ERR_INVALID, "negative dimension");
    total *= shape[d];
  }
  if (total == 0) return AB_OK;
  if (!out) return fail(AB_ERR_INVALID, "null out pointer");

  // operands 0..n_params-1: the parameters; operand n_params: the C-contiguous output
  const int nops = n_params + 1;
  std::vector<int64_t> strides((size_t)nops * ndim);
  for (int k = 0; k < n_params; ++k)
    for (int d = 0; d < ndim; ++d) strides[(size_t)k * ndim + d] = param_strides[(size_t)k * ndim + d];
  int64_t acc = 1;
  for (int d = ndim - 1; d >= 0; --d) {
    strides[(size_t)n_params * ndim + d] = acc;
    acc *= shape[d];
  }
  std::vector<int64_t> shp;
  std::vector<std::vector<int64_t>> st;
  collapse_dims(nops, ndim, shape, strides.data(), n_params, shp, st);
  if (shp.size() > AB_MAX_DIMS)
    return fail(AB_ERR_UNSUPPORTED, "random: parameters over %d non-mergeable dims (max %d)", (int)shp.size(), AB_MAX_DIMS);

  RngParams P = {};
  P.n = total;
  P.n_params = n_params;
  P.k0 = (unsigned)key;
  P.k1 = (unsigned)(key >> 32);
  if (shp.empty()) {  // a single element
    P.nd = 1;
    P.shape[0] = 1;
  } else {
    P.nd = (int)shp.size();
    for (int d = 0; d < P.nd; ++d) P.shape[d] = shp[d];
    for (int k = 0; k < n_params; ++k)
      for (int d = 0; d < P.nd; ++d) P.st[k][d] = st[k][d];
  }
  for (int k = 0; k < n_params; ++k) {
    if (!params[k]) return fail(AB_ERR_INVALID, "null parameter %d", k);
    P.p[k] = params[k];
  }
  P.vec = reinterpret_cast<uintptr_t>(out) % 16 == 0;
  if (check) {
    P.err = error_flag();
    if (!P.err) return fail(AB_ERR_CUDA, "cannot allocate the parameter-error flag");
  }
  const int e = dist == DIST_UNIFORM || dist == DIST_NORMAL ? (dtype == AB_F32 ? 4 : 2) : 4;
  P.blocks = (total + e - 1) / e;
  cudaStream_t st_ = as_stream(stream);
  int rc;
  if (dist == DIST_UNIFORM) rc = dtype == AB_F32 ? launch<DIST_UNIFORM, float>(P, out, st_) : launch<DIST_UNIFORM, double>(P, out, st_);
  else if (dist == DIST_NORMAL) rc = dtype == AB_F32 ? launch<DIST_NORMAL, float>(P, out, st_) : launch<DIST_NORMAL, double>(P, out, st_);
  else rc = launch<DIST_BERNOULLI, long long>(P, out, st_);
  if (rc || !check) return rc;
  int host = 0;
  AB_CUDA(cudaMemcpyAsync(&host, P.err, sizeof(int), cudaMemcpyDeviceToHost, st_));
  AB_CUDA(cudaStreamSynchronize(st_));
  if (host) {
    clear_flag_kernel<<<1, 1, 0, st_>>>(P.err);
    return fail(AB_ERR_INVALID, dist == DIST_NORMAL ? "scale < 0" : "p < 0, p > 1 or p is NaN");
  }
  return AB_OK;
}
