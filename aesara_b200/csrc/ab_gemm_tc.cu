// ab_gemm_tc.cu — float32 Gemm/Dot22 on the Hopper tensor cores (wgmma).
//
// Reference op: aesara/tensor/blas.py:872 Gemm / :1659 Dot22 (C template
// :518-869 dispatching to sgemm_ by stride case :765-776).  The reference is a
// true-fp32 sgemm, so the default mode here is fp32-faithful:
//
//   precision 0  3xTF32: each operand x is split into hi = tf32(x) and
//                lo = tf32(x - hi); D += Ahi*Bhi + Ahi*Blo + Alo*Bhi with FP32
//                accumulation over 128-element K segments that are summed
//                round-to-nearest (rtol 1e-5 holds at any K);
//   precision 1  one TF32 pass straight from the fp32 operands;
//   precision 2  BF16 operands, FP32 accumulation (the "bf16 compute policy"
//                of BASELINE config 3; stated looser rtol).
//
// Structure (one 128 x 128 output tile at a time per CTA, persistent, 512 threads):
//   warpgroup 0   TMA producer: cp.async.bulk.tensor 2-D loads of 128-byte-swizzled
//                 operand tiles into a multi-stage smem ring, completion on mbarriers
//                 (expect_tx);
//   warpgroups 1-2  wgmma.mma_async (M = 64 rows each, N = 128) from the ring into
//                 register accumulators, every finished K segment added into a running
//                 total in registers, stored once per tile into a float32 accumulator in
//                 shared memory;
//   warpgroup 3   epilogue: reads that accumulator with one row per lane, applies
//                 alpha/beta (or the fused region) and stores C with arbitrary strides,
//                 while warpgroups 1-2 run the next tile's main loop.
//
// Operands that are not K-major / 16-byte-pitched in global memory (the
// DimShuffle{1,0} views of the MLP backward pass, blas.py:719-726 "unit" cases)
// and every operand of modes 0 and 2 go through pack_kernel first, which
// writes the K-major hi/lo (or bf16) planes the tensor maps describe.
#include <cuda.h>
#include <cuda_bf16.h>

#include <algorithm>

#include "ab_common.h"
#include "ab_tc.cuh"

namespace ab {

namespace {

using namespace ab::tc;

#include "ab_gemm_tc_kernel.cuh"

template <int KIND, int CL>
__global__ void __launch_bounds__(kThreads, 1)
gemm_tc_kernel(const __grid_constant__ CUtensorMap map_a0,
               const __grid_constant__ CUtensorMap map_a1,
               const __grid_constant__ CUtensorMap map_b0,
               const __grid_constant__ CUtensorMap map_b1,
               const __grid_constant__ GemmParams p) {
  gemm_body<KIND, CL>(map_a0, map_a1, map_b0, map_b1, p);
}
// ------------------------------------------------------------------ operand packing
// out planes are [R, pitch] row-major (K-major): out[r*pitch + c] = f(in[r*s_r + c*s_c]).
// MODE 0: hi/lo tf32 split (two f32 planes), 1: f32 copy, 2: bf16.
// Fast path of the operand pack: the source is contiguous along the plane's column index
// (s_c == 1) with 16-byte aligned rows.  Each thread converts 8 consecutive elements
// (two 128-bit loads -> one 128-bit bf16 store, or 128-bit stores to the hi/lo planes);
// a pure streaming kernel instead of the 32 x 32 shared-memory transpose below.
template <int MODE>
__global__ void __launch_bounds__(256)
pack_rows_kernel(const float* __restrict__ in, long long R, long long Kc, long long s_r,
                 void* __restrict__ out0, void* __restrict__ out1, long long pitch) {
  const long long groups = Kc >> 3;  // groups of 8 columns per row (Kc % 8 == 0)
  const long long total = R * groups;
  for (long long g = (long long)blockIdx.x * 256 + threadIdx.x; g < total;
       g += (long long)gridDim.x * 256) {
    const long long r = g / groups, c = (g - r * groups) << 3;
    const float4 a = __ldcs(reinterpret_cast<const float4*>(in + r * s_r + c));
    const float4 b = __ldcs(reinterpret_cast<const float4*>(in + r * s_r + c + 4));
    const float v[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
    if (MODE == 2) {
      __nv_bfloat162 q[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) q[j] = __floats2bfloat162_rn(v[2 * j], v[2 * j + 1]);
      *reinterpret_cast<uint4*>(static_cast<__nv_bfloat16*>(out0) + r * pitch + c) =
          *reinterpret_cast<const uint4*>(q);
    } else if (MODE == 1) {
      float* o = static_cast<float*>(out0) + r * pitch + c;
      *reinterpret_cast<float4*>(o) = a;
      *reinterpret_cast<float4*>(o + 4) = b;
    } else {
      float hi[8], lo[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) tf32_split(v[j], hi[j], lo[j]);
      float* oh = static_cast<float*>(out0) + r * pitch + c;
      float* ol = static_cast<float*>(out1) + r * pitch + c;
      *reinterpret_cast<float4*>(oh) = make_float4(hi[0], hi[1], hi[2], hi[3]);
      *reinterpret_cast<float4*>(oh + 4) = make_float4(hi[4], hi[5], hi[6], hi[7]);
      *reinterpret_cast<float4*>(ol) = make_float4(lo[0], lo[1], lo[2], lo[3]);
      *reinterpret_cast<float4*>(ol + 4) = make_float4(lo[4], lo[5], lo[6], lo[7]);
    }
  }
}

template <int MODE>
__global__ void __launch_bounds__(256)
pack_kernel(const float* __restrict__ in, long long R, long long Kc, long long s_r, long long s_c,
            void* __restrict__ out0, void* __restrict__ out1, long long pitch) {
  __shared__ float tile[32][33];
  const long long r0 = (long long)blockIdx.y * 32, c0 = (long long)blockIdx.x * 32;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;  // 32 x 8
  const bool r_fast = (s_r == 1) || (s_c != 1 && llabs(s_r) < llabs(s_c));
#pragma unroll
  for (int i = 0; i < 32; i += 8) {
    long long r, c;
    if (r_fast) { r = r0 + tx; c = c0 + ty + i; } else { r = r0 + ty + i; c = c0 + tx; }
    float v = 0.0f;
    if (r < R && c < Kc) v = in[r * s_r + c * s_c];
    if (r_fast) tile[tx][ty + i] = v; else tile[ty + i][tx] = v;
  }
  __syncthreads();
#pragma unroll
  for (int i = 0; i < 32; i += 8) {
    const long long r = r0 + ty + i, c = c0 + tx;
    if (r < R && c < Kc) {
      const float v = tile[ty + i][tx];
      if (MODE == 0) {
        float hi, lo;
        tf32_split(v, hi, lo);
        static_cast<float*>(out0)[r * pitch + c] = hi;
        static_cast<float*>(out1)[r * pitch + c] = lo;
      } else if (MODE == 1) {
        static_cast<float*>(out0)[r * pitch + c] = v;
      } else {
        static_cast<__nv_bfloat16*>(out0)[r * pitch + c] = __float2bfloat16_rn(v);
      }
    }
  }
}

// ------------------------------------------------------------------ host side
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*,
                                  const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                  const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

EncodeTiledFn get_encode() {
  static EncodeTiledFn fn = nullptr;
  static bool tried = false;
  if (!tried) {
    tried = true;
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) == cudaSuccess &&
        qres == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(p);
    else
      cudaGetLastError();
  }
  return fn;
}

// tensor map over a plane whose contiguous ("inner") index has `inner` elements and whose
// rows are `pitch_elems` apart; box = {128 bytes of the inner index, box_outer rows}
int make_map(CUtensorMap* map, const void* base, bool bf16, long long inner, long long outer,
             long long pitch_elems, int box_outer) {
  EncodeTiledFn enc = get_encode();
  if (!enc) return fail(AB_ERR_CUDA, "cuTensorMapEncodeTiled is not available from the driver");
  const int es = bf16 ? 2 : 4;
  cuuint64_t dims[2] = {(cuuint64_t)inner, (cuuint64_t)outer};
  cuuint64_t strides[1] = {(cuuint64_t)pitch_elems * es};
  cuuint32_t box[2] = {(cuuint32_t)(SW_BYTES / es), (cuuint32_t)box_outer};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = enc(map, bf16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2,
                   const_cast<void*>(base), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                   CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return fail(AB_ERR_CUDA, "cuTensorMapEncodeTiled failed with code %d", (int)r);
  return AB_OK;
}

inline size_t align_up(size_t x, size_t a) { return (x + a - 1) / a * a; }

bool eligible(long long M, long long N, long long K) {
  return M >= 64 && N >= 64 && K >= 32 && (double)M * N * K >= (double)(1 << 21) &&
         M < (1LL << 31) && N < (1LL << 31) && K < (1LL << 31);
}

int sm_count() {
  static int sms = 0;
  if (!sms) {
    int dev = 0;
    cudaGetDevice(&dev);
    if (cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || sms <= 0)
      sms = 132;
  }
  return sms;
}

}  // namespace

// A GEMM operand in tensor-core form: logical [rows, k] (rows = M for A, N for B).
//   mn_major == 0: planes are [rows, pitch] with K contiguous;
//   mn_major == 1: planes are [k, pitch] with the M/N index contiguous.
// plane[1] is the tf32 "lo" plane of the 3xTF32 split (precision 0), else null.
struct PackedOperand {
  const void* plane[2];
  long long rows, k, pitch;
  int mn_major;
  int precision;
};

// Decide how the logical operand [rows, k] with element strides (s_r, s_k) is presented
// to the tensor cores.  `direct` = usable in place (precision 1 only: raw fp32, aligned).
static void plan_operand(int precision, long long rows, long long k, long long s_r, long long s_k,
                         const void* ptr, bool* direct, int* mn_major, long long* pitch,
                         size_t* plane_bytes, bool force_k = false) {
  const int es = precision == 2 ? 2 : 4;
  const bool aligned = (reinterpret_cast<uintptr_t>(ptr) % 16 == 0);
  if (s_k == 1 || k == 1) {
    *mn_major = 0;
    *direct = precision == 1 && aligned && (s_r % 4 == 0) && s_r >= k;
    *pitch = *direct ? s_r : (long long)align_up((size_t)k, 16 / es);
    *plane_bytes = *direct ? 0 : align_up((size_t)rows * (size_t)*pitch * es, 1024);
  } else if (s_r == 1 && precision == 2 && !force_k && getenv("AB_GEMM_NO_MN") == nullptr) {
    // MN-major is used for 16-bit operands only: a 32-bit (TF32) MN-major operand needs the
    // SWIZZLE_128B_BASE32B shared-memory layout (and the matching 32B-atom TMA swizzle);
    // TF32 operands that are not K-contiguous are gathered into a K-major plane below.
    *mn_major = 1;
    *direct = precision == 1 && aligned && (s_k % 4 == 0) && s_k >= rows;
    *pitch = *direct ? s_k : (long long)align_up((size_t)rows, 16 / es);
    *plane_bytes = *direct ? 0 : align_up((size_t)k * (size_t)*pitch * es, 1024);
  } else {  // doubly strided: gather into a K-major plane
    *mn_major = 0;
    *direct = false;
    *pitch = (long long)align_up((size_t)k, 16 / es);
    *plane_bytes = align_up((size_t)rows * (size_t)*pitch * es, 1024);
  }
}

size_t gemm_pack_bytes(int precision, long long rows, long long k, long long s_r, long long s_k,
                       bool force_k = false) {
  bool direct;
  int mn;
  long long pitch;
  size_t pb;
  plan_operand(precision, rows, k, s_r, s_k, reinterpret_cast<const void*>(1), &direct, &mn, &pitch, &pb,
               force_k);
  return (precision == 0 ? 2 : 1) * pb + 1024;
}

int gemm_pack(int precision, const float* src, long long rows, long long k, long long s_r,
              long long s_k, void* dst, size_t dst_bytes, PackedOperand* out, cudaStream_t st,
              bool force_k = false) {
  bool direct;
  int mn;
  long long pitch;
  size_t pb;
  plan_operand(precision, rows, k, s_r, s_k, src, &direct, &mn, &pitch, &pb, force_k);
  out->rows = rows; out->k = k; out->pitch = pitch; out->mn_major = mn; out->precision = precision;
  out->plane[0] = src; out->plane[1] = nullptr;
  if (direct) return AB_OK;
  const int parts = precision == 0 ? 2 : 1;
  uint8_t* ws = reinterpret_cast<uint8_t*>(align_up(reinterpret_cast<uintptr_t>(dst), 1024));
  if (!dst || ws + parts * pb > reinterpret_cast<uint8_t*>(dst) + dst_bytes)
    return fail(AB_ERR_INVALID, "Gemm pack buffer too small: need %zu bytes, have %zu",
                parts * pb + 1024, dst_bytes);
  void* o0 = ws;
  void* o1 = parts == 2 ? ws + pb : nullptr;
  // plane rows/cols: K-major plane is [rows, k]; MN-major plane is [k, rows]
  const long long R = mn ? k : rows, Cc = mn ? rows : k;
  const long long sr = mn ? s_k : s_r, sc = mn ? s_r : s_k;
  if (sc == 1 && Cc % 8 == 0 && sr % 4 == 0 && pitch % 8 == 0 &&
      (reinterpret_cast<uintptr_t>(src) & 15) == 0) {
    const long long total = R * (Cc / 8);
    const unsigned blocks = (unsigned)std::min<long long>((total + 255) / 256, (long long)sm_count() * 16);
    if (precision == 0) pack_rows_kernel<0><<<blocks, 256, 0, st>>>(src, R, Cc, sr, o0, o1, pitch);
    else if (precision == 1) pack_rows_kernel<1><<<blocks, 256, 0, st>>>(src, R, Cc, sr, o0, o1, pitch);
    else pack_rows_kernel<2><<<blocks, 256, 0, st>>>(src, R, Cc, sr, o0, o1, pitch);
    g_launches++;
    AB_CUDA(cudaGetLastError());
    out->plane[0] = o0;
    out->plane[1] = o1;
    return AB_OK;
  }
  dim3 grid((unsigned)((Cc + 31) / 32), (unsigned)((R + 31) / 32));
  if (grid.y > 65535) {
    // tall planes: fold the row-tile index into x instead (both are limited to 2^31-1 / 65535)
    return fail(AB_ERR_UNSUPPORTED, "gemm operand with more than 2M rows in the pack plane");
  }
  if (precision == 0) pack_kernel<0><<<grid, 256, 0, st>>>(src, R, Cc, sr, sc, o0, o1, pitch);
  else if (precision == 1) pack_kernel<1><<<grid, 256, 0, st>>>(src, R, Cc, sr, sc, o0, o1, pitch);
  else pack_kernel<2><<<grid, 256, 0, st>>>(src, R, Cc, sr, sc, o0, o1, pitch);
  g_launches++;
  AB_CUDA(cudaGetLastError());
  out->plane[0] = o0;
  out->plane[1] = o1;
  return AB_OK;
}

bool gemm_tc_eligible(long long M, long long N, long long K) { return eligible(M, N, K); }

// CTAs per cluster: 2 (gemm_body<KIND, 2>: two CTAs stacked along M share the B tile, each
// loading half of it by TMA multicast, so a k-block reads 24 KB from L2 per CTA instead of 32)
// for bf16 products of at least two tile rows that are not split along K; 1 otherwise.
// AB_GEMM_CLUSTER=1|2 forces the choice (probing knob).
int cluster_ctas(int precision, long long M, bool fused, int k_splits) {
  if (const char* env = getenv("AB_GEMM_CLUSTER")) return (atoi(env) == 2 && !fused) ? 2 : 1;
  return (precision == 2 && !fused && M >= 2 * BLOCK_M && k_splits == 1) ? 2 : 1;
}

// launch configuration of a persistent grid of `clusters` clusters of `ctas` CTAs; `attr`
// receives the cluster dimension and has to outlive the use of the result
cudaLaunchConfig_t cluster_config(int ctas, long long clusters, size_t smem, cudaStream_t st,
                                  cudaLaunchAttribute* attr) {
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3((unsigned)(ctas * clusters));
  cfg.blockDim = dim3(kThreads);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  attr->id = cudaLaunchAttributeClusterDimension;
  attr->val.clusterDim.x = ctas;
  attr->val.clusterDim.y = 1;
  attr->val.clusterDim.z = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  return cfg;
}

cudaError_t active_clusters(const void* kern, int ctas, size_t smem, int* n) {
  cudaLaunchAttribute attr;
  const cudaLaunchConfig_t cfg = cluster_config(ctas, sm_count() / ctas, smem, nullptr, &attr);
  return cudaOccupancyMaxActiveClusters(n, kern, &cfg);
}

// the ahead-of-time kernel of (bf16, CTAs per cluster), its dynamic shared memory limit raised
// on first use
int plain_kernel(bool bf16, int cl, const void** kern) {
  static const void* const kernels[2][2] = {
      {(const void*)gemm_tc_kernel<0, 1>, (const void*)gemm_tc_kernel<0, 2>},
      {(const void*)gemm_tc_kernel<1, 1>, (const void*)gemm_tc_kernel<1, 2>}};
  static bool raised[2][2] = {};
  *kern = kernels[bf16][cl - 1];
  if (!raised[bf16][cl - 1]) {
    AB_CUDA(cudaFuncSetAttribute(*kern, cudaFuncAttributeMaxDynamicSharedMemorySize, kMaxSmemGemm));
    raised[bf16][cl - 1] = true;
  }
  return AB_OK;
}

// how many clusters of `ctas` CTAs of this kernel can be resident at once (the persistent grid)
int max_clusters(const void* kern, int ctas, size_t smem) {
  int n = 0;
  if (active_clusters(kern, ctas, smem, &n) != cudaSuccess || n <= 0) {
    cudaGetLastError();
    n = sm_count() / ctas;
  }
  return std::min(n, sm_count() / ctas);
}

// ------------------------------------------------------------------------ split-K
// The persistent grid has one CTA per SM; a problem whose tile count is a little above a
// multiple of that leaves most of the last wave idle.  When K is long the K loop is cut into
// k_splits ranges, so the unit count fills the waves; range 0 writes C, ranges >= 1 write
// alpha * partial planes that splitk_reduce_kernel adds to C.
int plan_k_splits(int precision, long long M, long long N, long long K) {
  const char* env = getenv("AB_GEMM_SPLITK");  // 0/1 = off, n = force n ranges
  const long long tiles = ((M + BLOCK_M - 1) / BLOCK_M) * ((N + BLOCK_N - 1) / BLOCK_N);
  const long long groups = sm_count();
  const long long k_elems = SW_BYTES / (precision == 2 ? 2 : 4);
  const long long num_kb = (K + k_elems - 1) / k_elems;
  if (env) {
    const int f = atoi(env);
    return (int)std::max<long long>(1, std::min<long long>(f, num_kb));
  }
  if (num_kb < 128 || (double)M * (double)N > 64.0 * 1024 * 1024) return 1;
  auto eff = [&](long long s) {
    const long long units = tiles * s;
    return (double)units / (double)(((units + groups - 1) / groups) * groups);
  };
  int best = 1;
  double best_score = eff(1);
  for (int s = 2; s <= 8; ++s) {
    if (num_kb / s < 64) break;
    const double score = eff(s) * (1.0 - 0.01 * (s - 1));  // the partial planes are not free
    if (score > best_score * 1.05) { best = s; best_score = score; }
  }
  return best;
}

size_t gemm_splitk_bytes(int precision, long long M, long long N, long long K) {
  const int s = plan_k_splits(precision, M, N, K);
  return s > 1 ? (size_t)(s - 1) * (size_t)M * (size_t)N * sizeof(float) + 256 : 0;
}

__global__ void __launch_bounds__(256)
splitk_reduce_kernel(float* __restrict__ C, long long c_rs, long long c_cs,
                     const float* __restrict__ partial, long long M, long long N, int planes) {
  const bool vec = c_cs == 1 && (N & 3) == 0 && (c_rs & 3) == 0 && (reinterpret_cast<uintptr_t>(C) & 15) == 0;
  if (vec) {
    const long long n4 = N >> 2, total = M * n4;
    for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < total; i += (long long)gridDim.x * 256) {
      const long long r = i / n4, c = (i - r * n4) << 2;
      float4 v = *reinterpret_cast<const float4*>(C + r * c_rs + c);
      for (int s = 0; s < planes; ++s) {
        const float4 q = __ldcs(reinterpret_cast<const float4*>(partial + ((long long)s * M + r) * N + c));
        v.x += q.x; v.y += q.y; v.z += q.z; v.w += q.w;
      }
      *reinterpret_cast<float4*>(C + r * c_rs + c) = v;
    }
  } else {
    const long long total = M * N;
    for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < total; i += (long long)gridDim.x * 256) {
      const long long r = i / N, c = i - r * N;
      float v = C[r * c_rs + c * c_cs];
      for (int s = 0; s < planes; ++s) v += partial[((long long)s * M + r) * N + c];
      C[r * c_rs + c * c_cs] = v;
    }
  }
}

// Fused consumer (see ab_gemm_tc_kernel.cuh / codegen/gemm_epilogue.py): the NVRTC
// module holding the AB_EPILOGUE build of the kernels, its memory operands and the
// optional bf16 shadow plane.
struct EpilogueSpec {
  Module* module = nullptr;
  int nops = 0;
  const float* ptr[4] = {};
  long long rs[4] = {}, cs[4] = {};
  int nout = 1;
  float* out_ptr[3] = {};      // values 1.. (value 0 goes to C)
  long long out_rs[3] = {};
  void* shadow[3] = {};
  long long shadow_pitch[3] = {};
  void* shadow_t = nullptr;    // transposed bf16 plane of the module's AB_EP_TPLANE value, [N, pitch]
  long long shadow_t_pitch = 0;
  double* colsum_ws = nullptr;
  double* fullsum_ws = nullptr;
};

int fused_kernel(Module* m, const char* name, cudaKernel_t* out) {
  auto it = m->named.find(name);
  if (it != m->named.end()) { *out = it->second; return AB_OK; }
  cudaKernel_t kern = nullptr;
  if (cudaLibraryGetKernel(&kern, m->lib, name) != cudaSuccess) {
    cudaGetLastError();
    return fail(AB_ERR_INVALID, "fused GEMM module has no kernel %s", name);
  }
  cudaError_t e = cudaFuncSetAttribute((const void*)kern, cudaFuncAttributeMaxDynamicSharedMemorySize, kMaxSmemGemm);
  if (e != cudaSuccess) {
    cudaGetLastError();
    return fail(AB_ERR_CUDA, "cannot raise the dynamic shared memory limit of %s: %s", name, cudaGetErrorString(e));
  }
  m->named[name] = kern;
  *out = kern;
  return AB_OK;
}

int splitk_finish(const GemmParams& p, cudaStream_t st) {
  if (p.k_splits <= 1) return AB_OK;
  const long long work = (p.M * p.N + 3) / 4;
  const unsigned blocks = (unsigned)std::min<long long>((work + 255) / 256, (long long)sm_count() * 16);
  splitk_reduce_kernel<<<blocks, 256, 0, st>>>(p.C, p.c_rs, p.c_cs, p.partial, p.M, p.N, p.k_splits - 1);
  g_launches++;
  AB_CUDA(cudaGetLastError());
  return AB_OK;
}

int gemm_run(int precision, long long M, long long N, long long K, float alpha,
             const PackedOperand& A, const PackedOperand& B, float beta, float* C, long long c_rs,
             long long c_cs, cudaStream_t st, const float* Cin = nullptr, long long cin_rs = 0,
             long long cin_cs = 0, void* splitk_ws = nullptr, size_t splitk_bytes = 0,
             const EpilogueSpec* ep = nullptr) {
  if (precision < 0 || precision > 2) return fail(AB_ERR_INVALID, "bad gemm precision %d", precision);
  if (A.precision != precision || B.precision != precision || A.rows != M || B.rows != N ||
      A.k != K || B.k != K)
    return fail(AB_ERR_INVALID, "packed operands do not match the gemm call");
  const int parts = precision == 0 ? 2 : 1;
  const bool bf16 = precision == 2;
  const int es = bf16 ? 2 : 4;
  GemmParams p{};
  p.M = M; p.N = N; p.K = K;
  p.alpha = alpha; p.beta = beta;
  p.C = C; p.c_rs = c_rs; p.c_cs = c_cs;
  p.Cin = Cin ? Cin : C; p.cin_rs = Cin ? cin_rs : c_rs; p.cin_cs = Cin ? cin_cs : c_cs;
  // a fused epilogue may leave C unwritten (C == nullptr); beta*C_in then needs its own matrix
  if (beta != 0.0f && !p.Cin) return fail(AB_ERR_INVALID, "beta != 0 needs C_in (or C)");
  p.block_n = BLOCK_N;
  p.nparts = parts;
  p.k_elems_per_row = SW_BYTES / es;          // K elements per stage (64 bf16 / 32 tf32)
  p.a_tile_bytes = BLOCK_M * SW_BYTES;
  p.b_tile_bytes = p.block_n * SW_BYTES;
  p.a_mn = A.mn_major; p.b_mn = B.mn_major;
  p.mn_per_chunk = SW_BYTES / es;
  p.chunk_bytes = p.k_elems_per_row * SW_BYTES;
  p.a_chunks = BLOCK_M / p.mn_per_chunk;
  p.b_chunks = p.block_n / p.mn_per_chunk;
  const int mma_k = 32 / es;                   // K per instruction: 16 (bf16) / 8 (tf32)
  p.a_kstep = A.mn_major ? mma_k * SW_BYTES : 32;
  p.b_kstep = B.mn_major ? mma_k * SW_BYTES : 32;
  const int stage_bytes = parts * (p.a_tile_bytes + p.b_tile_bytes);
  const int stage_reserve = kAccBytes + (ep ? kStageBytes : 0);  // the fused epilogue's staging chunks
  p.stages = std::max(2, std::min(8, (kMaxSmemGemm - 1024 - stage_reserve) / stage_bytes));
  if (const char* st_env = getenv("AB_GEMM_STAGES"))  // probing knob
    p.stages = std::max(2, std::min(p.stages, atoi(st_env)));
  {
    // L2 priority of the operands (GemmParams::a_l2): a small operand that every tile row (or
    // column) of the other one re-reads -- the weight matrix of a batched layer -- is kept in L2
    static const bool no_hint = getenv("AB_GEMM_NO_L2_HINT") != nullptr;
    const double a_bytes = (double)M * (double)K * es * parts, b_bytes = (double)N * (double)K * es * parts;
    const double keep_max = 48.0 * 1024 * 1024;
    if (!no_hint) {
      if (b_bytes <= keep_max && a_bytes >= 4.0 * b_bytes) p.b_l2 = 2;
      else if (a_bytes <= keep_max && b_bytes >= 4.0 * a_bytes) p.a_l2 = 2;
    }
  }
  {
    // K segments (see "segments" in ab_gemm_tc_kernel.cuh): 4 k-blocks = 128 K elements for
    // the fp32-faithful mode, 16 for the others; AB_GEMM_SEG_KB overrides (0 = never fold, the
    // whole K loop stays in registers)
    static const char* seg_env = getenv("AB_GEMM_SEG_KB");
    const int num_kb = (int)((K + p.k_elems_per_row - 1) / p.k_elems_per_row);
    // split-K only with a scratch buffer from the caller (else one K range: still correct)
    p.k_splits = 1;
    const int want = ep ? 1 : plan_k_splits(precision, M, N, K);  // partial sums cannot be post-processed
    if (want > 1 && splitk_ws && splitk_bytes >= (size_t)(want - 1) * (size_t)M * (size_t)N * sizeof(float) + 256)
      p.k_splits = want;
    p.kb_per_split = (num_kb + p.k_splits - 1) / p.k_splits;
    int seg = precision == 0 ? 4 : 16;
    if (seg_env) seg = atoi(seg_env) > 0 ? atoi(seg_env) : p.kb_per_split;
    p.seg_kblocks = std::max(1, std::min(seg, std::max(1, p.kb_per_split)));
    if (p.k_splits > 1) {
      // whole segments per range, and no empty range
      p.kb_per_split = (p.kb_per_split + p.seg_kblocks - 1) / p.seg_kblocks * p.seg_kblocks;
      p.k_splits = (num_kb + p.kb_per_split - 1) / p.kb_per_split;
    }
    p.partial = reinterpret_cast<float*>((reinterpret_cast<uintptr_t>(splitk_ws) + 255) & ~(uintptr_t)255);
  }
  if (ep) {
    if (ep->nops < 0 || ep->nops > 4) return fail(AB_ERR_INVALID, "fused epilogue takes at most 4 operands");
    for (int k = 0; k < ep->nops; ++k) {
      if (!ep->ptr[k]) return fail(AB_ERR_INVALID, "null fused-epilogue operand");
      if (ep->cs[k] == 1 && ((reinterpret_cast<uintptr_t>(ep->ptr[k]) & 15) || (ep->rs[k] & 3)))
        return fail(AB_ERR_UNSUPPORTED, "fused-epilogue operand %d is not 16-byte aligned", k);
      p.ep_ptr[k] = ep->ptr[k]; p.ep_rs[k] = ep->rs[k]; p.ep_cs[k] = ep->cs[k];
    }
    if (ep->nout < 1 || ep->nout > 3) return fail(AB_ERR_INVALID, "fused epilogue yields 1..3 values");
    // the fused epilogue moves 8 columns at a time (ab_gemm_tc_kernel.cuh, fused_eval)
    if (N % 8) return fail(AB_ERR_UNSUPPORTED, "fused epilogue needs N %% 8 == 0");
    if (C && (c_cs != 1 || (c_rs & 3) || (reinterpret_cast<uintptr_t>(C) & 15)))
      return fail(AB_ERR_UNSUPPORTED, "fused epilogue needs a row-contiguous, 16-byte aligned C");
    if (beta != 0.0f && (p.cin_cs != 1 || (p.cin_rs & 3) || (reinterpret_cast<uintptr_t>(p.Cin) & 15)))
      return fail(AB_ERR_UNSUPPORTED, "fused epilogue needs a row-contiguous, 16-byte aligned Cin");
    for (int k = 0; k < 3; ++k)
      if (ep->shadow[k] && ((reinterpret_cast<uintptr_t>(ep->shadow[k]) & 15) || (ep->shadow_pitch[k] & 7)))
        return fail(AB_ERR_UNSUPPORTED, "bf16 shadow plane rows are not 16-byte aligned");
    for (int k = 0; k < 3; ++k) {
      if (ep->shadow[k] && ((reinterpret_cast<uintptr_t>(ep->shadow[k]) & 7) || (ep->shadow_pitch[k] & 3)))
        return fail(AB_ERR_UNSUPPORTED, "bf16 shadow plane is not 8-byte aligned");
      if (ep->out_ptr[k] && ((reinterpret_cast<uintptr_t>(ep->out_ptr[k]) & 15) || (ep->out_rs[k] & 3)))
        return fail(AB_ERR_UNSUPPORTED, "extra epilogue output %d is not 16-byte aligned", k);
      p.shadow[k] = ep->shadow[k]; p.shadow_pitch[k] = ep->shadow_pitch[k];
      p.out_ptr[k] = ep->out_ptr[k]; p.out_rs[k] = ep->out_rs[k];
    }
    if (ep->shadow_t && ((reinterpret_cast<uintptr_t>(ep->shadow_t) & 15) || (ep->shadow_t_pitch & 7) ||
                         ep->shadow_t_pitch < M))
      return fail(AB_ERR_UNSUPPORTED, "transposed bf16 shadow plane rows are not 16-byte aligned / too short");
    p.shadow_t = ep->shadow_t;
    p.shadow_t_pitch = ep->shadow_t_pitch;
    p.colsum_ws = ep->colsum_ws;
    p.fullsum_ws = ep->fullsum_ws;
    p.fullsum_cols = 2 * ((N + p.block_n - 1) / p.block_n);
  } else if (!C) {
    return fail(AB_ERR_INVALID, "null output matrix");
  }
  CUtensorMap ma[2], mb[2];
  int rc;
  // same arithmetic per output element in a pair, so the same result bit for bit
  const int cl = cluster_ctas(precision, M, ep != nullptr, p.k_splits);
  {
    // Unit order inside a K range (AB_UNIT_DECODE): groups of 8 tile rows (4 pair rows),
    // columns outer, so that the units in flight share A and B panels in L2.  A tall tile grid
    // always takes it; a square bf16 one once it has more tiles than the persistent grid has
    // CTAs.  There, in row order, a wave of 132 CTAs over 32 x 32 tiles reads 5 A and 32 B
    // panels (16 MB each at the weight gradients' K = 65536), in groups of 8 rows 8 A and 17 B
    // panels.  Groups of 11 (11 + 12 panels) measured slower than 8 on those products, and the
    // 3xTF32 weight gradients measured slower grouped than in row order.
    const char* gm_env = getenv("AB_GEMM_GROUP_M");  // probing knob, in rows of cluster tiles
    const long long tm = (M + BLOCK_M - 1) / BLOCK_M, tn = (N + BLOCK_N - 1) / BLOCK_N;
    p.group_m = (tm >= 4 * tn || (precision == 2 && tm * tn > sm_count())) ? 8 / cl : 1;
    if (gm_env) p.group_m = std::max(1, atoi(gm_env));
  }
  for (int i = 0; i < parts; ++i) {
    if (A.mn_major) rc = make_map(&ma[i], A.plane[i], bf16, M, K, A.pitch, p.k_elems_per_row);
    else rc = make_map(&ma[i], A.plane[i], bf16, K, M, A.pitch, BLOCK_M);
    if (rc) return rc;
    if (B.mn_major) rc = make_map(&mb[i], B.plane[i], bf16, N, K, B.pitch, p.k_elems_per_row / cl);
    else rc = make_map(&mb[i], B.plane[i], bf16, K, N, B.pitch, p.block_n / cl);
    if (rc) return rc;
  }
  if (parts == 1) { ma[1] = ma[0]; mb[1] = mb[0]; }
  const size_t smem = (size_t)p.stages * stage_bytes + 1024 + stage_reserve;
  p.stage_bytes = stage_bytes;
  p.num_k_blocks = (int)((K + p.k_elems_per_row - 1) / p.k_elems_per_row);
  p.tiles_n = (N + p.block_n - 1) / p.block_n;
  p.num_tiles = ((M + (long long)cl * BLOCK_M - 1) / ((long long)cl * BLOCK_M)) * p.tiles_n;
  p.num_units = p.num_tiles * p.k_splits;
  const long long num_units = p.num_units;
  void* args[] = {&ma[0], &ma[1], &mb[0], &mb[1], &p};
  if (ep) {
    // one entry point per MMA-loop layout (ab_gemm_tc_kernel.cuh, AB_EP_KERNEL)
    static const char* const f16_names[4] = {"ab_gemm_ep_f16", "ab_gemm_ep_f16_km", "ab_gemm_ep_f16_mk",
                                             "ab_gemm_ep_f16_mm"};
    const char* name = bf16 ? f16_names[2 * p.a_mn + p.b_mn] : (parts == 2 ? "ab_gemm_ep_tf32" : "ab_gemm_ep_tf32_1p");
    cudaKernel_t kern;
    if ((rc = fused_kernel(ep->module, name, &kern))) return rc;
    dim3 grid((unsigned)std::min<long long>(num_units, sm_count()));  // persistent: one CTA per SM
    AB_CUDA(cudaLaunchKernel((const void*)kern, grid, dim3(kThreads), args, smem, st));
    g_launches++;
    return AB_OK;
  }
  const void* kern;
  if ((rc = plain_kernel(bf16, cl, &kern))) return rc;
  // persistent: one cluster per SM (cl = 1), or as many pairs as fit at once (asked once per kernel)
  static int resident[2] = {0, 0};
  int& res = resident[bf16];
  if (cl > 1 && !res) res = max_clusters(kern, cl, smem);
  cudaLaunchAttribute attr;
  cudaLaunchConfig_t cfg =
      cluster_config(cl, std::min<long long>(num_units, cl > 1 ? res : sm_count()), smem, st, &attr);
  // Single CTAs are launched without the attribute: a cluster dimension of 1 is still a cluster
  // launch, which places the CTAs on the SMs in another order, and the units in flight
  // (AB_UNIT_DECODE) then share less in L2 (measured on an H100 80GB HBM3, 700 W, at the cfg3
  // shapes: the bf16 single-CTA kernel ran at 345 instead of 425 TFLOP/s).
  if (cl == 1) cfg.numAttrs = 0;
  AB_CUDA(cudaLaunchKernelExC(&cfg, kern, args));
  g_launches++;
  return splitk_finish(p, st);
}

size_t gemm_tc_workspace(int precision, long long M, long long N, long long K, long long a_rs,
                              long long a_cs, long long b_rs, long long b_cs) {
  if (!eligible(M, N, K)) return 0;
  return gemm_pack_bytes(precision, M, K, a_rs, a_cs) + gemm_pack_bytes(precision, N, K, b_cs, b_rs);
}

int gemm_tc_f32(int precision, long long M, long long N, long long K, float alpha,
                     const float* A, long long a_rs, long long a_cs, const float* B, long long b_rs,
                     long long b_cs, float beta, float* C, long long c_rs, long long c_cs,
                     void* workspace, size_t workspace_bytes, cudaStream_t st, bool* handled) {
  *handled = false;
  if (precision < 0 || precision > 2) return fail(AB_ERR_INVALID, "bad gemm precision %d", precision);
  if (!eligible(M, N, K)) return AB_OK;
  *handled = true;
  PackedOperand pa{}, pb{};
  const size_t a_bytes = gemm_pack_bytes(precision, M, K, a_rs, a_cs);
  uint8_t* ws = static_cast<uint8_t*>(workspace);
  int rc = gemm_pack(precision, A, M, K, a_rs, a_cs, ws, std::min(a_bytes, workspace_bytes), &pa, st);
  if (rc) return rc;
  const size_t rest = workspace_bytes > a_bytes ? workspace_bytes - a_bytes : 0;
  rc = gemm_pack(precision, B, N, K, b_cs, b_rs, ws ? ws + a_bytes : nullptr, rest, &pb, st);
  if (rc) return rc;
  return gemm_run(precision, M, N, K, alpha, pa, pb, beta, C, c_rs, c_cs, st);
}

}  // namespace ab

// ---- C ABI for callers that keep packed operands across several products -------------
static int pack_bytes_abi(int precision, int64_t rows, int64_t k, int64_t s_r, int64_t s_k, size_t* bytes,
                          bool force_k) {
  if (!bytes) return ab::fail(AB_ERR_INVALID, "null out pointer");
  *bytes = ab::gemm_pack_bytes(precision, rows, k, s_r, s_k, force_k);
  return AB_OK;
}

static ab::PackedOperand from_abi(const ab_gemm_operand& o) {
  return ab::PackedOperand{{o.plane0, o.plane1}, o.rows, o.k, o.pitch, o.mn_major, o.precision};
}

static void to_abi(const ab::PackedOperand& po, ab_gemm_operand* out) {
  out->plane0 = po.plane[0]; out->plane1 = po.plane[1];
  out->rows = po.rows; out->k = po.k; out->pitch = po.pitch;
  out->mn_major = po.mn_major; out->precision = po.precision;
}

static int pack_abi(int precision, const void* src, int64_t rows, int64_t k, int64_t s_r, int64_t s_k,
                    void* dst, size_t dst_bytes, ab_gemm_operand* out, void* stream, bool force_k) {
  if (!out) return ab::fail(AB_ERR_INVALID, "null ab_gemm_operand");
  ab::PackedOperand po{};
  int rc = ab::gemm_pack(precision, static_cast<const float*>(src), rows, k, s_r, s_k, dst,
                         dst_bytes, &po, ab::as_stream(stream), force_k);
  if (rc) return rc;
  to_abi(po, out);
  return AB_OK;
}

extern "C" int ab_gemm_pack_bytes(int precision, int64_t rows, int64_t k, int64_t s_r, int64_t s_k,
                                  size_t* bytes) {
  return pack_bytes_abi(precision, rows, k, s_r, s_k, bytes, false);
}

extern "C" int ab_gemm_pack(int precision, const void* src, int64_t rows, int64_t k, int64_t s_r,
                            int64_t s_k, void* dst, size_t dst_bytes, ab_gemm_operand* out,
                            void* stream) {
  return pack_abi(precision, src, rows, k, s_r, s_k, dst, dst_bytes, out, stream, false);
}

// The same with the planes forced K-major ([rows, pitch], K contiguous) whatever the strides:
// a view that is contiguous along its rows (the transpose of a row-major matrix) is turned
// while it is packed.  For small matrices (weights) that are read with the contraction along
// their rows: the tensor cores read a K-major operand at full rate, and a tf32 operand can
// only be read K-major.
extern "C" int ab_gemm_pack_kmajor_bytes(int precision, int64_t rows, int64_t k, int64_t s_r,
                                         int64_t s_k, size_t* bytes) {
  return pack_bytes_abi(precision, rows, k, s_r, s_k, bytes, true);
}

extern "C" int ab_gemm_pack_kmajor(int precision, const void* src, int64_t rows, int64_t k,
                                   int64_t s_r, int64_t s_k, void* dst, size_t dst_bytes,
                                   ab_gemm_operand* out, void* stream) {
  return pack_abi(precision, src, rows, k, s_r, s_k, dst, dst_bytes, out, stream, true);
}

extern "C" int ab_gemm_packed(int precision, int64_t m, int64_t n, int64_t k, double alpha,
                              const ab_gemm_operand* A, const ab_gemm_operand* B, double beta,
                              const void* Cin, int64_t cin_rs, int64_t cin_cs, void* C,
                              int64_t c_rs, int64_t c_cs, void* workspace, size_t workspace_bytes,
                              void* stream) {
  if (!A || !B) return ab::fail(AB_ERR_INVALID, "null packed operand");
  if (!ab::gemm_tc_eligible(m, n, k))
    return ab::fail(AB_ERR_UNSUPPORTED, "problem too small for the tensor-core path; use ab_gemm");
  const ab::PackedOperand pa = from_abi(*A), pb = from_abi(*B);
  return ab::gemm_run(precision, m, n, k, (float)alpha, pa, pb, (float)beta, static_cast<float*>(C),
                      c_rs, c_cs, ab::as_stream(stream), static_cast<const float*>(Cin), cin_rs,
                      cin_cs, workspace, workspace_bytes);
}

extern "C" int ab_gemm_packed_fused(int precision, int64_t m, int64_t n, int64_t k, double alpha,
                                    const ab_gemm_operand* A, const ab_gemm_operand* B, double beta,
                                    const void* Cin, int64_t cin_rs, int64_t cin_cs, void* C,
                                    int64_t c_rs, int64_t c_cs, const ab_gemm_epilogue* ep,
                                    void* stream) {
  if (!A || !B || !ep || !ep->module) return ab::fail(AB_ERR_INVALID, "null argument");
  if (!ab::gemm_tc_eligible(m, n, k))
    return ab::fail(AB_ERR_UNSUPPORTED, "problem too small for the tensor-core path");
  const ab::PackedOperand pa = from_abi(*A), pb = from_abi(*B);
  ab::EpilogueSpec spec;
  spec.module = reinterpret_cast<ab::Module*>(ep->module);
  spec.nops = ep->n_operands;
  for (int i = 0; i < 4; ++i) {
    spec.ptr[i] = static_cast<const float*>(ep->ptr[i]);
    spec.rs[i] = ep->rs[i];
    spec.cs[i] = ep->cs[i];
  }
  spec.nout = ep->n_outputs;
  for (int i = 0; i < 3; ++i) {
    spec.out_ptr[i] = static_cast<float*>(ep->out_f32[i]);
    spec.out_rs[i] = ep->out_rs[i];
    spec.shadow[i] = ep->shadow_bf16[i];
    spec.shadow_pitch[i] = ep->shadow_pitch[i];
  }
  spec.shadow_t = ep->shadow_t_bf16;
  spec.shadow_t_pitch = ep->shadow_t_pitch;
  spec.colsum_ws = static_cast<double*>(ep->colsum_ws);
  spec.fullsum_ws = static_cast<double*>(ep->fullsum_ws);
  return ab::gemm_run(precision, m, n, k, (float)alpha, pa, pb, (float)beta, static_cast<float*>(C),
                      c_rs, c_cs, ab::as_stream(stream), static_cast<const float*>(Cin), cin_rs,
                      cin_cs, nullptr, 0, &spec);
}

extern "C" int ab_gemm_fused_layout(int64_t m, int64_t n, int64_t* row_blocks, int64_t* fullsum_cols) {
  if (!row_blocks || !fullsum_cols) return ab::fail(AB_ERR_INVALID, "null out pointer");
  *row_blocks = (m + 31) / 32;
  *fullsum_cols = 2 * ((n + ab::BLOCK_N - 1) / ab::BLOCK_N);
  return AB_OK;
}

extern "C" int ab_gemm_packed_workspace_bytes(int precision, int64_t m, int64_t n, int64_t k,
                                              size_t* bytes) {
  if (!bytes) return ab::fail(AB_ERR_INVALID, "null out pointer");
  *bytes = ab::gemm_tc_eligible(m, n, k) ? ab::gemm_splitk_bytes(precision, m, n, k) : 0;
  return AB_OK;
}

extern "C" int ab_gemm_tensorcore_eligible(int64_t m, int64_t n, int64_t k) {
  return ab::gemm_tc_eligible(m, n, k) ? 1 : 0;
}

extern "C" int ab_gemm_max_clusters(int precision, int ctas, int* clusters) {
  if (!clusters) return ab::fail(AB_ERR_INVALID, "null out pointer");
  if (ctas < 1 || ctas > 8) return ab::fail(AB_ERR_INVALID, "cluster of %d CTAs", ctas);
  const void* kern;
  if (int rc = ab::plain_kernel(precision == 2, 2, &kern)) return rc;
  AB_CUDA(ab::active_clusters(kern, ctas, ab::kMaxSmemGemm, clusters));
  return AB_OK;
}
