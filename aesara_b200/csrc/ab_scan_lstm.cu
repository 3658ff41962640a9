// ab_scan_lstm.cu — Scan fast path: an LSTM-cell recurrence as ONE persistent kernel.
//
// Reference: aesara/scan/op.py:637 (Scan), loop :1799-2103 — for every step the
// reference calls an inner compiled function (Gemm + four column-slice Subtensors + two
// fused Elemwise nodes, SURVEY.md App. A.4) from a Python/Cython loop.  When
// runtime/scan.py recognises that inner graph
//     pre = x_t + h_{t-1} @ U                      (Gemm, alpha = beta = 1)
//     c_t = sigmoid(pre_f) * c_{t-1} + sigmoid(pre_i) * tanh(pre_g)
//     h_t = sigmoid(pre_o) * tanh(c_t)              (gate order i, f, o, g)
// the whole T-step loop runs here without returning to the host:
//
//   * the grid is one CTA per SM (cooperative launch, all CTAs co-resident); every step
//     the [B, 4H] pre-activation is produced as 64 x 256 wgmma tiles (3xTF32,
//     fp32-faithful like ab_gemm) whose 256 columns are the four gates of 64 hidden units
//     (U is packed once with its columns gate-interleaved);
//   * the LSTM cell is the tile's epilogue, in the accumulator registers: x_t and
//     c_{t-1} are read once, c_t / h_t are written to the Scan's circular output buffers
//     and h_t is ALSO written as the hi/lo TF32 planes the next step's TMA loads — the
//     pre-activations never touch HBM and there is no per-step pack or copy kernel;
//     K is accumulated in 256-element segments (fresh register accumulator each, summed
//     in FP32) because the tensor core's own accumulate truncates;
//   * there is no barrier between steps.  Batch rows are independent, so a tile of step
//     t+1 only needs the h_t rows of ITS row block: every finished tile is counted on its
//     row block (release: bar.sync of the epilogue warps, __threadfence, atomicAdd) and the
//     TMA producer of a step-t+1 tile waits until all tiles of that row block are counted
//     (acquire load, then fence.proxy.async before the loads).  The h planes are double
//     buffered by step parity; a step-t+1 tile overwrites rows that only step-t tiles of
//     the same row block read, and those are complete by then.
//
// State lives in L2 (h planes 2 x 2 x B x H x 4 B, c in the output ring): 8192 x 1024
// state rows do not fit the register file / shared memory of the SMs.
#include <cooperative_groups.h>

#include <algorithm>
#include <cstdio>
#include <vector>

#include "ab_common.h"
#include "ab_tc.cuh"

namespace ab {

namespace {

using namespace ab::tc;

// ---- the ahead-of-time member of the family: the LSTM cell of BASELINE config 4 ----------
// gates (i, f, o, g) = pre[:, 0:H], [H:2H], [2H:3H], [3H:4H]; states (h, c).  Products are
// rounded on their own (no FMA contraction), as in the generated cells (codegen/scan_cell.py).
#define AB_CELL_GATES 4
#define AB_CELL_STATES 2
#define AB_CELL_EVAL(G, P, O)                                                                           \
  {                                                                                                     \
    (O)[1] = __fmul_rn(sigmoidf_ref((G)[1]), (P)[1]) + __fmul_rn(sigmoidf_ref((G)[0]), tanhf((G)[3])); \
    (O)[0] = __fmul_rn(sigmoidf_ref((G)[2]), tanhf((O)[1]));                                           \
  }
#include "ab_scan_cell_kernel.cuh"

__global__ void __launch_bounds__(kCellThreads, 1)
lstm_scan_kernel(const __grid_constant__ CUtensorMap map_h00, const __grid_constant__ CUtensorMap map_h01,
                 const __grid_constant__ CUtensorMap map_h10, const __grid_constant__ CUtensorMap map_h11,
                 const __grid_constant__ CUtensorMap map_u0, const __grid_constant__ CUtensorMap map_u1,
                 const __grid_constant__ CellParams p) {
  cell_scan_body(map_h00, map_h01, map_h10, map_h11, map_u0, map_u1, p);
}

// hi/lo TF32 planes of a [R, K] row-major-able matrix; rows optionally gate-interleaved:
// plane row n' = tile*(G*64) + gate*64 + u  <-  source column gate*H + tile*64 + u of U[K, G*H]
__global__ void __launch_bounds__(256)
split_planes_kernel(const float* __restrict__ src, long long R, long long K, long long s_r,
                    long long s_k, int interleave_h, int gates, float* __restrict__ hi,
                    float* __restrict__ lo) {
  const long long i = (long long)blockIdx.x * 256 + threadIdx.x;
  if (i >= R * K) return;
  const long long r = i / K, k = i - r * K;
  long long rs = r;
  if (interleave_h > 0) {
    const long long tile_n = (long long)gates * CELL_UNITS;
    const long long tile = r / tile_n, rem = r % tile_n;
    const long long gate = rem / CELL_UNITS, u = rem % CELL_UNITS;
    rs = gate * interleave_h + tile * CELL_UNITS + u;
  }
  const float v = src[rs * s_r + k * s_k];
  uint32_t hb, lb;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(hb) : "f"(v));
  const float h = __uint_as_float(hb);
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(lb) : "f"(v - h));
  hi[i] = h;
  lo[i] = __uint_as_float(lb);
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*,
                                  const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                  const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

int make_map_f32(CUtensorMap* map, const void* base, long long k, long long rows, int box_rows) {
  static EncodeTiledFn enc = nullptr;
  if (!enc) {
    void* fp = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fp, cudaEnableDefault, &qres) != cudaSuccess ||
        qres != cudaDriverEntryPointSuccess)
      return fail(AB_ERR_CUDA, "cuTensorMapEncodeTiled is not available from the driver");
    enc = reinterpret_cast<EncodeTiledFn>(fp);
  }
  cuuint64_t dims[2] = {(cuuint64_t)k, (cuuint64_t)rows};
  cuuint64_t strides[1] = {(cuuint64_t)k * 4};
  cuuint32_t box[2] = {(cuuint32_t)CELL_KB, (cuuint32_t)box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = enc(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<void*>(base), dims, strides, box,
                   estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                   CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return fail(AB_ERR_CUDA, "cuTensorMapEncodeTiled failed with code %d", (int)r);
  return AB_OK;
}

inline size_t align_up(size_t x, size_t a) { return (x + a - 1) / a * a; }
inline size_t row_flag_bytes(long long b) { return align_up((size_t)((b + CELL_BLOCK_M - 1) / CELL_BLOCK_M) * 4, 256); }

}  // namespace
}  // namespace ab

using namespace ab;

namespace {

size_t cell_ws_bytes(int gates, long long b, long long h) {
  const size_t hp = align_up((size_t)b * h * 4, 1024);
  const size_t up = align_up((size_t)gates * h * h * 4, 1024);
  return 4 * hp + 2 * up + 1024 + row_flag_bytes(b);
}

bool cell_supported(int gates, int states, long long t, long long b, long long h) {
  return gates >= 1 && gates <= 4 && states >= 1 && states <= 3 && t >= 1 && b >= 1 && h >= CELL_UNITS &&
         h % CELL_UNITS == 0 && b < (1LL << 31) && h < (1LL << 29) && t * (h / CELL_UNITS) * 2 < (1LL << 31);
}

// kern: the ahead-of-time LSTM kernel, or the kernel of an NVRTC module for a generated cell
int cell_scan_launch(const void* kern, int gates, int states, int hs, int64_t T,
                     int64_t B, int64_t H, const void* x, int64_t x_ts, int64_t x_rs, const void* U,
                     int64_t u_rs, int64_t u_cs, void* const* bufs, const int64_t* lens,
                     const int64_t* pos, void* workspace, size_t workspace_bytes, cudaStream_t st) {
  if (!cell_supported(gates, states, T, B, H)) return fail(AB_ERR_UNSUPPORTED, "Scan cell shape not supported");
  if (hs < 0 || hs >= states) return fail(AB_ERR_INVALID, "bad recurrent state index");
  if ((x_rs % 4) || (x_ts % 4) || (reinterpret_cast<uintptr_t>(x) % 16))
    return fail(AB_ERR_UNSUPPORTED, "x must be 16-byte aligned with 16-byte aligned rows");
  const size_t need = cell_ws_bytes(gates, B, H);
  if (!workspace || workspace_bytes < need)
    return fail(AB_ERR_INVALID, "Scan cell workspace too small: need %zu bytes, have %zu", need, workspace_bytes);
  const int tile_n = gates * CELL_UNITS;
  uint8_t* ws = reinterpret_cast<uint8_t*>(align_up(reinterpret_cast<uintptr_t>(workspace), 1024));
  const size_t hp = align_up((size_t)B * H * 4, 1024);
  const size_t up = align_up((size_t)gates * H * H * 4, 1024);
  CellParams p{};
  p.T = T; p.B = B; p.H = H;
  p.x = static_cast<const float*>(x); p.x_ts = x_ts; p.x_rs = x_rs;
  for (int k = 0; k < states; ++k) {
    if (reinterpret_cast<uintptr_t>(bufs[k]) % 16) return fail(AB_ERR_UNSUPPORTED, "state ring not 16-byte aligned");
    p.sbuf[k] = static_cast<float*>(bufs[k]); p.slen[k] = lens[k]; p.spos[k] = pos[k];
  }
  p.hs = hs;
  for (int s = 0; s < 2; ++s)
    for (int k = 0; k < 2; ++k) p.hplane[s][k] = reinterpret_cast<float*>(ws + (size_t)(2 * s + k) * hp);
  float* u_hi = reinterpret_cast<float*>(ws + 4 * hp);
  float* u_lo = reinterpret_cast<float*>(ws + 4 * hp + up);
  p.row_done = reinterpret_cast<unsigned int*>(ws + 4 * hp + 2 * up);
  AB_CUDA(cudaMemsetAsync(p.row_done, 0, row_flag_bytes(B), st));
  // planes of the recurrent state at step -1: the ring row just before its position
  const float* h_init = p.sbuf[hs] + ((pos[hs] - 1 + lens[hs]) % lens[hs]) * B * H;
  {
    const long long n = B * H;
    split_planes_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(h_init, B, H, H, 1, 0, gates,
                                                                    p.hplane[0][0], p.hplane[0][1]);
    g_launches++;
    // U[K=H, N=G*H] -> planes [G*H (gate-interleaved), K=H]: element (n, k) = U[k*u_rs + n*u_cs]
    const long long nu = (long long)gates * H * H;
    split_planes_kernel<<<(unsigned)((nu + 255) / 256), 256, 0, st>>>(
        static_cast<const float*>(U), (long long)gates * H, H, u_cs, u_rs, (int)H, gates, u_hi, u_lo);
    g_launches++;
    AB_CUDA(cudaGetLastError());
  }
  int dev = 0, sms = 0;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  CUtensorMap mh[2][2], mu[2];
  int rc;
  for (int s = 0; s < 2; ++s)
    for (int k = 0; k < 2; ++k)
      if ((rc = make_map_f32(&mh[s][k], p.hplane[s][k], H, B, CELL_BLOCK_M))) return rc;
  void* args[] = {&mh[0][0], &mh[0][1], &mh[1][0], &mh[1][1], &mu[0], &mu[1], &p};
  p.a_tile_bytes = CELL_BLOCK_M * SW_BYTES;
  p.b_tile_bytes = tile_n * SW_BYTES;
  const int stage_bytes = 2 * (p.a_tile_bytes + p.b_tile_bytes);
  p.stages = std::max(2, std::min(8, (kMaxSmemGemm - 1024) / stage_bytes));
  if ((rc = make_map_f32(&mu[0], u_hi, H, (long long)gates * H, tile_n))) return rc;
  if ((rc = make_map_f32(&mu[1], u_lo, H, (long long)gates * H, tile_n))) return rc;
  AB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, kMaxSmemGemm));
  const size_t smem = (size_t)p.stages * stage_bytes + 1024;
  int per_sm = 0;
  AB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, kCellThreads, smem));
  if (per_sm < 1) return fail(AB_ERR_CUDA, "the Scan cell kernel does not fit on an SM");
  const long long num_tiles = ((B + CELL_BLOCK_M - 1) / CELL_BLOCK_M) * (H / CELL_UNITS);
  // every CTA must be resident (tiles spin on the previous step's counters): cooperative, <= 1 per SM
  const unsigned grid = (unsigned)std::max<long long>(1, std::min<long long>(num_tiles, sms));
  AB_CUDA(cudaLaunchCooperativeKernel(kern, dim3(grid), dim3(kCellThreads), args, smem, st));
  g_launches++;
  return AB_OK;
}

}  // namespace

extern "C" int ab_lstm_scan_workspace_bytes(int64_t b, int64_t h, size_t* bytes) {
  if (!bytes) return fail(AB_ERR_INVALID, "null out pointer");
  *bytes = cell_ws_bytes(4, b, h);
  return AB_OK;
}

extern "C" int ab_lstm_scan_supported(int64_t t, int64_t b, int64_t h) {
  return cell_supported(4, 2, t, b, h) ? 1 : 0;
}

// h0 / c0 are expected to be already written into the rings at row (pos - 1) by the caller
// (Scan's IncSubtensor{InplaceSet} initial-state placement).
extern "C" int ab_lstm_scan(int64_t T, int64_t B, int64_t H, const void* x, int64_t x_ts,
                            int64_t x_rs, const void* U, int64_t u_rs, int64_t u_cs, void* hbuf,
                            int64_t sh, int64_t pos_h, void* cbuf, int64_t sc, int64_t pos_c,
                            void* workspace, size_t workspace_bytes, void* stream) {
  void* bufs[2] = {hbuf, cbuf};
  const int64_t lens[2] = {sh, sc}, pos[2] = {pos_h, pos_c};
  return cell_scan_launch((const void*)lstm_scan_kernel, 4, 2, 0, T, B, H,
                          x, x_ts, x_rs, U, u_rs, u_cs, bufs, lens, pos, workspace, workspace_bytes,
                          as_stream(stream));
}

// ---- generated cells (codegen/scan_cell.py): `module` is the NVRTC build of
// ab_scan_cell_kernel.cuh with the cell of the Scan's inner graph ----------------------------
extern "C" int ab_cell_scan_workspace_bytes(int gates, int64_t b, int64_t h, size_t* bytes) {
  if (!bytes) return fail(AB_ERR_INVALID, "null out pointer");
  *bytes = cell_ws_bytes(gates, b, h);
  return AB_OK;
}

extern "C" int ab_cell_scan_supported(int gates, int states, int64_t t, int64_t b, int64_t h) {
  return cell_supported(gates, states, t, b, h) ? 1 : 0;
}

extern "C" int ab_cell_scan(ab_module* module, int gates, int states, int hs, int64_t T, int64_t B,
                            int64_t H, const void* x, int64_t x_ts, int64_t x_rs, const void* U,
                            int64_t u_rs, int64_t u_cs, void* const* state_bufs,
                            const int64_t* state_lens, const int64_t* state_pos, void* workspace,
                            size_t workspace_bytes, void* stream) {
  if (!module || !state_bufs || !state_lens || !state_pos) return fail(AB_ERR_INVALID, "null argument");
  Module* m = reinterpret_cast<Module*>(module);
  cudaKernel_t k = nullptr;
  if (cudaLibraryGetKernel(&k, m->lib, "ab_cell_scan") != cudaSuccess) {
    cudaGetLastError();
    return fail(AB_ERR_INVALID, "the module is not a Scan cell build");
  }
  return cell_scan_launch((const void*)k, gates, states, hs, T, B, H, x, x_ts, x_rs, U,
                          u_rs, u_cs, state_bufs, state_lens, state_pos, workspace, workspace_bytes,
                          as_stream(stream));
}
