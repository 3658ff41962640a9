// ab_scan_cell_kernel.cuh — device code of the persistent Scan kernel for the family
//
//     pre  = x_t + s_hs[t-1] @ U                     one Gemm, alpha = beta = 1, [B, G*H]
//     s'_k = f_k(pre[:, 0:H], ..., pre[:, (G-1)H:GH], s_0[t-1], ..., s_{S-1}[t-1])   k < S
//
// i.e. "one Gemm(x_t, 1, h, U, 1) + Elemwise nodes on its column slices" (aesara/scan/op.py:637,
// loop :1799-2103, drives such an inner function from a Python/Cython loop, one BLAS call and
// several Elemwise thunks per step).  The LSTM cell of BASELINE config 4 is the member with
// G = 4, S = 2 (compiled ahead of time in ab_scan_lstm.cu); a tanh-RNN (G = 1, S = 1), gated
// units with G = 2 or 3 etc. are compiled at run time with the cell emitted from the inner
// graph's scalar expressions (codegen/scan_cell.py), exactly as the GEMM epilogues are.
//
// Macros the includer defines:  AB_CELL_GATES (1..4), AB_CELL_STATES (1..3) and
// AB_CELL_EVAL(G, P, O): float G[GATES] pre-activations, float P[STATES] previous states ->
// float O[STATES] new states, for one (row, hidden unit).
//
//   * persistent cooperative grid, one CTA per SM; every step the [B, G*H] pre-activation is
//     produced as 64 x (G*64) wgmma tiles (3xTF32, fp32-faithful like ab_gemm) whose columns
//     are the G gates of 64 hidden units (U is packed once with its columns gate-interleaved);
//   * the cell is the tile's epilogue, run in the accumulator registers: x_t and the previous
//     states are read once, the new states go to the Scan's circular output buffers and the
//     state that feeds the Gemm is ALSO written as the hi/lo TF32 planes the next step's TMA
//     loads; K is accumulated in 256-element segments (fresh register accumulator each, summed
//     in FP32 with round-to-nearest) because the tensor core's own accumulate truncates;
//   * no barrier between steps: batch rows are independent, so a tile of step t+1 waits only
//     for the step-t tiles of ITS row block (per-row-block counters: bar.sync of the consumer
//     warps, __threadfence, atomicAdd; acquire load + fence.proxy.async on the producer side);
//   * three warpgroups: {TMA producer, three idle warps} give most of their registers back
//     (setmaxnreg.dec) and the two consumer warpgroups take them (setmaxnreg.inc); consumer
//     warpgroup s issues the wgmma of hidden units [32 s, 32 s + 32) of the tile (G products
//     of N = 32 per K step) and evaluates the cell on them: G x 16 accumulator registers plus
//     as many for the running sum.
#pragma once

constexpr int kCellThreads = 384;
constexpr int kCellEpiThreads = 256;
constexpr int CELL_BLOCK_M = 64;                         // batch rows per tile
constexpr int CELL_UNITS = 64;                           // hidden units per tile
constexpr int CELL_TILE_N = AB_CELL_GATES * CELL_UNITS;  // accumulator columns
constexpr int CELL_KB = 32;                              // K elements (tf32) per 128-byte smem row
constexpr int CELL_SEG_KB = 8;                           // k-blocks per accumulation segment (256 K)

struct CellParams {
  long long T, B, H;
  const float* x;            // [T, B, G*H]
  long long x_ts, x_rs;      // element strides of x: step, row (columns contiguous)
  float* sbuf[3];            // Scan output rings of the states: [slen, B, H] contiguous rows
  long long slen[3], spos[3];
  int hs;                    // the state that multiplies U
  float* hplane[2][2];       // [set][hi/lo] K-major planes [B, H] of that state for the tensor cores
  unsigned int* row_done;    // per row block: tiles completed so far, all steps (zero-initialised)
  int stages;
  int a_tile_bytes, b_tile_bytes;
};

__device__ __forceinline__ float sigmoidf_ref(float v) { return 1.0f / (1.0f + expf(-v)); }

__device__ __forceinline__ void cell_scan_body(const CUtensorMap& map_h00, const CUtensorMap& map_h01,
                                               const CUtensorMap& map_h10, const CUtensorMap& map_h11,
                                               const CUtensorMap& map_u0, const CUtensorMap& map_u1,
                                               const CellParams& p) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) &
                                             ~static_cast<uintptr_t>(1023));
  __shared__ __align__(8) uint64_t full_bar[8];
  __shared__ __align__(8) uint64_t empty_bar[8];

  constexpr int G = AB_CELL_GATES, S = AB_CELL_STATES;
  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int stage_bytes = 2 * (p.a_tile_bytes + p.b_tile_bytes);  // hi + lo of A and B
  const int num_k_blocks = (int)((p.H + CELL_KB - 1) / CELL_KB);
  const long long tiles_n = p.H / CELL_UNITS;
  const long long num_tiles = ((p.B + CELL_BLOCK_M - 1) / CELL_BLOCK_M) * tiles_n;

  if (threadIdx.x == 0) {
    for (int s = 0; s < p.stages; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], kCellEpiThreads / 32);  // one arrival per consumer warp
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  }
  __syncthreads();

  // Register budget per SM sub-partition (3 warps each): 56 + 2 x 224 <= 512.  Each role runs
  // its whole T-step loop inside its own branch: ptxas allocates the code that follows a
  // setmaxnreg up to that count only while the branches do not merge again.
  if (warp < 4) {
    asm volatile("setmaxnreg.dec.sync.aligned.u32 56;");
    if (warp == 0 && elect_one()) {
      // ================= TMA producer =================
      int stage = 0;
      uint32_t phase = 0;
      for (long long t = 0; t < p.T; ++t) {
        const int set = (int)(t & 1);  // planes read this step; the other set is written
        const CUtensorMap* mh0 = set ? &map_h10 : &map_h00;
        const CUtensorMap* mh1 = set ? &map_h11 : &map_h01;
        for (long long tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
          const int m0 = (int)((tile / tiles_n) * CELL_BLOCK_M);
          const int n0 = (int)((tile % tiles_n) * CELL_TILE_N);
          if (t > 0) {
            // rows of s_hs[t-1] for this row block exist once all of its step t-1 tiles are counted
            const unsigned int target = (unsigned int)(t * tiles_n);
            const unsigned int* flag = p.row_done + tile / tiles_n;
            unsigned int seen;
            do {
              asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(seen) : "l"(flag) : "memory");
              if (seen < target) __nanosleep(32);
            } while (seen < target);
            asm volatile("fence.proxy.async;" ::: "memory");  // generic-proxy writes -> TMA reads
          }
          for (int kb = 0; kb < num_k_blocks; ++kb) {
            mbar_wait(&empty_bar[stage], phase ^ 1);
            uint8_t* sbase = smem + (size_t)stage * stage_bytes;
            mbar_expect_tx(&full_bar[stage], (uint32_t)stage_bytes);
            const int kc = kb * CELL_KB;
            uint8_t* b_hi = sbase + 2 * p.a_tile_bytes;
            tma_load_2d(sbase, mh0, &full_bar[stage], kc, m0);
            tma_load_2d(sbase + p.a_tile_bytes, mh1, &full_bar[stage], kc, m0);
            tma_load_2d(b_hi, &map_u0, &full_bar[stage], kc, n0);
            tma_load_2d(b_hi + p.b_tile_bytes, &map_u1, &full_bar[stage], kc, n0);
            if (++stage == p.stages) { stage = 0; phase ^= 1; }
          }
        }
      }
    }
  } else {
    asm volatile("setmaxnreg.inc.sync.aligned.u32 224;");
    // ================= consumers: wgmma, then the cell (warps 4..11) =================
    const int s = (warp - 4) >> 2;                 // hidden units [32 s, 32 s + 32) of the tile
    const int r_lo = 16 * (warp & 3) + (lane >> 2);  // tile rows r_lo and r_lo + 8 of this thread
    const int u_lane = 32 * s + 2 * (lane & 3);    // + 8 j (+ 1): the thread's units in the tile
    int stage = 0;
    uint32_t phase = 0;
    for (long long t = 0; t < p.T; ++t) {
      const int set = (int)(t & 1);
      float* out_row[S];
      const float* prev_row[S];
#pragma unroll
      for (int k = 0; k < S; ++k) {
        const long long r_now = (p.spos[k] + t) % p.slen[k];                    // ring rows written now
        const long long r_prev = (p.spos[k] + t - 1 + p.slen[k]) % p.slen[k];   // state[t-1]
        out_row[k] = p.sbuf[k] + r_now * p.B * p.H;
        prev_row[k] = p.sbuf[k] + r_prev * p.B * p.H;
      }
      float* hp_hi = p.hplane[set ^ 1][0];
      float* hp_lo = p.hplane[set ^ 1][1];
      const float* xt = p.x + t * p.x_ts;
      for (long long tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        const long long m0 = (tile / tiles_n) * CELL_BLOCK_M;
        const long long u0 = (tile % tiles_n) * CELL_UNITS;
        // The running sum starts out as this thread's x_t gate pre-activations (the Gemm's
        // "+ 1 * x_t", blas.py:984-1017): the loads are in flight while the tensor core
        // produces the first K segment.  f[g][4 j + 2 h + e] = (row r_lo + 8 h, unit u_lane + 8 j + e)
        float f[G][16];
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const long long row = m0 + r_lo + 8 * h;
#pragma unroll
          for (int g = 0; g < G; ++g)
#pragma unroll
            for (int j = 0; j < 4; ++j) {
              const float2 xv = row < p.B ? __ldcs(reinterpret_cast<const float2*>(xt + row * p.x_rs + g * p.H + u0 + u_lane + 8 * j))
                                          : make_float2(0.0f, 0.0f);
              f[g][4 * j + 2 * h] = xv.x;
              f[g][4 * j + 2 * h + 1] = xv.y;
            }
        }
        for (int kb0 = 0; kb0 < num_k_blocks; kb0 += CELL_SEG_KB) {
          const int kb1 = min(kb0 + CELL_SEG_KB, num_k_blocks);
          float d[G][16];
          int prev = -1;
          for (int kb = kb0; kb < kb1; ++kb) {
            mbar_wait(&full_bar[stage], phase);
            const uint32_t sbase = smem_u32(smem + (size_t)stage * stage_bytes);
            const uint32_t a_hi = sbase, a_lo = sbase + p.a_tile_bytes;
            // this warpgroup's 32 rows of gate g in the B tile: 32 x 128 B at g * 64 + 32 s
            const uint32_t b_hi = sbase + 2 * p.a_tile_bytes + (uint32_t)(s * 32 * SW_BYTES);
            const uint32_t b_lo = b_hi + p.b_tile_bytes;
            wgmma_fence();
#pragma unroll
            for (int k = 0; k < SW_BYTES / 32; ++k) {
              const uint32_t ko = k * 32;
              const uint32_t acc = (kb > kb0 || k > 0) ? 1u : 0u;
#pragma unroll
              for (int g = 0; g < G; ++g) {
                const uint32_t bo = (uint32_t)(g * CELL_UNITS * SW_BYTES) + ko;
                wgmma_m64n32k8_tf32(d[g], make_smem_desc(a_lo + ko, 16), make_smem_desc(b_hi + bo, 16), acc);
                wgmma_m64n32k8_tf32(d[g], make_smem_desc(a_hi + ko, 16), make_smem_desc(b_lo + bo, 16), 1u);
                wgmma_m64n32k8_tf32(d[g], make_smem_desc(a_hi + ko, 16), make_smem_desc(b_hi + bo, 16), 1u);
              }
            }
            wgmma_commit();
            wgmma_wait<1>();  // the previous k-block's products have retired: free its stage
            if (prev >= 0 && lane == 0) mbar_arrive(&empty_bar[prev]);
            prev = stage;
            if (++stage == p.stages) { stage = 0; phase ^= 1; }
          }
          wgmma_wait<0>();
          if (lane == 0) mbar_arrive(&empty_bar[prev]);
#pragma unroll
          for (int g = 0; g < G; ++g)
#pragma unroll
            for (int i = 0; i < 16; ++i) f[g][i] = __fadd_rn(f[g][i], d[g][i]);
        }
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const long long row = m0 + r_lo + 8 * h;
          if (row >= p.B) continue;
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            const long long so = row * p.H + u0 + u_lane + 8 * j;
            float pv[S][2], ov[S][2];
#pragma unroll
            for (int k = 0; k < S; ++k) {
              const float2 q2 = *reinterpret_cast<const float2*>(prev_row[k] + so);
              pv[k][0] = q2.x; pv[k][1] = q2.y;
            }
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              float gv[G], pe[S], oe[S];
#pragma unroll
              for (int g = 0; g < G; ++g) gv[g] = f[g][4 * j + 2 * h + e];
#pragma unroll
              for (int k = 0; k < S; ++k) pe[k] = pv[k][e];
              AB_CELL_EVAL(gv, pe, oe);  // the Elemwise nodes of the inner graph on pre = x_t + s_hs @ U
#pragma unroll
              for (int k = 0; k < S; ++k) ov[k][e] = oe[k];
            }
#pragma unroll
            for (int k = 0; k < S; ++k) {
              *reinterpret_cast<float2*>(out_row[k] + so) = make_float2(ov[k][0], ov[k][1]);
              if (p.hs == k) {
                // the state that feeds the next step's Gemm, also as its hi/lo TF32 planes
                float hh[2], hl[2];
#pragma unroll
                for (int e = 0; e < 2; ++e) tf32_split(ov[k][e], hh[e], hl[e]);
                *reinterpret_cast<float2*>(hp_hi + so) = make_float2(hh[0], hh[1]);
                *reinterpret_cast<float2*>(hp_lo + so) = make_float2(hl[0], hl[1]);
              }
            }
          }
        }
        // the new states of this tile are written: count the tile on its row block so that the
        // producer of step t+1 may load those rows (all 256 consumer threads' stores first)
        asm volatile("bar.sync 1, %0;" ::"r"(kCellEpiThreads) : "memory");
        if (warp == 4 && lane == 0) {
          __threadfence();
          atomicAdd(p.row_done + tile / tiles_n, 1u);
        }
      }
    }
  }
}

#ifdef AB_CELL_JIT
// NVRTC build: C-linkage entry point (looked up by name from ab_cell_scan)
extern "C" __global__ void __launch_bounds__(kCellThreads, 1)
ab_cell_scan(const __grid_constant__ CUtensorMap h00, const __grid_constant__ CUtensorMap h01,
             const __grid_constant__ CUtensorMap h10, const __grid_constant__ CUtensorMap h11,
             const __grid_constant__ CUtensorMap u0, const __grid_constant__ CUtensorMap u1,
             const __grid_constant__ CellParams p) { cell_scan_body(h00, h01, h10, h11, u0, u1, p); }
#endif
