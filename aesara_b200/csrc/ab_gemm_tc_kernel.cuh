// ab_gemm_tc_kernel.cuh — device code of the Hopper tensor-core GEMM (parameters, TMA producer,
// wgmma warpgroups, epilogue warpgroup).  Included by ab_gemm_tc.cu (ahead-of-time kernels with
// the plain alpha/beta epilogue) and, with AB_EPILOGUE defined, concatenated behind a generated
// `ab_ep_body` and compiled by NVRTC (codegen/gemm_epilogue.py): the Elemwise node that consumes
// a Gemm/Dot22 result is then applied to the accumulator before the only store.
#pragma once

// Thread layout (512 threads, one 128 x BLOCK_N output tile at a time, persistent):
//   warpgroup 0     TMA producer (one elected thread of warp 0; warps 1..3 idle);
//   warpgroups 1-2  MMA: warpgroup c issues the wgmma of tile rows [64 c, 64 c + 64) into 64
//                   accumulator registers per thread and adds each finished K segment into a
//                   running total held in 64 more registers; at the end of the unit it stores
//                   the total ONCE into the tile's float32 accumulator in shared memory;
//   warpgroup 3     epilogue: warp q reads tile rows [32 q, 32 q + 32) of that accumulator,
//                   one row per lane, all BLOCK_N columns (the layout the generated epilogue
//                   regions are written for), while the MMA warpgroups run the next unit's
//                   main loop.
// The shared accumulator is a single hand-off buffer between the two sides (mbarriers
// acc_full: one arrival per MMA warp after its stores; acc_empty: one arrival per epilogue
// warp after its last read): the MMA side needs it again only at the end of its next unit.
// Registers (setmaxnreg, multiples of 8; 512 threads launch with 128 each = 65 536):
//   producer 24, MMA 160 (d[64] + tot[64] + addressing), epilogue 168:
//   128 * 24 + 256 * 160 + 128 * 168 = 3 072 + 40 960 + 21 504 = 65 536.
// The cluster variant's producer, which multicasts, keeps 56 and its (plain) epilogue 136:
//   128 * 56 + 256 * 160 + 128 * 136 = 7 168 + 40 960 + 17 408 = 65 536.
constexpr int kGemmThreads = kThreads;
constexpr int kMmaWarp0 = 4;   // first warp of the MMA warpgroups
constexpr int kEpiWarp0 = 12;  // first warp of the epilogue warpgroup
#define AB_SETMAXNREG_CONTROL(CL)                                         \
  if (CL > 1) asm volatile("setmaxnreg.dec.sync.aligned.u32 56;");        \
  else asm volatile("setmaxnreg.dec.sync.aligned.u32 24;")
#define AB_SETMAXNREG_MMA(CL) asm volatile("setmaxnreg.inc.sync.aligned.u32 160;")
#define AB_SETMAXNREG_EPILOGUE(CL)                                        \
  if (CL > 1) asm volatile("setmaxnreg.inc.sync.aligned.u32 136;");       \
  else asm volatile("setmaxnreg.inc.sync.aligned.u32 168;")
constexpr int kMmaThreads = 256;  // 8 MMA warps
constexpr int kEpiThreads = 128;  // 4 epilogue warps
constexpr int BLOCK_N = 128;
constexpr int kAccBytes = BLOCK_M * BLOCK_N * 4;  // the tile's float32 accumulator in shared memory

struct GemmParams {
  long long M, N, K;      // K in elements of the packed type
  float alpha, beta;
  float* C;
  long long c_rs, c_cs;
  const float* Cin;       // beta term source (== C for the in-place Gemm, another buffer otherwise)
  long long cin_rs, cin_cs;
  int block_n;            // BLOCK_N
  int seg_kblocks;        // k-blocks accumulated inside the tensor core before the partial sum
                          // is folded into the shared-memory accumulator (see "segments")
  int group_m;            // tile rows per group of the grouped unit order (AB_UNIT_DECODE)
  int k_splits;           // split-K: work unit = (K range, tile)
  int kb_per_split;       // k-blocks per K range
  float* partial;         // [k_splits - 1][M][N] alpha * (A@B over K range s), s >= 1
  int stages;
  int nparts;             // 1, or 2 for the hi/lo split (3 MMAs per k-step)
  int k_elems_per_row;    // K elements per stage = per 128-byte K-major row: 32 (tf32) / 64 (bf16)
  int a_tile_bytes, b_tile_bytes;
  int a_mn, b_mn;         // operand is MN-major
  int a_mn3d, b_mn3d;     // ... and its tensor map is 3-D {128 B of MN, K rows, MN chunks}: the
                          // whole tile arrives with ONE bulk copy instead of one per chunk
  int a_chunks, b_chunks; // MN-major: 128-byte MN chunks per tile (tile_rows * elem_size / 128)
  int chunk_bytes;        // MN-major: k_elems_per_row rows * 128 B
  int mn_per_chunk;       // MN-major: elements per chunk (128 / elem_size)
  int a_kstep, b_kstep;   // descriptor advance per MMA K-step: 32 B (K-major) or mma_k rows * 128 B
  // fused consumer (AB_EPILOGUE builds only; zero otherwise): out = ab_ep_body(v, e0..e3)
  // with v = alpha*acc + beta*Cin and e_k = ep_ptr[k][row * ep_rs[k] + col * ep_cs[k]]
  // (stride 0 = broadcast); `shadow` receives the bf16 copy of out as a [M, shadow_pitch]
  // K-major operand plane for the GEMM that consumes it next
  const float* ep_ptr[4];
  long long ep_rs[4], ep_cs[4];
  // the epilogue program yields AB_EP_NOUT values per element.  Value 0 goes to C (when C is
  // not null), value k >= 1 to out_ptr[k] ([M, out_rs[k]] rows, unit column stride; null =
  // not materialised); shadow[k] (optional) receives the bf16 copy of value k as a
  // [M, shadow_pitch[k]] K-major operand plane for the GEMM that consumes it next.
  float* out_ptr[3];
  long long out_rs[3];
  void* shadow[3];
  long long shadow_pitch[3];
  // shadow_t (optional, value AB_EP_TPLANE only): the TRANSPOSED bf16 copy, an [N, shadow_t_pitch]
  // plane whose rows are the columns of the value -- the K-major operand of a product that
  // contracts over the ROWS of the value (h.T @ dout, X.T @ dpre: both operands of a weight
  // gradient), so that the weight-gradient product reads both operands K-major.
  void* shadow_t;
  long long shadow_t_pitch;
  // reductions of one value each, accumulated in float64 like the reference's CAReduce
  // (tensor/elemwise.py:1371-1385): colsum_ws[rb][col] = sum over the 32 rows of row block
  // rb of value AB_EP_COLSUM; fullsum_ws[rb][cb] = sum of value AB_EP_FULLSUM over row block
  // rb and column block cb (half a tile).  A second, deterministic pass adds the partials.
  double* colsum_ws;
  double* fullsum_ws;
  long long fullsum_cols;
  // L2 eviction priority of the operands' tiles (make_l2_policy): a weight matrix that every
  // tile row re-reads is kept (evict_last) against the stream of the large operand and of the
  // epilogue's reads and writes (those use .cs accesses), which would otherwise push it out of
  // L2 between the tile rows that re-read it.
  int a_l2, b_l2;
  // derived on the host, read from the parameter space where used (held in registers across
  // the main loop and the epilogue they cost the larger generated regions their registers)
  int stage_bytes;        // nparts * (a_tile_bytes + b_tile_bytes)
  int num_k_blocks;
  long long tiles_n, num_tiles, num_units;  // tiles of one CTA, or of a cluster (CL > 1)
};

// one operand tile -> shared memory.  K-major: a single box {128 B of K, tile rows};
// MN-major: one box {128 B of MN, BLOCK_K rows} per chunk.
// Loop-invariant description of one operand's tile loads.  The producer and the MMA issuer
// copy what they need from GemmParams into locals BEFORE their loops: the kernel parameter
// lives in constant memory, every mbarrier / TMA asm statement carries a "memory" clobber, and
// a field read through `p` inside the loop is re-loaded (LDCU + dependent UISETP) after each
// of them, on the single producer thread's critical path.
struct OperandLoad {
  int mn_major, chunks, mn3d, chunk_bytes, mn_per_chunk;
  uint64_t policy;
};
__device__ __forceinline__ OperandLoad operand_load_a(const GemmParams& p) {
  return OperandLoad{p.a_mn, p.a_chunks, p.a_mn3d, p.chunk_bytes, p.mn_per_chunk, make_l2_policy(p.a_l2)};
}
__device__ __forceinline__ OperandLoad operand_load_b(const GemmParams& p) {
  return OperandLoad{p.b_mn, p.b_chunks, p.b_mn3d, p.chunk_bytes, p.mn_per_chunk, make_l2_policy(p.b_l2)};
}
__device__ __forceinline__ void load_tile(uint8_t* dst, const CUtensorMap* map, uint64_t* bar,
                                          int kc, int mn0, const OperandLoad& o) {
  if (!o.mn_major) {
    tma_load_2d_hint(dst, map, bar, kc, mn0, o.policy);
  } else if (o.mn3d) {
    tma_load_3d(dst, map, bar, 0, kc, mn0 / o.mn_per_chunk);
  } else {
    for (int c = 0; c < o.chunks; ++c)
      tma_load_2d_hint(dst + c * o.chunk_bytes, map, bar, mn0 + c * o.mn_per_chunk, kc, o.policy);
  }
}

// ---------------------------------------------------------------------- segments
// The tensor core adds each MMA's products into its FP32 accumulator with truncation (round
// toward zero), a bias that grows linearly with the number of accumulation steps; an
// unsegmented 3xTF32 K = 4096 product drifts well past a true-fp32 sgemm
// (tests/test_gpu_blas.py::test_gemm_long_k_accuracy).  So the K loop is cut into segments of
// seg_kblocks k-blocks: each segment starts a fresh register accumulator, and the MMA
// warpgroup adds the finished segment into the unit's float32 total (registers, acc_fold)
// with round-to-nearest.  For precision 0 a segment is 128 K elements (48 truncating steps);
// the tf32 / bf16 policies use segments of 16 k-blocks (512 / 1024 K elements), so that a long
// K (a weight gradient over a 65536-row batch) does not depend on the order of its rows beyond
// the rounding of those folds.
constexpr int kAccRegs = BLOCK_N / 2;  // accumulator columns the plain epilogue holds at once (half a tile row)

// shared-memory accumulator: [BLOCK_M][BLOCK_N] float32, 16-byte group g of row r stored at
// group (g & ~7) | ((g ^ r) & 7) -- conflict-free for the row-per-lane reads of the epilogue
__device__ __forceinline__ uint32_t acc_off(int r, int c) {
  const int g = c >> 2;
  return (uint32_t)(r * (BLOCK_N * 4) + (((g & ~7) | ((g ^ r) & 7)) << 4) + ((c & 3) << 2));
}
// add a finished segment into the warpgroup's running total, kept in registers beside the
// wgmma accumulator.  A unit's total starts at -0.0f, the identity of the round-to-nearest
// add (-0 + x == x for every x, zeros of either sign included): the first segment is added
// like the others, so the fold is one FADD per register in place (a select between d and the
// sum costs a second copy of the total and spills it)
__device__ __forceinline__ void acc_fold(float (&tot)[64], const float (&d)[64]) {
#pragma unroll
  for (int i = 0; i < 64; ++i) tot[i] = __fadd_rn(tot[i], d[i]);
}
// the warpgroup's 64 x BLOCK_N total of a unit -> the tile's accumulator in shared memory
// (acc_off layout).  Element 4 j + 2 h + e of the fragment is row row0 + lane / 4 + 8 h, column
// 8 j + 2 (lane % 4) + e, and row0 % 8 == 0: the swizzle term (g ^ r) & 7 depends only on the
// lane and on j % 4.  So four addresses per thread and immediate offsets cover the 32 stores
// (32 addresses from acc_off are hoisted out of the unit loop and take registers from tot).
__device__ __forceinline__ void acc_store(uint32_t acc_base, const float (&tot)[64], int row0, int lane) {
  const uint32_t y = (uint32_t)(((lane >> 1) & 1) ^ (lane >> 2));  // ((column / 4) ^ row) % 8 at j = 0
  const uint32_t base = acc_base + (uint32_t)((row0 + (lane >> 2)) * (BLOCK_N * 4) + ((lane & 1) << 3));
#pragma unroll
  for (int jj = 0; jj < 4; ++jj) {
    const uint32_t a = base + ((y ^ (uint32_t)(2 * jj)) << 4);
#pragma unroll
    for (int jq = 0; jq < BLOCK_N / 32; ++jq) {
      const int j = 4 * jq + jj;
#pragma unroll
      for (int h = 0; h < 2; ++h)
        asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(a + (uint32_t)(jq * 128 + h * 8 * BLOCK_N * 4)),
                     "f"(tot[4 * j + 2 * h]), "f"(tot[4 * j + 2 * h + 1])
                     : "memory");
    }
  }
}
// 32 consecutive accumulator columns c0 .. c0 + 31 (c0 % 32 == 0) of tile row r
__device__ __forceinline__ void acc_ld_x32(uint32_t acc_base, int r, int c0, float (&x)[32]) {
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const float4 v = lds128(acc_base + acc_off(r, c0 + 4 * i));
    x[4 * i] = v.x; x[4 * i + 1] = v.y; x[4 * i + 2] = v.z; x[4 * i + 3] = v.w;
  }
}

// C[row, n0 + ...] = alpha * acc + beta * Cin for one thread's row and column range
// 8 consecutive floats as two 128-bit accesses (16-byte alignment is the caller's precondition;
// sm_90 has no 256-bit global access)
#define AB_HAS_V8 0
// STREAM: the access belongs to a fused epilogue region -- [M, N] operands read once and values
// written once, far larger than L2: evict-first, so that they do not push the products' small
// operand (a weight matrix, GemmParams::b_l2) out of L2.  The plain alpha/beta epilogue keeps
// the default policy (a small result is usually the next node's operand).
template <bool STREAM>
__device__ __forceinline__ void ld8(const float* q, float (&o)[8], bool wide) {
#if AB_HAS_V8
  if (wide) {
    if (STREAM)
      asm volatile("ld.global.L1::no_allocate.L2::evict_first.v8.f32 {%0,%1,%2,%3,%4,%5,%6,%7}, [%8];"
                   : "=f"(o[0]), "=f"(o[1]), "=f"(o[2]), "=f"(o[3]), "=f"(o[4]), "=f"(o[5]), "=f"(o[6]), "=f"(o[7])
                   : "l"(q));
    else
      asm volatile("ld.global.v8.f32 {%0,%1,%2,%3,%4,%5,%6,%7}, [%8];"
                   : "=f"(o[0]), "=f"(o[1]), "=f"(o[2]), "=f"(o[3]), "=f"(o[4]), "=f"(o[5]), "=f"(o[6]), "=f"(o[7])
                   : "l"(q));
  } else
#endif
  {
    const float4 a = STREAM ? __ldcs(reinterpret_cast<const float4*>(q)) : *reinterpret_cast<const float4*>(q);
    const float4 b = STREAM ? __ldcs(reinterpret_cast<const float4*>(q + 4)) : *reinterpret_cast<const float4*>(q + 4);
    o[0] = a.x; o[1] = a.y; o[2] = a.z; o[3] = a.w; o[4] = b.x; o[5] = b.y; o[6] = b.z; o[7] = b.w;
  }
}
template <bool STREAM>
__device__ __forceinline__ void st8(float* q, const float (&v)[8], bool wide) {
#if AB_HAS_V8
  if (wide) {
    if (STREAM)
      asm volatile("st.global.L2::evict_first.v8.f32 [%0], {%1,%2,%3,%4,%5,%6,%7,%8};" ::"l"(q), "f"(v[0]), "f"(v[1]),
                   "f"(v[2]), "f"(v[3]), "f"(v[4]), "f"(v[5]), "f"(v[6]), "f"(v[7])
                   : "memory");
    else
      asm volatile("st.global.v8.f32 [%0], {%1,%2,%3,%4,%5,%6,%7,%8};" ::"l"(q), "f"(v[0]), "f"(v[1]), "f"(v[2]),
                   "f"(v[3]), "f"(v[4]), "f"(v[5]), "f"(v[6]), "f"(v[7])
                   : "memory");
  } else
#endif
  {
    if (STREAM) {
      __stcs(reinterpret_cast<float4*>(q), make_float4(v[0], v[1], v[2], v[3]));
      __stcs(reinterpret_cast<float4*>(q + 4), make_float4(v[4], v[5], v[6], v[7]));
    } else {
      *reinterpret_cast<float4*>(q) = make_float4(v[0], v[1], v[2], v[3]);
      *reinterpret_cast<float4*>(q + 4) = make_float4(v[4], v[5], v[6], v[7]);
    }
  }
}

#ifndef AB_EP_STAGED
#define AB_EP_STAGED 0
#endif
constexpr int kStageBytesPerWarp = 32 * 32 * 4;                     // one 32 x 32 float32 chunk
constexpr int kStageBytes = (kEpiThreads / 32) * kStageBytesPerWarp;  // behind the operand ring

struct EpilogueOut {
  const GemmParams& p;
  bool vec_ok, wide_out, wide_in;
  uint32_t stage;  // AB_EP_STAGED builds: shared-space address of this warp's 4 KB (see fused_reduce)
  __device__ explicit EpilogueOut(const GemmParams& p_, uint32_t stage_ = 0) : p(p_), stage(stage_) {
    vec_ok = (p.c_cs == 1) && ((p.c_rs & 3) == 0) && ((reinterpret_cast<uintptr_t>(p.C) & 15) == 0) &&
             (p.beta == 0.0f || ((p.cin_cs == 1) && ((p.cin_rs & 3) == 0) &&
                                 ((reinterpret_cast<uintptr_t>(p.Cin) & 15) == 0)));
    wide_out = ((p.c_rs & 7) == 0) && ((reinterpret_cast<uintptr_t>(p.C) & 31) == 0);
    wide_in = ((p.cin_rs & 7) == 0) && ((reinterpret_cast<uintptr_t>(p.Cin) & 31) == 0);
  }
  // split-K: alpha * acc of K range `split` (>= 1) into its [M, N] scratch plane
  __device__ __forceinline__ void store_partial(const float (&acc)[kAccRegs], long long row,
                                                long long n0, int nchunks, int split) const {
    if (row >= p.M) return;
    float* prow = p.partial + ((long long)(split - 1) * p.M + row) * p.N;
    const bool vec = (p.N & 3) == 0;
#pragma unroll
    for (int c = 0; c < kAccRegs / 32; ++c) {
      if (c < nchunks) {
        const long long col0 = n0 + c * 32;
        if (vec && col0 + 32 <= p.N) {
#pragma unroll
          for (int j = 0; j < 32; j += 4)
            *reinterpret_cast<float4*>(prow + col0 + j) =
                make_float4(p.alpha * acc[c * 32 + j], p.alpha * acc[c * 32 + j + 1],
                            p.alpha * acc[c * 32 + j + 2], p.alpha * acc[c * 32 + j + 3]);
        } else {
#pragma unroll
          for (int j = 0; j < 32; ++j)
            if (col0 + j < p.N) prow[col0 + j] = p.alpha * acc[c * 32 + j];
        }
      }
    }
  }
  __device__ __forceinline__ void store(const float (&acc)[kAccRegs], long long row, long long n0,
                                        int nchunks) const {
    if (row >= p.M) return;
    float* crow = p.C + row * p.c_rs;
    const float* irow = p.Cin + row * p.cin_rs;
#pragma unroll
    for (int c = 0; c < kAccRegs / 32; ++c) {
      if (c < nchunks) {
        const long long col0 = n0 + c * 32;
        if (vec_ok && col0 + 32 <= p.N) {
          // 8 columns per step: one 256-bit access per 32-byte sector where the rows are
          // 32-byte aligned (each L2 sector is touched by one request instead of two)
#pragma unroll
          for (int j = 0; j < 32; j += 8) {
            float v[8];
#pragma unroll
            for (int t = 0; t < 8; ++t) v[t] = p.alpha * acc[c * 32 + j + t];
            if (p.beta != 0.0f) {
              float o[8];
              ld8<false>(irow + col0 + j, o, wide_in);
#pragma unroll
              for (int t = 0; t < 8; ++t) v[t] += p.beta * o[t];
            }
            st8<false>(crow + col0 + j, v, wide_out);
          }
        } else {
#pragma unroll
          for (int j = 0; j < 32; ++j) {
            const long long col = col0 + j;
            if (col < p.N) {
              float v = p.alpha * acc[c * 32 + j];
              if (p.beta != 0.0f) v += p.beta * irow[col * p.cin_cs];
              crow[col * p.c_cs] = v;
            }
          }
        }
      }
    }
  }
#ifdef AB_EPILOGUE
  // ---- fused consumer region (codegen/gemm_epilogue.py) -------------------------------
  // The generated AB_EP_EVAL(V, E, T, O) evaluates the region's scalar program on
  // v = alpha*acc + beta*Cin and the memory operands E[k][T], leaving its AB_EP_NOUT values
  // in O[0..][T].  Contract (gemm_run refuses the fused launch otherwise): N % 8 == 0, every
  // matrix that is read or written 8 columns at a time (C, Cin, extra outputs, operands with
  // unit column stride) has 16-byte aligned rows.
  //
  // The work is organised per 32-column chunk of one accumulator row (`fused_chunk`), so that
  // the body exists ONCE in the instruction stream: an epilogue unrolled over all 128
  // columns of a thread (tanh, IEEE division, float64 sums per element) is several hundred KB
  // of SASS, which every warp re-fetches from L2 for every tile (measured: the region with
  // two values and two reductions ran 1.5 ms slower than its five separate kernels).
  struct FusedScalars { float v[4]; bool is[4]; bool vec[4]; };
  // Sums of the region are kept as unevaluated float pairs (hi + lo, error-free TwoSum) while
  // they stay inside a thread or a warp, and become float64 where they leave it: one DADD +
  // one F2F.F64 per element on the narrow FP64 pipe would make the epilogue of a region with
  // reductions its critical path.  A pair carries ~48 bits: the float64 accumulator of the reference's
  // CAReduce (tensor/elemwise.py:1371-1385) to well below the float32 rounding of the result.
  struct FF { float hi, lo; };
  static __device__ __forceinline__ void ff_add(FF& a, float x) {
    const float t = __fadd_rn(a.hi, x);
    const float bp = __fsub_rn(t, a.hi);
    a.lo = __fadd_rn(a.lo, __fadd_rn(__fsub_rn(a.hi, __fsub_rn(t, bp)), __fsub_rn(x, bp)));
    a.hi = t;
  }
  static __device__ __forceinline__ void ff_add(FF& a, const FF& b) {
    const float lo = a.lo;
    a.lo = 0.0f;
    ff_add(a, b.hi);
    a.lo = __fadd_rn(a.lo, __fadd_rn(lo, b.lo));
  }
  // non-finite sums: hi already is the inf / nan the float64 sum would be (lo is nan then)
  static __device__ __forceinline__ double ff_double(const FF& a) {
    return (a.hi - a.hi == 0.0f) ? (double)a.hi + (double)a.lo : (double)a.hi;
  }
  __device__ __forceinline__ FusedScalars load_scalars() const {
    FusedScalars s;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      s.is[k] = k < AB_EP_NOPS && p.ep_rs[k] == 0 && p.ep_cs[k] == 0;  // a [1,1] operand
      s.v[k] = s.is[k] ? p.ep_ptr[k][0] : 0.0f;
      s.vec[k] = k < AB_EP_NOPS && p.ep_rs[k] == 0 && p.ep_cs[k] == 1;  // a [1,N] row (a bias)
    }
    return s;
  }
  // SKIP: the value that leaves through the shared-memory staging buffer instead (-1: none)
  template <int SKIP>
  __device__ __forceinline__ void put_outputs(const float (&o)[AB_EP_NOUT][8], long long row, long long col) const {
#pragma unroll
    for (int k = 0; k < AB_EP_NOUT; ++k) {
      if (k == SKIP) continue;
      float* dst = k == 0 ? p.C : p.out_ptr[k];
      const long long rs = k == 0 ? p.c_rs : p.out_rs[k];
      if (dst)
        st8<true>(dst + row * rs + col, o[k], ((rs & 7) == 0) && ((reinterpret_cast<uintptr_t>(dst) & 31) == 0));
      if (p.shadow[k]) {
        uint32_t h[4];
#pragma unroll
        for (int t = 0; t < 4; ++t)
          asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(h[t]) : "f"(o[k][2 * t + 1]), "f"(o[k][2 * t]));
        uint16_t* sp = static_cast<uint16_t*>(p.shadow[k]) + row * p.shadow_pitch[k] + col;
        __stcs(reinterpret_cast<uint4*>(sp), make_uint4(h[0], h[1], h[2], h[3]));
      }
    }
  }
  // Matrix-shaped reads of a 32-column chunk (the Gemm's z; one [M, N] operand such as h in
  // g * (1 - h^2)) are issued as one batch, ONE CHUNK AHEAD of their use (store_fused*): the
  // loads of all four column groups are in flight together and their DRAM latency passes
  // under the evaluation of the previous chunk.  Loaded group by group right before their
  // use, such an epilogue is latency-bound (16 dependent round trips per tile); loaded per chunk
  // but consumed at once, it still waits one DRAM latency per chunk.
  //
  // A [1, N] operand (a bias row) is the same for all 32 rows of a warp: lane l fetches the
  // value of column col0 + l (one coalesced 128-byte read per chunk, a chunk ahead like the
  // matrices) and the evaluation takes column j's value from lane j by shuffle.  Read through
  // ld8 per column group instead, every one of the four groups of a chunk waits for an L2
  // round trip (L1 is swept by the matrix reads).
  // AB_EP_ROWMASK: operands known at code-generation time to be [1, N] rows.  Those are read
  // 8 values at a time with two 128-bit loads at a warp-uniform address (one wavefront each, L1
  // hits after the first warp of the CTA) at the point of use, instead of one value per lane plus
  // 32 SHFL.IDX per chunk.  Not read a chunk ahead: 32 more live registers per row operand
  // make the dout region spill within the epilogue warpgroup's 168.  A row operand that is
  // only recognised at run time keeps the one-register shuffle path.
#ifndef AB_EP_ROWMASK
#define AB_EP_ROWMASK 0
#endif
  static __device__ __forceinline__ constexpr bool is_row_op(int k) { return ((AB_EP_ROWMASK >> k) & 1) != 0; }
  struct ChunkPre {
    // [M, N] reads of the next chunk.  Register-only builds: this lane's row, 32 columns.
    // AB_EP_STAGED builds: the COALESCED layout -- q[i] = row 4 i + lane / 8 of the warp's 32,
    // columns 4 (lane % 8) .. + 3, so that every LDG.128 covers four full 128-byte lines
    // (read row-per-lane, an instruction touches 32 lines, 16 bytes of each: the loads then
    // queue in the LSU) -- and turned
    // into the row-per-lane layout through the staging buffer at the top of fused_eval.
#if AB_EP_CIN
#if AB_EP_STAGED
    float4 cinq[8];
#else
    float cin[32];
#endif
#endif
#if AB_EP_PRE_OP >= 0
#if AB_EP_STAGED
    float4 opq[8];
#else
    float op[32];
#endif
#endif
    float vec[AB_EP_NOPS > 0 ? AB_EP_NOPS : 1];
  };
  __device__ __forceinline__ void prefetch_chunk(ChunkPre& pre, long long row, long long col0, bool live,
                                                 const FusedScalars& sc, int lane) const {
    const long long r = live ? row : 0;
    (void)r; (void)sc; (void)pre; (void)col0;
#pragma unroll
    for (int k = 0; k < AB_EP_NOPS; ++k) {
      if (sc.vec[k] && !is_row_op(k)) {
        pre.vec[k] = (col0 + lane < p.N) ? __ldg(p.ep_ptr[k] + col0 + lane) : 0.0f;
      }
    }
#if AB_EP_STAGED
    {
      const long long row0 = row - lane, col = col0 + 4 * (lane & 7);
      (void)row0; (void)col;
#if AB_EP_CIN
      if (p.beta != 0.0f) {
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const long long grow = row0 + 4 * i + (lane >> 3);
          pre.cinq[i] = (grow < p.M && col < p.N) ? __ldcs(reinterpret_cast<const float4*>(p.Cin + grow * p.cin_rs + col))
                                                  : make_float4(0.0f, 0.0f, 0.0f, 0.0f);
        }
      }
#endif
#if AB_EP_PRE_OP >= 0
      if (!sc.is[AB_EP_PRE_OP] && p.ep_cs[AB_EP_PRE_OP] == 1) {
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const long long grow = row0 + 4 * i + (lane >> 3);
          pre.opq[i] = (grow < p.M && col < p.N)
                           ? __ldcs(reinterpret_cast<const float4*>(p.ep_ptr[AB_EP_PRE_OP] + grow * p.ep_rs[AB_EP_PRE_OP] + col))
                           : make_float4(0.0f, 0.0f, 0.0f, 0.0f);
        }
      }
#endif
    }
#else
#if AB_EP_CIN
    if (live && p.beta != 0.0f) {
#pragma unroll
      for (int j = 0; j < 32; j += 8)
        if (col0 + j < p.N) ld8<true>(p.Cin + r * p.cin_rs + col0 + j, *reinterpret_cast<float(*)[8]>(&pre.cin[j]), wide_in);
    }
#endif
#if AB_EP_PRE_OP >= 0
    if (live && !sc.is[AB_EP_PRE_OP] && p.ep_cs[AB_EP_PRE_OP] == 1) {
      const bool wide = ((reinterpret_cast<uintptr_t>(p.ep_ptr[AB_EP_PRE_OP]) & 31) == 0) && ((p.ep_rs[AB_EP_PRE_OP] & 7) == 0);
#pragma unroll
      for (int j = 0; j < 32; j += 8)
        if (col0 + j < p.N)
          ld8<true>(p.ep_ptr[AB_EP_PRE_OP] + r * p.ep_rs[AB_EP_PRE_OP] + col0 + j, *reinterpret_cast<float(*)[8]>(&pre.op[j]), wide);
    }
#endif
#endif
  }
#if AB_EP_STAGED
  // coalesced layout (ChunkPre) -> this lane's row, through the staging buffer
  __device__ __forceinline__ void restage(const float4 (&q)[8], float (&out)[32], int lane) const {
#pragma unroll
    for (int i = 0; i < 8; ++i) sts128(stage + 4u * st_off(4 * i + (lane >> 3), lane & 7), q[i].x, q[i].y, q[i].z, q[i].w);
    __syncwarp();
#pragma unroll
    for (int g = 0; g < 8; ++g) {
      const float4 v = lds128(stage + 4u * st_off(lane, g));
      out[4 * g] = v.x; out[4 * g + 1] = v.y; out[4 * g + 2] = v.z; out[4 * g + 3] = v.w;
    }
    __syncwarp();
  }
#endif
  // ---- one 32-column chunk of one accumulator row, in two parts -------------------------
  // fused_eval:   x[32] (raw accumulator values of columns col0 .. col0+31 of `row`) -> the
  //               region's values; consumes the read-ahead buffer `pre`, stores the outputs and
  //               their natural bf16 planes, adds to the thread's total `fs`, and leaves the
  //               value that is reduced / transposed in x[] (0 for rows and columns outside).
  // fused_reduce: the cross-lane part: column sums of the warp's 32 rows and the transposed
  //               bf16 plane.
  // The caller issues the NEXT chunk's reads between the two: `pre` is dead after fused_eval,
  // and the ~300 shuffle/select instructions of fused_reduce give those reads their latency.
  // (Two alternating buffers and a loop body of two chunks would do the same at twice the code,
  // and the larger body waits on instruction fetch.)
  __device__ __forceinline__ void fused_eval(float (&x)[32], long long row, long long col0, bool live,
                                             int lane, const FusedScalars& sc, FF& fs, const ChunkPre& pre) const {
    const long long r = live ? row : 0;
    (void)lane; (void)fs;
#if AB_EP_PRE_OP >= 0
    const bool pre_ok = live && !sc.is[AB_EP_PRE_OP] && p.ep_cs[AB_EP_PRE_OP] == 1;
#endif
#if AB_EP_STAGED
#if AB_EP_CIN
    float cin_l[32];
    if (p.beta != 0.0f) restage(pre.cinq, cin_l, lane);
#endif
#if AB_EP_PRE_OP >= 0
    float op_l[32];
    if (!sc.is[AB_EP_PRE_OP] && p.ep_cs[AB_EP_PRE_OP] == 1) restage(pre.opq, op_l, lane);
#endif
#else
#if AB_EP_CIN
    const float (&cin_l)[32] = pre.cin;
#endif
#if AB_EP_PRE_OP >= 0
    const float (&op_l)[32] = pre.op;
#endif
#endif
#pragma unroll
    for (int j = 0; j < 32; j += 8) {
      const long long col = col0 + j;
      // row operands: column j + t's value sits in lane j + t (all 32 lanes take part)
      float ev[AB_EP_NOPS > 0 ? AB_EP_NOPS : 1][8];
#pragma unroll
      for (int k = 0; k < AB_EP_NOPS; ++k) {
        if (is_row_op(k) && sc.vec[k]) {
          // N % 8 == 0 and 16-byte aligned rows (the fused launch's contract)
          const bool in = col < p.N;
          const float4 a = in ? __ldg(reinterpret_cast<const float4*>(p.ep_ptr[k] + col)) : make_float4(0.0f, 0.0f, 0.0f, 0.0f);
          const float4 b = in ? __ldg(reinterpret_cast<const float4*>(p.ep_ptr[k] + col + 4)) : make_float4(0.0f, 0.0f, 0.0f, 0.0f);
          ev[k][0] = a.x; ev[k][1] = a.y; ev[k][2] = a.z; ev[k][3] = a.w;
          ev[k][4] = b.x; ev[k][5] = b.y; ev[k][6] = b.z; ev[k][7] = b.w;
        } else if (sc.vec[k]) {
#pragma unroll
          for (int t = 0; t < 8; ++t) ev[k][t] = __shfl_sync(0xffffffffu, pre.vec[k], j + t);
        }
      }
      if (live && col < p.N) {  // N % 8 == 0: a group of 8 columns is inside or outside as a whole
        float v[8];
#pragma unroll
        for (int t = 0; t < 8; ++t) v[t] = p.alpha * x[j + t];
        if (p.beta != 0.0f) {
#if AB_EP_CIN
#pragma unroll
          for (int t = 0; t < 8; ++t) v[t] += p.beta * cin_l[j + t];
#else
          float ci[8];
          ld8<true>(p.Cin + r * p.cin_rs + col, ci, wide_in);
#pragma unroll
          for (int t = 0; t < 8; ++t) v[t] += p.beta * ci[t];
#endif
        }
        float e[4][8];
#pragma unroll
        for (int k = 0; k < AB_EP_NOPS; ++k) {
#if AB_EP_PRE_OP >= 0
          if (k == AB_EP_PRE_OP && pre_ok) {
#pragma unroll
            for (int t = 0; t < 8; ++t) e[k][t] = op_l[j + t];
            continue;
          }
#endif
          if (sc.vec[k]) {
#pragma unroll
            for (int t = 0; t < 8; ++t) e[k][t] = ev[k][t];
          } else if (sc.is[k]) {
#pragma unroll
            for (int t = 0; t < 8; ++t) e[k][t] = sc.v[k];
          } else if (p.ep_cs[k] == 1) {
            ld8<true>(p.ep_ptr[k] + r * p.ep_rs[k] + col, e[k],
                ((reinterpret_cast<uintptr_t>(p.ep_ptr[k]) & 31) == 0) && ((p.ep_rs[k] & 7) == 0));
          } else {
            const float* q = p.ep_ptr[k] + r * p.ep_rs[k] + col * p.ep_cs[k];
#pragma unroll
            for (int t = 0; t < 8; ++t) e[k][t] = q[t * p.ep_cs[k]];
          }
        }
        float o[AB_EP_NOUT][8];
#pragma unroll
        for (int t = 0; t < 8; ++t) { AB_EP_EVAL(v[t], e, t, o); }
#if AB_EP_STAGED
        put_outputs<kStageValue>(o, r, col);
        sts128(stage + 4u * st_off(lane, j >> 2), o[kStageValue][0], o[kStageValue][1], o[kStageValue][2], o[kStageValue][3]);
        sts128(stage + 4u * st_off(lane, (j >> 2) + 1), o[kStageValue][4], o[kStageValue][5], o[kStageValue][6], o[kStageValue][7]);
#else
        put_outputs<-1>(o, r, col);
#if AB_EP_COLSUM >= 0
#pragma unroll
        for (int t = 0; t < 8; ++t) x[j + t] = o[AB_EP_COLSUM][t];
#elif AB_EP_TPLANE >= 0
#pragma unroll
        for (int t = 0; t < 8; ++t) x[j + t] = o[AB_EP_TPLANE][t];
#endif
#endif
#if AB_EP_FULLSUM >= 0
#if AB_EP_EXACT_SUMS
        {
          // four independent pairs per group of 8 (the single running pair was a chain of 8
          // dependent TwoSums per group), folded into the thread's total once per group
          FF q4[4];
#pragma unroll
          for (int t = 0; t < 4; ++t) {
            q4[t].hi = o[AB_EP_FULLSUM][t];
            q4[t].lo = 0.0f;
            ff_add(q4[t], o[AB_EP_FULLSUM][t + 4]);
          }
          ff_add(q4[0], q4[1]);
          ff_add(q4[2], q4[3]);
          ff_add(q4[0], q4[2]);
          ff_add(fs, q4[0]);
        }
#else
        {
          // reduced-precision products (tf32 / bf16 operands): 8 values summed as a float32
          // tree, the groups as float pairs
          const float* w = o[AB_EP_FULLSUM];
          ff_add(fs, __fadd_rn(__fadd_rn(__fadd_rn(w[0], w[1]), __fadd_rn(w[2], w[3])),
                               __fadd_rn(__fadd_rn(w[4], w[5]), __fadd_rn(w[6], w[7]))));
        }
#endif
#endif
      } else {
#if AB_EP_STAGED
        sts128(stage + 4u * st_off(lane, j >> 2), 0.0f, 0.0f, 0.0f, 0.0f);
        sts128(stage + 4u * st_off(lane, (j >> 2) + 1), 0.0f, 0.0f, 0.0f, 0.0f);
#elif AB_EP_COLSUM >= 0 || AB_EP_TPLANE >= 0
#pragma unroll
        for (int t = 0; t < 8; ++t) x[j + t] = 0.0f;
#endif
      }
    }
  }
  // ---- AB_EP_STAGED: the value that is stored / reduced / transposed goes through 4 KB of
  // shared memory per warp (a 32 x 32 float32 chunk, 16-byte groups XOR-swizzled with the row:
  // the SWIZZLE_128B pattern, conflict-free for the row writes of fused_eval, for the row
  // reads of pass 1 and for the column reads of pass 2):
  //   pass 1  lanes 8 i .. 8 i + 7 read one row as 8 float4 and store it as ONE full 128-byte
  //           line (float32 output) / 64 contiguous bytes (bf16 plane).  Stored from the
  //           accumulator layout (lane = row) every STG touches 32 different lines, half a
  //           sector each, and the epilogue warps wait on the store queue;
  //   pass 2  lane c reads column c (32 LDS, one per row): the transpose that took 48 shuffles
  //           and ~130 selects, and the column sum becomes 31 adds without any shuffle.
  // The buffers (4 warps x 4 KB) live behind the tile's accumulator, at the end of the operand
  // ring: the bf16 / tf32 ring keeps 4 stages with them (5 without), the hi/lo ring 2.
  static constexpr int kStageValue = AB_EP_COLSUM >= 0 ? AB_EP_COLSUM : (AB_EP_TPLANE >= 0 ? AB_EP_TPLANE : 0);
  static __device__ __forceinline__ uint32_t st_off(int r, int g) { return (uint32_t)(r * 32 + ((g ^ (r & 7)) << 2)); }
#if AB_EP_STAGED
  __device__ __forceinline__ void fused_reduce(float (&x)[32], long long row, long long col0, int lane) const {
    (void)x;
    __syncwarp();
    const long long row0 = row - lane;
    {
      float* dst = kStageValue == 0 ? p.C : p.out_ptr[kStageValue];
      const long long rs = kStageValue == 0 ? p.c_rs : p.out_rs[kStageValue];
      uint16_t* sp = static_cast<uint16_t*>(p.shadow[kStageValue]);
      if (dst != nullptr || sp != nullptr) {
        const int g = lane & 7;
        const long long col = col0 + 4 * g;
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const int r = 4 * i + (lane >> 3);
          const float4 v = lds128(stage + 4u * st_off(r, g));
          const long long grow = row0 + r;
          if (grow < p.M && col < p.N) {
            if (dst != nullptr) __stcs(reinterpret_cast<float4*>(dst + grow * rs + col), v);
            if (sp != nullptr) {
              uint32_t h0, h1;
              asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(h0) : "f"(v.y), "f"(v.x));
              asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(h1) : "f"(v.w), "f"(v.z));
              __stcs(reinterpret_cast<uint2*>(sp + grow * p.shadow_pitch[kStageValue] + col), make_uint2(h0, h1));
            }
          }
        }
      }
    }
#if AB_EP_COLSUM >= 0 || AB_EP_TPLANE >= 0
    {
#if AB_EP_TPLANE >= 0
      const bool want_t = p.shadow_t != nullptr;
#else
      const bool want_t = false;
#endif
      if (AB_EP_COLSUM >= 0 || want_t) {
        float v[32];
        const int cg = lane >> 2, cw = lane & 3;
#pragma unroll
        for (int r = 0; r < 32; ++r) v[r] = lds32(stage + 4u * (r * 32 + ((cg ^ (r & 7)) << 2) + cw));
        const long long c = col0 + lane;
#if AB_EP_COLSUM >= 0
        {
          // lane = column: its sum over the warp's 32 rows (rows / columns outside were staged
          // as zeros).  float pairs under the fp32-faithful policy, a float32 tree otherwise
          const long long rb = row >> 5;
#if AB_EP_EXACT_SUMS
          // a tree of float pairs (depth 5): one running pair would be a chain of 31 dependent
          // TwoSums per lane
          FF tp[16];
#pragma unroll
          for (int r = 0; r < 16; ++r) {
            tp[r].hi = v[2 * r];
            tp[r].lo = 0.0f;
            ff_add(tp[r], v[2 * r + 1]);
          }
#pragma unroll
          for (int w = 8; w >= 1; w >>= 1) {
#pragma unroll
            for (int r = 0; r < w; ++r) {
              tp[r] = tp[2 * r];
              ff_add(tp[r], tp[2 * r + 1]);
            }
          }
          const double tot = ff_double(tp[0]);
#else
          float t16[16];
#pragma unroll
          for (int r = 0; r < 16; ++r) t16[r] = __fadd_rn(v[2 * r], v[2 * r + 1]);
#pragma unroll
          for (int w = 8; w >= 1; w >>= 1) {
#pragma unroll
            for (int r = 0; r < w; ++r) t16[r] = __fadd_rn(t16[2 * r], t16[2 * r + 1]);
          }
          const double tot = (double)t16[0];
#endif
          if (rb * 32 < p.M && c < p.N) p.colsum_ws[rb * p.N + c] = tot;
        }
#endif
#if AB_EP_TPLANE >= 0
        if (want_t && c < p.N && row0 < p.M) {
          uint16_t* dst = static_cast<uint16_t*>(p.shadow_t) + c * p.shadow_t_pitch + row0;
          if (row0 + 32 <= p.M) {
            uint32_t h[16];
#pragma unroll
            for (int t = 0; t < 16; ++t)
              asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(h[t]) : "f"(v[2 * t + 1]), "f"(v[2 * t]));
#pragma unroll
            for (int t = 0; t < 4; ++t)
              __stcs(reinterpret_cast<uint4*>(dst) + t, make_uint4(h[4 * t], h[4 * t + 1], h[4 * t + 2], h[4 * t + 3]));
          } else {
#pragma unroll
            for (int i = 0; i < 32; ++i)
              if (row0 + i < p.M) {
                uint16_t b;
                asm("cvt.rn.bf16.f32 %0, %1;" : "=h"(b) : "f"(v[i]));
                dst[i] = b;
              }
          }
        }
#endif
      }
    }
#endif
    __syncwarp();  // the buffer is free for the next chunk's values
  }
#else
  __device__ __forceinline__ void fused_reduce(float (&x)[32], long long row, long long col0, int lane) const {
    (void)x; (void)row; (void)col0; (void)lane;
#if AB_EP_TPLANE >= 0
    // Transposed bf16 plane, first half: rows are lanes, so two vertically adjacent values sit
    // in lanes l and l ^ 1.  Even lanes keep the even columns, odd lanes the odd ones: after
    // one exchange, P[i] of lane l is column 2 i + (l & 1) of the row pair (l & ~1, l | 1),
    // packed (low half = even row).  The remaining four exchanges (below, after the column
    // sums have consumed x[]) work on 16 packed registers instead of 32 floats.
    uint32_t P[16];
    const bool want_t = p.shadow_t != nullptr;
    if (want_t) {
      const bool odd = (lane & 1) != 0;
#pragma unroll
      for (int i = 0; i < 16; ++i) {
        const float mine = odd ? x[2 * i + 1] : x[2 * i];
        const float send = odd ? x[2 * i] : x[2 * i + 1];
        const float got = __shfl_xor_sync(0xffffffffu, send, 1);
        uint32_t h;  // low half <- second source operand
        asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(h) : "f"(got), "f"(mine));
        P[i] = __byte_perm(h, 0u, odd ? 0x1032u : 0x3210u);
      }
    }
#endif
#if AB_EP_COLSUM >= 0
    {
      // 32 x 32 transpose-reduce over the warp's rows: after the step with distance h every
      // lane keeps the half of its columns selected by bit h of its lane index; lane l ends
      // with the sum of column col0 + l.  The reference's CAReduce accumulates float32 sums in
      // float64 (tensor/elemwise.py:1371-1385): under the fp32-faithful policy the 32 rows are
      // added as float pairs (see FF above); under the tf32 / bf16 policies -- the addends
      // carry 2^-11 / 2^-8 relative error themselves -- as a float32 tree.  Either way the
      // partial sum leaves the warp as float64.
      const long long rb = row >> 5;  // row - lane is a multiple of 32
#if AB_EP_EXACT_SUMS
      FF d[16];
      {
        const bool up = (lane & 16) != 0;
#pragma unroll
        for (int i = 0; i < 16; ++i) {
          const float keep = up ? x[16 + i] : x[i];
          const float send = up ? x[i] : x[16 + i];
          d[i].hi = keep;
          d[i].lo = 0.0f;
          ff_add(d[i], __shfl_xor_sync(0xffffffffu, send, 16));
        }
      }
#define AB_COLSUM_STEP(H)                                                      \
      {                                                                        \
        const bool up = (lane & (H)) != 0;                                     \
        _Pragma("unroll") for (int i = 0; i < (H); ++i) {                      \
          const FF keep = up ? d[(H) + i] : d[i];                              \
          const FF send = up ? d[i] : d[(H) + i];                              \
          FF got;                                                              \
          got.hi = __shfl_xor_sync(0xffffffffu, send.hi, (H));                 \
          got.lo = __shfl_xor_sync(0xffffffffu, send.lo, (H));                 \
          d[i] = keep;                                                         \
          ff_add(d[i], got);                                                   \
        }                                                                      \
      }
      AB_COLSUM_STEP(8) AB_COLSUM_STEP(4) AB_COLSUM_STEP(2) AB_COLSUM_STEP(1)
#undef AB_COLSUM_STEP
      if (rb * 32 < p.M && col0 + lane < p.N) p.colsum_ws[rb * p.N + col0 + lane] = ff_double(d[0]);
#else
#define AB_COLSUM_STEP(H)                                                      \
      {                                                                        \
        const bool up = (lane & (H)) != 0;                                     \
        _Pragma("unroll") for (int i = 0; i < (H); ++i) {                      \
          const float keep = up ? x[(H) + i] : x[i];                           \
          const float send = up ? x[i] : x[(H) + i];                           \
          x[i] = __fadd_rn(keep, __shfl_xor_sync(0xffffffffu, send, (H)));     \
        }                                                                      \
      }
      AB_COLSUM_STEP(16) AB_COLSUM_STEP(8) AB_COLSUM_STEP(4) AB_COLSUM_STEP(2) AB_COLSUM_STEP(1)
#undef AB_COLSUM_STEP
      if (rb * 32 < p.M && col0 + lane < p.N) p.colsum_ws[rb * p.N + col0 + lane] = (double)x[0];
#endif
    }
#endif
#if AB_EP_TPLANE >= 0
    if (want_t) {
      // second half: register index bit b <-> lane bit b + 1 (b = 0..3).  Before: lane bits
      // 1..4 = row pair k, register index i = column / 2.  After: lane l = column col0 + l,
      // P[k] = rows (row0 + 2 k, row0 + 2 k + 1): 64 contiguous bytes of the transposed plane.
#define AB_T_STEP(B)                                                            \
      {                                                                         \
        const bool up = (lane & (2 << (B))) != 0;                               \
        _Pragma("unroll") for (int i = 0; i < 16; ++i) {                        \
          if ((i & (1 << (B))) == 0) {                                          \
            const uint32_t send = up ? P[i] : P[i | (1 << (B))];                \
            const uint32_t got = __shfl_xor_sync(0xffffffffu, send, 2 << (B));  \
            if (up) P[i] = got; else P[i | (1 << (B))] = got;                   \
          }                                                                     \
        }                                                                       \
      }
      AB_T_STEP(0) AB_T_STEP(1) AB_T_STEP(2) AB_T_STEP(3)
#undef AB_T_STEP
      const long long row0 = row - lane;
      const long long c = col0 + lane;
      if (c < p.N && row0 < p.M) {
        uint16_t* dst = static_cast<uint16_t*>(p.shadow_t) + c * p.shadow_t_pitch + row0;
        if (row0 + 32 <= p.M) {
#pragma unroll
          for (int t = 0; t < 4; ++t)
            __stcs(reinterpret_cast<uint4*>(dst) + t, make_uint4(P[4 * t], P[4 * t + 1], P[4 * t + 2], P[4 * t + 3]));
        } else {
#pragma unroll
          for (int i = 0; i < 32; ++i)
            if (row0 + i < p.M) dst[i] = (uint16_t)((i & 1) ? (P[i >> 1] >> 16) : (P[i >> 1] & 0xffffu));
        }
      }
    }
#endif
  }
#endif  // AB_EP_STAGED
  __device__ __forceinline__ void finish_fullsum(const FF& acc, long long row, long long n0, int lane) const {
#if AB_EP_FULLSUM >= 0
    double fs = ff_double(acc);
#pragma unroll
    for (int h = 16; h >= 1; h >>= 1) fs += __shfl_xor_sync(0xffffffffu, fs, h);
    const long long rb = row >> 5;
    if (lane == 0 && rb * 32 < p.M) p.fullsum_ws[rb * p.fullsum_cols + n0 / (p.block_n >> 1)] = fs;
#endif
  }
  // the tile's accumulator (shared memory, see acc_off): 32 columns at a time in a rolled loop
  // -- 32 live accumulator registers, and the body exists once.  The total of a half tile
  // (fullsum_ws has one entry per 64 columns) is finished before the next half starts.  Once
  // the last chunk's values have been consumed, the warp arrives on `acc_free`.
  __device__ __forceinline__ void store_fused(uint32_t acc_base, int r, long long row, long long n0, int nchunks,
                                              int lane, const FusedScalars& sc, uint64_t* acc_free) const {
    const bool live = row < p.M;
    const int half_chunks = p.block_n >> 6;
    FF fs = {0.0f, 0.0f};
    ChunkPre pre;
    prefetch_chunk(pre, row, n0, live, sc, lane);
#pragma unroll 1
    for (int c = 0; c < nchunks; ++c) {
      float x[32];
      acc_ld_x32(acc_base, r, c * 32, x);
      const long long col0 = n0 + c * 32;
      fused_eval(x, row, col0, live, lane, sc, fs, pre);
      if (c + 1 == nchunks) {
        __syncwarp();
        if (lane == 0) mbar_arrive(acc_free);
      }
      if (c + 1 < nchunks) prefetch_chunk(pre, row, col0 + 32, live, sc, lane);
      fused_reduce(x, row, col0, lane);
      if ((c + 1) % half_chunks == 0) {
        finish_fullsum(fs, row, col0 + 32 - (p.block_n >> 1), lane);
        fs = FF{0.0f, 0.0f};
      }
    }
  }
#endif  // AB_EPILOGUE
};

// Work unit -> (K range, tile).  Units are K-range major and, inside a K range, follow a grouped
// order (groups of p.group_m tile rows, columns outer, rows inner): the units in flight then
// form a compact block of the tile grid over ONE K range, so they share A and B panels in L2
// instead of re-reading the B operand for every tile row.
#define AB_UNIT_DECODE                                                          \
  const int split = (int)(unit / p.num_tiles);                                  \
  const long long tile_lin = unit - (long long)split * p.num_tiles;             \
  const long long tiles_m_ = p.num_tiles / p.tiles_n;                           \
  const long long gsz_ = (long long)p.group_m * p.tiles_n;                      \
  const long long first_m_ = (tile_lin / gsz_) * p.group_m;                     \
  const long long gm_ = min((long long)p.group_m, tiles_m_ - first_m_);         \
  const long long loc_ = tile_lin % gsz_;                                       \
  const long long tile_m = first_m_ + loc_ % gm_;                               \
  const long long tile_n = loc_ / gm_;                                          \
  const int kb_begin = split * p.kb_per_split;                                  \
  const int kb_end = min(kb_begin + p.kb_per_split, p.num_k_blocks);            \
  (void)split; (void)tile_m; (void)tile_n;

// one k-block of an MMA warpgroup: 4 K steps of 32 bytes, 3 products each for the
// hi/lo split (NP == 2: small cross terms first, the dominant hi*hi term last)
template <int KIND, int TA, int TB, int NP>
__device__ __forceinline__ void mma_kblock(float (&d)[64], uint32_t a_hi, uint32_t a_lo, uint32_t b_hi,
                                           uint32_t b_lo, uint32_t a_kstep, uint32_t b_kstep, uint32_t a_lbo,
                                           uint32_t b_lbo, bool fresh) {
#pragma unroll
  for (int k = 0; k < SW_BYTES / 32; ++k) {
    const uint32_t ka = k * a_kstep, kb_off = k * b_kstep;
    const uint32_t acc = (!fresh || k > 0) ? 1u : 0u;
    if (KIND == 1) {
      wgmma_m64n128k16_bf16<TA, TB>(d, make_smem_desc(a_hi + ka, a_lbo), make_smem_desc(b_hi + kb_off, b_lbo), acc);
    } else if (NP == 2) {
      wgmma_m64n128k8_tf32(d, make_smem_desc(a_lo + ka, a_lbo), make_smem_desc(b_hi + kb_off, b_lbo), acc);
      wgmma_m64n128k8_tf32(d, make_smem_desc(a_hi + ka, a_lbo), make_smem_desc(b_lo + kb_off, b_lbo), 1u);
      wgmma_m64n128k8_tf32(d, make_smem_desc(a_hi + ka, a_lbo), make_smem_desc(b_hi + kb_off, b_lbo), 1u);
    } else {
      wgmma_m64n128k8_tf32(d, make_smem_desc(a_hi + ka, a_lbo), make_smem_desc(b_hi + kb_off, b_lbo), acc);
    }
  }
}

// CL > 1 (ahead-of-time kernels, AB_GEMM_CLUSTER4): a cluster of CL CTAs stacked along M computes
// one (CL * 128) x 128 tile; they share the B tile, each CTA loading 1/CL of it and multicasting
// that part into the shared memory of all CL CTAs (cp.async.bulk.tensor ... multicast::cluster).
// A ring stage of a CTA is then written by every CTA of the cluster, so it is free only when the
// MMA warpgroups of all of them have released it: every MMA warp arrives on the empty barrier of
// every CTA (count 8 * CL).  The arithmetic per output element is the single-CTA kernel's.
template <int CL>
__device__ __forceinline__ void release_stage(uint64_t* bar) {
  if (CL == 1) {
    mbar_arrive(bar);
  } else {
#pragma unroll
    for (uint32_t c = 0; c < (uint32_t)CL; ++c) mbar_arrive_cluster(bar, c);
  }
}
template <int CL>
__device__ __forceinline__ void load_b_part(uint8_t* dst, const CUtensorMap* map, uint64_t* bar, int kc,
                                            int n0, uint32_t crank, const OperandLoad& o, int b_tile_bytes,
                                            int block_n, int k_per_kb) {
  constexpr uint16_t mask = (uint16_t)((1u << CL) - 1u);
  if (!o.mn_major) {
    // K-major: box {128 B of K, block_n / CL rows}, this CTA's rows of the tile
    tma_load_2d_mc(dst + crank * (b_tile_bytes / CL), map, bar, kc, n0 + (int)crank * (block_n / CL), mask);
  } else {
    // MN-major: box {128 B of MN, k_per_kb / CL K rows} per chunk, this CTA's K rows of each chunk
    for (int c = 0; c < o.chunks; ++c)
      tma_load_2d_mc(dst + c * o.chunk_bytes + crank * (o.chunk_bytes / CL), map, bar, n0 + c * o.mn_per_chunk,
                     kc + (int)crank * (k_per_kb / CL), mask);
  }
}

// The MMA warpgroups' unit loop for ONE operand layout, fixed at compile time: TA / TB = 1 for an
// MN-major A / B (bf16 only), NP = 2 for the hi/lo split.  gemm_body picks the instantiation
// once, before the loop.  A layout chosen by a branch around each k-block's wgmmas cost the
// pipelining: ptxas closes a wgmma group at the end of each branch (warning C7519), the commit
// after the join then commits an empty group, and wait_group 1 waits for the real k-block.
// The accumulator d is declared once, outside the segment loop, and nothing but wgmma writes it
// between the fence and the wait: a fresh segment starts with scale-d = 0 on its first wgmma,
// and acc_fold reads d only after wait_group 0.  So wait_group 1 keeps the previous k-block in
// flight, and the only full waits are the segment drains.  Every field of p the loop reads is
// copied into a local before it (see OperandLoad).
template <int KIND, int TA, int TB, int NP, int CL>
__device__ __forceinline__ void mma_loop(const GemmParams& p, uint32_t ring, uint64_t* full_bar, uint64_t* empty_bar,
                                         uint64_t* acc_full, uint64_t* acc_empty, uint32_t acc_base,
                                         long long group, long long n_groups, int cw, int lane, int mma_row0) {
  const long long num_units = p.num_units, num_tiles = p.num_tiles;
  const int kb_per_split = p.kb_per_split, num_k_blocks = p.num_k_blocks, seg_kblocks = p.seg_kblocks;
  const int stages = p.stages;
  const uint32_t stage_bytes = (uint32_t)p.stage_bytes;
  const uint32_t a_tile_bytes = (uint32_t)p.a_tile_bytes, b_tile_bytes = (uint32_t)p.b_tile_bytes;
  const uint32_t chunk_bytes = (uint32_t)p.chunk_bytes;
  const uint32_t a_kstep = (uint32_t)p.a_kstep, b_kstep = (uint32_t)p.b_kstep;
  const uint32_t a_lbo = TA ? chunk_bytes : 16u, b_lbo = TB ? chunk_bytes : 16u;
  // this warpgroup's 64 rows of the A tile: 64 K-major rows of 128 B, or MN chunk cw
  const uint32_t a_off = TA ? (uint32_t)cw * chunk_bytes : (uint32_t)(cw * 64 * SW_BYTES);
  const uint32_t b_off = NP * a_tile_bytes;
  float d[64], tot[64];
  // Defined once, before any wgmma: a segment's first wgmma ignores d (scale-d = 0), but the
  // CUDA 12.8 ptxas (NVRTC as bundled with PyTorch) counts an undefined accumulator input as a
  // non-wgmma definition inside the pipeline stage and serialises every wgmma of the kernel
  // (C7515: one wait_group 0 after each).
#pragma unroll
  for (int i = 0; i < 64; ++i) d[i] = 0.0f;
  int stage = 0;
  uint32_t phase = 0, acc_phase = 0;
  for (long long unit = group; unit < num_units; unit += n_groups) {
    const int split = (int)(unit / num_tiles);  // the K range of the unit (AB_UNIT_DECODE)
    const int kb_begin = split * kb_per_split;
    const int kb_end = min(kb_begin + kb_per_split, num_k_blocks);
#pragma unroll
    for (int i = 0; i < 64; ++i) tot[i] = -0.0f;
    for (int kb0 = kb_begin; kb0 < kb_end; kb0 += seg_kblocks) {
      const int kb1 = min(kb0 + seg_kblocks, kb_end);
      int prev = -1;
      for (int kb = kb0; kb < kb1; ++kb) {
        mbar_wait(&full_bar[stage], phase);
        const uint32_t sbase = ring + (uint32_t)stage * stage_bytes;
        const uint32_t a_hi = sbase + a_off, b_hi = sbase + b_off;
        wgmma_fence();
        mma_kblock<KIND, TA, TB, NP>(d, a_hi, a_hi + a_tile_bytes, b_hi, b_hi + b_tile_bytes, a_kstep, b_kstep,
                                     a_lbo, b_lbo, kb == kb0);
        wgmma_commit();
        // the previous k-block's products have retired: its stage goes back to the producer
        wgmma_wait<1>();
        if (prev >= 0 && lane == 0) release_stage<CL>(&empty_bar[prev]);
        prev = stage;
        if (++stage == stages) { stage = 0; phase ^= 1; }
      }
      wgmma_wait<0>();
      if (lane == 0) release_stage<CL>(&empty_bar[prev]);
      acc_fold(tot, d);
    }
    // the shared accumulator is free once the epilogue warps have read the previous unit
    // (parity 1 of the fresh barrier counts as complete: the first unit does not wait)
    mbar_wait(acc_empty, acc_phase ^ 1);
    acc_phase ^= 1;
    acc_store(acc_base, tot, mma_row0, lane);
    __syncwarp();
    if (lane == 0) mbar_arrive(acc_full);
  }
}

// LAYOUT: the MMA loop's layout, fixed by the kernel -- 2 * a_mn + b_mn for KIND 1, nparts for
// KIND 0 -- or -1: chosen from p at run time, once, before the unit loop (the ahead-of-time
// kernels).  The NVRTC build has one entry point per layout instead: with the four bf16 loops in
// one kernel, the CUDA 12.8 ptxas spills in the larger epilogue regions (560-byte stack frame).
template <int KIND, int CL = 1, int LAYOUT = -1>
__device__ __forceinline__ void gemm_body(const CUtensorMap& map_a0, const CUtensorMap& map_a1,
                                          const CUtensorMap& map_b0, const CUtensorMap& map_b1,
                                          const GemmParams& p) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  // dynamic smem base is only guaranteed 16-byte aligned: round up to 1024 for SWIZZLE_128B
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) &
                                             ~static_cast<uintptr_t>(1023));
  __shared__ __align__(8) uint64_t full_bar[8];
  __shared__ __align__(8) uint64_t empty_bar[8];
  __shared__ __align__(8) uint64_t acc_full;   // the shared accumulator holds a finished unit
  __shared__ __align__(8) uint64_t acc_empty;  // ... and has been read by the epilogue

  const int warp = threadIdx.x >> 5;
  const int stage_bytes = p.stage_bytes;
  const long long num_units = p.num_units;
  // persistent tile scheduler: CTA b handles units b, b + gridDim.x, ... (AB_UNIT_DECODE)
  // behind the operand ring: the tile's float32 accumulator, then (AB_EP_STAGED) the epilogue's
  // per-warp staging chunks
  const uint32_t acc_base = smem_u32(smem + (size_t)p.stages * p.stage_bytes);
  const uint32_t crank = CL > 1 ? cluster_ctarank() : 0u;  // position of this CTA along M
  const long long group = blockIdx.x / CL, n_groups = gridDim.x / CL;

  if (threadIdx.x == 0) {
    for (int s = 0; s < p.stages; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], CL * kMmaThreads / 32);  // one arrival per MMA warp (of each CTA)
    }
    mbar_init(&acc_full, kMmaThreads / 32);
    mbar_init(&acc_empty, kEpiThreads / 32);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  }
  __syncthreads();
  if (CL > 1) cluster_sync_all();  // every CTA's barriers exist before any multicast or remote arrive

  if (warp < kMmaWarp0) {
    AB_SETMAXNREG_CONTROL(CL);
    if (warp == 0 && elect_one()) {
      // ================= TMA producer =================
      asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&map_a0)) : "memory");
      asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&map_b0)) : "memory");
      int stage = 0;
      uint32_t phase = 0;
      const OperandLoad la = operand_load_a(p), lb = operand_load_b(p);
      const int nparts = p.nparts, a_tile_bytes = p.a_tile_bytes, b_tile_bytes = p.b_tile_bytes;
      const int stages = p.stages, k_per_kb = p.k_elems_per_row, block_n = p.block_n;
      for (long long unit = group; unit < num_units; unit += n_groups) {
        AB_UNIT_DECODE
        const int m0 = (int)(tile_m * (CL * BLOCK_M)) + (int)crank * BLOCK_M;
        const int n0 = (int)(tile_n * block_n);
        for (int kb = kb_begin; kb < kb_end; ++kb) {
          mbar_wait(&empty_bar[stage], phase ^ 1);
          uint8_t* sbase = smem + (size_t)stage * stage_bytes;
          mbar_expect_tx(&full_bar[stage], (uint32_t)stage_bytes);
          const int kc = kb * k_per_kb;
          load_tile(sbase, &map_a0, &full_bar[stage], kc, m0, la);
          if (nparts == 2) load_tile(sbase + a_tile_bytes, &map_a1, &full_bar[stage], kc, m0, la);
          if (CL == 1) {
            load_tile(sbase + nparts * a_tile_bytes, &map_b0, &full_bar[stage], kc, n0, lb);
            if (nparts == 2)
              load_tile(sbase + 2 * a_tile_bytes + b_tile_bytes, &map_b1, &full_bar[stage], kc, n0, lb);
          } else {
            load_b_part<CL>(sbase + nparts * a_tile_bytes, &map_b0, &full_bar[stage], kc, n0, crank, lb,
                            b_tile_bytes, block_n, k_per_kb);
            if (nparts == 2)
              load_b_part<CL>(sbase + 2 * a_tile_bytes + b_tile_bytes, &map_b1, &full_bar[stage], kc, n0, crank,
                              lb, b_tile_bytes, block_n, k_per_kb);
          }
          if (++stage == stages) { stage = 0; phase ^= 1; }
        }
      }
    }
  } else if (warp < kEpiWarp0) {
    AB_SETMAXNREG_MMA(CL);
    // ================= MMA warpgroups (warps 4..11) =================
    const int cw = (warp - kMmaWarp0) >> 2;  // tile rows [64 cw, 64 cw + 64)
    uint32_t lane_reg;
    asm volatile("mov.u32 %0, %%laneid;" : "=r"(lane_reg));
    const int lane = (int)lane_reg;
    const int mma_row0 = 64 * cw + 16 * (warp & 3);  // first accumulator row of this warp's fragment
    const uint32_t ring = smem_u32(smem);
#define AB_MMA_LOOP(TA, TB, NP)                                                                          \
  mma_loop<KIND, TA, TB, NP, CL>(p, ring, full_bar, empty_bar, &acc_full, &acc_empty, acc_base, group, n_groups, \
                                 cw, lane, mma_row0)
    if constexpr (LAYOUT >= 0) {
      if constexpr (KIND == 0) AB_MMA_LOOP(0, 0, LAYOUT == 1 ? 1 : 2);
      else AB_MMA_LOOP((LAYOUT >> 1) & 1, LAYOUT & 1, 1);
    } else if (KIND == 0) {  // tf32 operands are always K-major (plan_operand)
      if (p.nparts == 2) AB_MMA_LOOP(0, 0, 2);
      else AB_MMA_LOOP(0, 0, 1);
    } else if (p.a_mn) {
      if (p.b_mn) AB_MMA_LOOP(1, 1, 1);
      else AB_MMA_LOOP(1, 0, 1);
    } else {
      if (p.b_mn) AB_MMA_LOOP(0, 1, 1);
      else AB_MMA_LOOP(0, 0, 1);
    }
#undef AB_MMA_LOOP
  } else {
    AB_SETMAXNREG_EPILOGUE(CL);
    // ================= epilogue warpgroup (warps 12..15) =================
    uint32_t lane_reg;
    asm volatile("mov.u32 %0, %%laneid;" : "=r"(lane_reg));
    const int lane = (int)lane_reg;
    const int q = warp & 3;       // tile rows [32 q, 32 q + 32), one per lane
    const int r = q * 32 + lane;
    uint32_t acc_phase = 0;
    for (long long unit = group; unit < p.num_units; unit += n_groups) {
      AB_UNIT_DECODE
      const long long m0 = tile_m * (CL * BLOCK_M) + (long long)crank * BLOCK_M;
      const long long n0 = tile_n * p.block_n;
      // built per tile: held across the wait, the epilogue's state would cost the larger
      // generated regions their registers
#if AB_EP_STAGED
      const EpilogueOut eo(p, acc_base + kAccBytes + (uint32_t)(q * kStageBytesPerWarp));
#else
      const EpilogueOut eo(p);
#endif
      mbar_wait(&acc_full, acc_phase);
      acc_phase ^= 1;
#ifdef AB_EPILOGUE
      const EpilogueOut::FusedScalars sc = eo.load_scalars();  // the region's [1, 1] operands
      eo.store_fused(acc_base, r, m0 + r, n0, p.block_n >> 5, lane, sc, &acc_empty);  // fused launches are never split along K
#else
#pragma unroll 1
      for (int h = 0; h < BLOCK_N / kAccRegs; ++h) {
        float acc[kAccRegs];
#pragma unroll
        for (int c = 0; c < kAccRegs / 32; ++c)
          acc_ld_x32(acc_base, r, h * kAccRegs + c * 32, *reinterpret_cast<float(*)[32]>(&acc[c * 32]));
        if (split == 0) eo.store(acc, m0 + r, n0 + h * kAccRegs, kAccRegs / 32);
        else eo.store_partial(acc, m0 + r, n0 + h * kAccRegs, kAccRegs / 32, split);
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(&acc_empty);
#endif
    }
  }
  if (CL > 1) cluster_sync_all();  // no CTA leaves while another may still multicast into it
}

#if AB_EP_STAGED
extern "C" __global__ void ab_gemm_ep_staged_marker() {}  // tells gemm_run to reserve kStageBytes
#endif
#ifdef AB_EPILOGUE
// NVRTC build: C-linkage entry points, one per MMA-loop layout (the module is loaded by name
// from gemm_run, which picks the kernel of the packed operands' layout)
#define AB_EP_KERNEL(NAME, KIND, LAYOUT)                                                               \
  extern "C" __global__ void __launch_bounds__(kGemmThreads, 1)                                       \
  NAME(const __grid_constant__ CUtensorMap a0, const __grid_constant__ CUtensorMap a1,                 \
       const __grid_constant__ CUtensorMap b0, const __grid_constant__ CUtensorMap b1,                 \
       const __grid_constant__ GemmParams p) { gemm_body<KIND, 1, LAYOUT>(a0, a1, b0, b1, p); }
AB_EP_KERNEL(ab_gemm_ep_tf32, 0, 2)     // 3xTF32: hi/lo planes
AB_EP_KERNEL(ab_gemm_ep_tf32_1p, 0, 1)  // one TF32 pass
AB_EP_KERNEL(ab_gemm_ep_f16, 1, 0)      // bf16, A and B K-major
AB_EP_KERNEL(ab_gemm_ep_f16_km, 1, 1)   // bf16, B MN-major
AB_EP_KERNEL(ab_gemm_ep_f16_mk, 1, 2)   // bf16, A MN-major
AB_EP_KERNEL(ab_gemm_ep_f16_mm, 1, 3)   // bf16, A and B MN-major
#undef AB_EP_KERNEL
#endif
