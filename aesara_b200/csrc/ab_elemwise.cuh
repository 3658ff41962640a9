// ab_elemwise.cuh — hand-written kernel skeleton for one fused
// Elemwise{Composite} node (reference: aesara/tensor/elemwise.py:835-1168 and
// the loop generators of aesara/tensor/elemwise_cgen.py:228-462).
//
// The Python code generator (aesara_b200/codegen/elemwise.py) emits, in front
// of this file:
//     #define AB_NIN / AB_NOUT / AB_VEC
//     #define AB_INPUTS(X)   X(0, float) X(1, float) ...        (k, element type)
//     #define AB_OUTPUTS(X)  X(0, float) ...
//     __device__ void ab_body(<in types...>, <out types&...>)   the scalar DAG
//     #define AB_CALL_BODY(IN, OUT) ab_body(IN(0), IN(1), ..., OUT(0), ...)
//
// Three kernels per module, each in a vectorised and a scalar flavour:
//   ab_ew_flat*  every operand is a contiguous run or a broadcast scalar
//                (element stride 1 or 0) — the 128-bit streaming path;
//   ab_ew_rows*  2-D [rows, cols] with inner stride 1/0 and arbitrary row
//                stride (bias broadcast [1,H]+[B,H], column-slice views);
//   ab_ew_tile   [batch,] rows x cols where some operands are contiguous along
//                the COLUMN index and others along the ROW index (a matrix and
//                a DimShuffle{1,0} view in one expression, a.T * b + 1): 32 x 32
//                tiles; operands contiguous along rows are read coalesced along
//                rows and turned through shared memory, so every global access
//                of the kernel is a full 128-byte line;
//   ab_ew_nd     anything else: DimShuffle / broadcast / negative strides
//                folded into index arithmetic (up to AB_MAX_DIMS merged dims).
// HBM-bound by construction: each operand element is read/written once.
#pragma once

#define AB_NOPS (AB_NIN + AB_NOUT)

struct AbEwParams {
  long long n;                  // number of output elements
  int ndim;                     // merged dims (ab_ew_nd), 1 (flat) or 2 (rows)
  int pad_;
  long long shape[AB_MAX_DIMS];
  void* ptr[AB_NOPS];           // inputs, then outputs
  long long stride[AB_NOPS][AB_MAX_DIMS];  // element strides, 0 = broadcast
};

#define AB_THREADS 256

// ------------------------------------------------------------------ flat ------
template <int VEC, int UNROLL>
__device__ __forceinline__ void ab_ew_flat_impl(const AbEwParams& p) {
  const long long nvec = p.n / VEC;
  const long long gstride = (long long)gridDim.x * AB_THREADS;
  long long v0 = (long long)blockIdx.x * AB_THREADS + threadIdx.x;

#define AB_DECL_IN(k, T)                                         \
  const T* ip##k = reinterpret_cast<const T*>(p.ptr[k]); \
  const bool bc##k = (p.stride[k][0] == 0);                      \
  T sc##k = T();                                                 \
  if (bc##k) sc##k = ip##k[0];
  AB_INPUTS(AB_DECL_IN)
#undef AB_DECL_IN
#define AB_DECL_OUT(k, T) T* op##k = reinterpret_cast<T*>(p.ptr[AB_NIN + k]);
  AB_OUTPUTS(AB_DECL_OUT)
#undef AB_DECL_OUT

  for (; v0 < nvec; v0 += gstride * UNROLL) {
#define AB_LD(k, T)                                               \
  ab_pack<T, VEC> in##k[UNROLL];                                  \
  _Pragma("unroll") for (int u = 0; u < UNROLL; ++u) {            \
    const long long v = v0 + u * gstride;                         \
    if (bc##k) {                                                  \
      _Pragma("unroll") for (int e = 0; e < VEC; ++e) in##k[u].v[e] = sc##k; \
    } else if (v < nvec) {                                        \
      ab_load_pack<T, VEC>(in##k[u], ip##k + v * VEC);            \
    }                                                             \
  }
    AB_INPUTS(AB_LD)
#undef AB_LD
#define AB_DO(k, T) ab_pack<T, VEC> out##k[UNROLL];
    AB_OUTPUTS(AB_DO)
#undef AB_DO
#pragma unroll
    for (int u = 0; u < UNROLL; ++u) {
      if (v0 + u * gstride < nvec) {
#pragma unroll
        for (int e = 0; e < VEC; ++e) {
#define AB_IN_E(k) in##k[u].v[e]
#define AB_OUT_E(k) out##k[u].v[e]
          AB_CALL_BODY(AB_IN_E, AB_OUT_E);
#undef AB_IN_E
#undef AB_OUT_E
        }
      }
    }
#define AB_ST(k, T)                                               \
  _Pragma("unroll") for (int u = 0; u < UNROLL; ++u) {            \
    const long long v = v0 + u * gstride;                         \
    if (v < nvec) ab_store_pack<T, VEC>(op##k + v * VEC, out##k[u]); \
  }
    AB_OUTPUTS(AB_ST)
#undef AB_ST
  }

  // tail (n % VEC elements) by the first threads of block 0
  if (VEC > 1 && blockIdx.x == 0) {
    const long long t = nvec * VEC + threadIdx.x;
    if (t < p.n) {
#define AB_TIN(k, T) const T tin##k = bc##k ? sc##k : ip##k[t];
      AB_INPUTS(AB_TIN)
#undef AB_TIN
#define AB_TOUT(k, T) T tout##k;
      AB_OUTPUTS(AB_TOUT)
#undef AB_TOUT
#define AB_IN_E(k) tin##k
#define AB_OUT_E(k) tout##k
      AB_CALL_BODY(AB_IN_E, AB_OUT_E);
#undef AB_IN_E
#undef AB_OUT_E
#define AB_TST(k, T) op##k[t] = tout##k;
      AB_OUTPUTS(AB_TST)
#undef AB_TST
    }
  }
}

extern "C" __global__ void __launch_bounds__(AB_THREADS, AB_MIN_BLOCKS)
ab_ew_flat_vec(const __grid_constant__ AbEwParams p) {
  ab_ew_flat_impl<AB_VEC, AB_UNROLL>(p);
}
extern "C" __global__ void __launch_bounds__(AB_THREADS)
ab_ew_flat(const __grid_constant__ AbEwParams p) {
  ab_ew_flat_impl<1, 4>(p);
}

// ------------------------------------------------------------------ rows ------
// shape = [rows, cols]; stride[k][1] in {0,1}; stride[k][0] arbitrary.
// grid.x covers column vectors, grid.y strides over rows.
template <int VEC, int UNROLL>
__device__ __forceinline__ void ab_ew_rows_impl(const AbEwParams& p) {
  const long long rows = p.shape[0];
  const long long cvec = p.shape[1] / VEC;  // launcher guarantees divisibility
  const long long cv = (long long)blockIdx.x * AB_THREADS + threadIdx.x;
  if (cv >= cvec) return;
#define AB_DECL_IN(k, T)                                               \
  const T* ip##k = reinterpret_cast<const T*>(p.ptr[k]) + \
                                (p.stride[k][1] ? cv * VEC : 0);      \
  const long long rs##k = p.stride[k][0];                              \
  const bool bc##k = (p.stride[k][1] == 0);
  AB_INPUTS(AB_DECL_IN)
#undef AB_DECL_IN
#define AB_DECL_OUT(k, T)                                              \
  T* op##k = reinterpret_cast<T*>(p.ptr[AB_NIN + k]) + cv * VEC;       \
  const long long ors##k = p.stride[AB_NIN + k][0];
  AB_OUTPUTS(AB_DECL_OUT)
#undef AB_DECL_OUT

  const long long rstep = gridDim.y;
  for (long long r0 = blockIdx.y; r0 < rows; r0 += rstep * UNROLL) {
#define AB_LD(k, T)                                               \
  ab_pack<T, VEC> in##k[UNROLL];                                  \
  _Pragma("unroll") for (int u = 0; u < UNROLL; ++u) {            \
    const long long r = r0 + u * rstep;                           \
    if (r < rows) {                                               \
      if (bc##k) {                                                \
        const T s = ip##k[r * rs##k];                             \
        _Pragma("unroll") for (int e = 0; e < VEC; ++e) in##k[u].v[e] = s; \
      } else {                                                    \
        ab_load_pack<T, VEC>(in##k[u], ip##k + r * rs##k);        \
      }                                                           \
    }                                                             \
  }
    AB_INPUTS(AB_LD)
#undef AB_LD
#define AB_DO(k, T) ab_pack<T, VEC> out##k[UNROLL];
    AB_OUTPUTS(AB_DO)
#undef AB_DO
#pragma unroll
    for (int u = 0; u < UNROLL; ++u) {
      if (r0 + u * rstep < rows) {
#pragma unroll
        for (int e = 0; e < VEC; ++e) {
#define AB_IN_E(k) in##k[u].v[e]
#define AB_OUT_E(k) out##k[u].v[e]
          AB_CALL_BODY(AB_IN_E, AB_OUT_E);
#undef AB_IN_E
#undef AB_OUT_E
        }
      }
    }
#define AB_ST(k, T)                                               \
  _Pragma("unroll") for (int u = 0; u < UNROLL; ++u) {            \
    const long long r = r0 + u * rstep;                           \
    if (r < rows) ab_store_pack<T, VEC>(op##k + r * ors##k, out##k[u]); \
  }
    AB_OUTPUTS(AB_ST)
#undef AB_ST
  }
}

extern "C" __global__ void __launch_bounds__(AB_THREADS, AB_MIN_BLOCKS)
ab_ew_rows_vec(const __grid_constant__ AbEwParams p) {
  ab_ew_rows_impl<AB_VEC, AB_UNROLL>(p);
}
extern "C" __global__ void __launch_bounds__(AB_THREADS)
ab_ew_rows(const __grid_constant__ AbEwParams p) {
  ab_ew_rows_impl<1, 4>(p);
}

// ------------------------------------------------------------------ tile ------
// shape = [R, C] (ndim 2) or [nb, R, C] (ndim 3).  Per operand: unit (or 0) stride along C
// ("row-major": read in output order) or unit stride along R with any stride along C
// ("column-major": staged through a 64 x 65 shared-memory tile).  Outputs are row-major.
// p.pad_ carries a bit mask of the column-major inputs; the launcher admits as many of them
// as tiles fit into the 48 KB of static shared memory (ab_ew_tile_slots).  Block = 32 x 8
// threads, 16 elements per thread: 16 independent loads per input in flight per thread.
#define AB_TILE 64
#ifndef AB_TILE_BAND
#define AB_TILE_BAND 1  // tile rows per CTA
#endif
__host__ __device__ constexpr int ab_max_input_size() {
  int m = 1;
#define AB_T_SZ(k, T) m = (int)sizeof(T) > m ? (int)sizeof(T) : m;
  AB_INPUTS(AB_T_SZ)
#undef AB_T_SZ
  return m;
}
__host__ __device__ constexpr int ab_ew_tile_slots() {
  return (48 * 1024) / (AB_TILE * (AB_TILE + 1) * ab_max_input_size());
}
extern "C" __global__ void __launch_bounds__(AB_THREADS)
ab_ew_tile(const __grid_constant__ AbEwParams p) {
  constexpr int kSlot = ab_max_input_size();
  constexpr int kSlots = ab_ew_tile_slots() > 0 ? ab_ew_tile_slots() : 1;
  __shared__ __align__(16) unsigned char tile_raw[kSlots * AB_TILE * (AB_TILE + 1) * kSlot];
#define AB_TSLOT(s, i, j) (tile_raw + ((((s) * AB_TILE + (i)) * (AB_TILE + 1) + (j)) * kSlot))
  const int nd = p.ndim;
  const long long R = p.shape[nd - 2], C = p.shape[nd - 1];
  const long long nb = nd == 3 ? p.shape[0] : 1;
  const long long tiles_c = (C + AB_TILE - 1) / AB_TILE, tiles_r = (R + AB_TILE - 1) / AB_TILE;
  const long long n_tiles = nb * tiles_r * tiles_c;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;  // 32 x 8
  const unsigned mask = (unsigned)p.pad_;
  for (long long t = blockIdx.x; t < n_tiles; t += gridDim.x) {
    // tile order: bands of AB_TILE_BAND tile rows, rows fastest inside a band (1 = row-major
    // tiles).  Wider bands make the tiles in flight cover AB_TILE_BAND * 256 contiguous bytes
    // of the turned operands, and measured slower (knob AB_EW_TILE_BAND kept for the sweep).
    const long long b = t / (tiles_r * tiles_c);
    const long long tb = t % (tiles_r * tiles_c);
    const long long band = tb / (AB_TILE_BAND * tiles_c), in_band = tb % (AB_TILE_BAND * tiles_c);
    const long long band_rows = (tiles_r - band * AB_TILE_BAND) < AB_TILE_BAND
                                    ? (tiles_r - band * AB_TILE_BAND) : AB_TILE_BAND;
    const long long tr = band * AB_TILE_BAND + in_band % band_rows, tc = in_band / band_rows;
    const long long r0 = tr * AB_TILE, c0 = tc * AB_TILE;
    // 1. column-major inputs: coalesced along rows -> shared[slot][c_local][r_local]
#define AB_T_STAGE(k, T)                                                              \
    if (mask & (1u << k)) {                                                           \
      const int slot = __popc(mask & ((1u << k) - 1u));                               \
      const T* ip = reinterpret_cast<const T*>(p.ptr[k]) + (nd == 3 ? b * p.stride[k][0] : 0); \
      const long long sr = p.stride[k][nd - 2], sc = p.stride[k][nd - 1];             \
      _Pragma("unroll") for (int i = 0; i < AB_TILE; i += 8) {                        \
        _Pragma("unroll") for (int h = 0; h < AB_TILE; h += 32) {                     \
          const long long r = r0 + tx + h, c = c0 + ty + i;                           \
          if (r < R && c < C)                                                         \
            *reinterpret_cast<T*>(AB_TSLOT(slot, ty + i, tx + h)) = ip[r * sr + c * sc]; \
        }                                                                             \
      }                                                                               \
    }
    AB_INPUTS(AB_T_STAGE)
#undef AB_T_STAGE
    __syncthreads();
    // 2. compute in output order (coalesced along columns)
#pragma unroll 4
    for (int i = 0; i < AB_TILE; i += 8) {
#pragma unroll
      for (int h = 0; h < AB_TILE; h += 32) {
        const long long r = r0 + ty + i, c = c0 + tx + h;
        if (r < R && c < C) {
#define AB_T_LD(k, T)                                                                 \
          T tin##k;                                                                   \
          if (mask & (1u << k)) {                                                     \
            tin##k = *reinterpret_cast<const T*>(AB_TSLOT(__popc(mask & ((1u << k) - 1u)), tx + h, ty + i)); \
          } else {                                                                    \
            const T* ip = reinterpret_cast<const T*>(p.ptr[k]) + (nd == 3 ? b * p.stride[k][0] : 0); \
            tin##k = ip[r * p.stride[k][nd - 2] + c * p.stride[k][nd - 1]];           \
          }
          AB_INPUTS(AB_T_LD)
#undef AB_T_LD
#define AB_T_OD(k, T) T tout##k;
          AB_OUTPUTS(AB_T_OD)
#undef AB_T_OD
#define AB_IN_E(k) tin##k
#define AB_OUT_E(k) tout##k
          AB_CALL_BODY(AB_IN_E, AB_OUT_E);
#undef AB_IN_E
#undef AB_OUT_E
#define AB_T_ST(k, T)                                                                 \
          (reinterpret_cast<T*>(p.ptr[AB_NIN + k]) + (nd == 3 ? b * p.stride[AB_NIN + k][0] : 0)) \
              [r * p.stride[AB_NIN + k][nd - 2] + c * p.stride[AB_NIN + k][nd - 1]] = tout##k;
          AB_OUTPUTS(AB_T_ST)
#undef AB_T_ST
        }
      }
    }
    __syncthreads();
  }
}

// -------------------------------------------------------------------- nd ------
extern "C" __global__ void __launch_bounds__(AB_THREADS)
ab_ew_nd(const __grid_constant__ AbEwParams p) {
  const long long gstride = (long long)gridDim.x * AB_THREADS;
  for (long long i = (long long)blockIdx.x * AB_THREADS + threadIdx.x; i < p.n; i += gstride) {
    long long off[AB_NOPS];
#pragma unroll
    for (int k = 0; k < AB_NOPS; ++k) off[k] = 0;
    long long rem = i;
    for (int d = p.ndim - 1; d >= 0; --d) {
      const long long sz = p.shape[d];
      const long long q = rem / sz;
      const long long idx = rem - q * sz;
      rem = q;
#pragma unroll
      for (int k = 0; k < AB_NOPS; ++k) off[k] += idx * p.stride[k][d];
    }
#define AB_NIN_LD(k, T) const T nin##k = reinterpret_cast<const T*>(p.ptr[k])[off[k]];
    AB_INPUTS(AB_NIN_LD)
#undef AB_NIN_LD
#define AB_NOUT_D(k, T) T nout##k;
    AB_OUTPUTS(AB_NOUT_D)
#undef AB_NOUT_D
#define AB_IN_E(k) nin##k
#define AB_OUT_E(k) nout##k
    AB_CALL_BODY(AB_IN_E, AB_OUT_E);
#undef AB_IN_E
#undef AB_OUT_E
#define AB_NOUT_ST(k, T) reinterpret_cast<T*>(p.ptr[AB_NIN + k])[off[AB_NIN + k]] = nout##k;
    AB_OUTPUTS(AB_NOUT_ST)
#undef AB_NOUT_ST
  }
}
