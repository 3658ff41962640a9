// ab_common.h — internal helpers of libaesara_b200.so (not part of the ABI)
#pragma once
#include <cuda_runtime.h>

#include <atomic>
#include <cstdarg>
#include <cstdio>
#include <cstring>
#include <map>
#include <string>
#include <vector>

#include "../../include/aesara_b200.h"

namespace ab {

std::string& last_error();
int fail(int code, const char* fmt, ...);
extern std::atomic<uint64_t> g_launches;

// The Elemwise launcher's dimension collapse (ab_elemwise_launch.cpp), shared with every launcher
// that walks several strided operands over one index space: drop size-1 dims, order the rest by
// |stride| of operand `order_by` (largest first, stable), and merge neighbours that are jointly
// contiguous for every operand.  strides[k*ndim + d] is operand k's stride along dim d; on return
// shp holds the merged extents and st[k] operand k's strides along them.
void collapse_dims(int nops, int ndim, const int64_t* shape, const int64_t* strides, int order_by,
                   std::vector<int64_t>& shp, std::vector<std::vector<int64_t>>& st);

inline cudaStream_t as_stream(void* s) { return reinterpret_cast<cudaStream_t>(s); }

struct Module {
  cudaLibrary_t lib = nullptr;
  // lazily resolved kernels (names fixed by the skeletons in csrc/*.cuh)
  enum { EW_FLAT_VEC, EW_FLAT, EW_ROWS_VEC, EW_ROWS, EW_ND, EW_TILE, RED_ROWS, RED_ROWS_P, RED_ROWS_F,
         RED_COLS, RED_COLS_P, RED_COLS_F, N_KERNELS };
  cudaKernel_t k[N_KERNELS] = {};
  bool tried[N_KERNELS] = {};
  std::map<std::string, cudaKernel_t> named;  // kernels launched by name (ab_kernel_launch)
  int get(int which, cudaKernel_t* out);
};

}  // namespace ab

#define AB_CUDA(call)                                                                   \
  do {                                                                                  \
    cudaError_t e_ = (call);                                                            \
    if (e_ != cudaSuccess)                                                              \
      return ab::fail(AB_ERR_CUDA, "%s failed: %s (%s:%d)", #call, cudaGetErrorString(e_), \
                      __FILE__, __LINE__);                                              \
  } while (0)
