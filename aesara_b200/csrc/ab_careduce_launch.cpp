// ab_careduce_launch.cpp — host side of the CAReduce kernels (ab_careduce.cuh).
//
// The reference builds a C loop nest ordered "kept dims outer, reduced dims
// inner" (aesara/tensor/elemwise.py:1560-1590, elemwise_cgen.py:502-570).  Here
// the same (shape, strides, reduce-mask) description is canonicalised — size-1
// dims dropped, neighbours of equal kind merged — and mapped to one of two
// access patterns, with the reduced range split across CTAs when there are too
// few outputs to fill the 132 SMs (two deterministic stages through `workspace`).
#include <algorithm>
#include <vector>

#include "ab_common.h"

using namespace ab;

namespace {

struct RedParamsHost {  // mirrors AbRedParams
  const void* in;
  void* out;
  long long n_keep, n_red;
  int nk, nr;
  long long keep_shape[AB_MAX_DIMS], keep_stride[AB_MAX_DIMS];
  long long red_shape[AB_MAX_DIMS], red_stride[AB_MAX_DIMS];
  long long split, slice;
  int vec_ok, pad_;
};

struct Plan {
  RedParamsHost p{};
  bool cols = false;
  long long split = 1;
};

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

int make_plan(int ndim, const int64_t* shape, const int64_t* strides, const int32_t* mask,
              int in_itemsize, Plan* plan) {
  if (ndim < 0 || ndim > AB_MAX_RAW_DIMS) return fail(AB_ERR_INVALID, "bad ndim %d", ndim);
  struct Dim { long long n, s; int red; };
  std::vector<Dim> dims;
  long long n_keep = 1, n_red = 1;
  for (int d = 0; d < ndim; ++d) {
    if (shape[d] < 0) return fail(AB_ERR_INVALID, "negative dimension");
    if (mask[d]) n_red *= shape[d]; else n_keep *= shape[d];
    if (shape[d] == 1) continue;
    dims.push_back({shape[d], strides ? strides[d] : 0, mask[d] ? 1 : 0});
  }
  for (int d = (int)dims.size() - 2; d >= 0; --d) {
    if (dims[d].red == dims[d + 1].red && dims[d].s == dims[d + 1].s * dims[d + 1].n) {
      dims[d].n *= dims[d + 1].n;
      dims[d].s = dims[d + 1].s;
      dims.erase(dims.begin() + d + 1);
    }
  }
  RedParamsHost& p = plan->p;
  p.n_keep = n_keep;
  p.n_red = n_red;
  p.nk = p.nr = 0;
  int last_keep = -1, last_red = -1;
  for (size_t i = 0; i < dims.size(); ++i) {
    if (dims[i].red) {
      if (p.nr == AB_MAX_DIMS) return fail(AB_ERR_UNSUPPORTED, "too many reduced dims");
      p.red_shape[p.nr] = dims[i].n; p.red_stride[p.nr] = dims[i].s; ++p.nr; last_red = (int)i;
    } else {
      if (p.nk == AB_MAX_DIMS) return fail(AB_ERR_UNSUPPORTED, "too many kept dims");
      p.keep_shape[p.nk] = dims[i].n; p.keep_stride[p.nk] = dims[i].s; ++p.nk; last_keep = (int)i;
    }
  }
  if (p.nr == 0) { p.nr = 1; p.red_shape[0] = n_red; p.red_stride[0] = 0; }  // n_red is 1 (or 0)
  const int vec = std::max(1, 16 / in_itemsize);
  const long long target = (long long)sm_count() * 8;
  // leading-axis pattern: [R, K] with K contiguous
  plan->cols = (p.nk == 1 && p.nr == 1 && p.keep_stride[0] == 1 && last_keep > last_red &&
                n_keep >= 64);
  long long split = 1;
  if (n_keep > 0 && n_red > 0) {
    if (plan->cols) {
      const long long gx = (n_keep + 255) / 256;
      split = std::max<long long>(1, std::min<long long>(target / gx, n_red / 32));
    } else if (n_keep < target) {
      const long long per_cta = 256LL * vec * 8;  // elements one CTA chews before it is worth splitting
      split = std::max<long long>(1, std::min<long long>((target + n_keep - 1) / n_keep,
                                                        (n_red + per_cta - 1) / per_cta));
    }
    split = std::min<long long>(split, 65535);
  }
  long long slice = n_red > 0 ? (n_red + split - 1) / split : 0;
  if (!plan->cols) slice = (slice + vec - 1) / vec * vec;  // keep 16-byte alignment per slice
  if (slice > 0) split = (n_red + slice - 1) / slice;
  p.split = split;
  p.slice = slice;
  plan->split = split;
  return AB_OK;
}

int launch(Module* m, int which, const RedParamsHost& p, dim3 grid, cudaStream_t st) {
  cudaKernel_t kern;
  int rc = m->get(which, &kern);
  if (rc) return rc;
  RedParamsHost copy = p;
  void* args[1] = {&copy};
  AB_CUDA(cudaLaunchKernel((const void*)kern, grid, dim3(256), args, 0, st));
  g_launches.fetch_add(1, std::memory_order_relaxed);
  return AB_OK;
}

}  // namespace

extern "C" int ab_careduce_workspace_bytes(int ndim, const int64_t* shape,
                                           const int32_t* reduce_mask, int acc_itemsize,
                                           size_t* bytes) {
  if (!bytes) return fail(AB_ERR_INVALID, "null out pointer");
  // strides are unknown here: assume the worst case (a split is used)
  long long n_keep = 1, n_red = 1;
  for (int d = 0; d < ndim; ++d) (reduce_mask[d] ? n_red : n_keep) *= shape[d];
  const long long target = (long long)sm_count() * 8;
  long long split = std::min<long long>(65535, std::max<long long>(1, target));
  if (n_keep >= target) {
    const long long gx = (n_keep + 255) / 256;
    split = std::max<long long>(1, target / gx);
  }
  *bytes = (size_t)(std::max<long long>(n_keep, 1) * (split + 1)) * (size_t)acc_itemsize;
  return AB_OK;
}

extern "C" int ab_careduce_launch(ab_module* mod, int ndim, const int64_t* shape,
                                  const int64_t* in_strides, const int32_t* reduce_mask,
                                  const void* in, void* out, void* workspace,
                                  size_t workspace_bytes, int in_itemsize, int acc_itemsize,
                                  int out_itemsize, void* stream) {
  Module* m = reinterpret_cast<Module*>(mod);
  if (!m) return fail(AB_ERR_INVALID, "null module");
  (void)out_itemsize;
  Plan plan;
  int rc = make_plan(ndim, shape, in_strides, reduce_mask, in_itemsize, &plan);
  if (rc) return rc;
  RedParamsHost& p = plan.p;
  if (p.n_keep == 0) return AB_OK;
  cudaStream_t st = as_stream(stream);
  const int vec = std::max(1, 16 / in_itemsize);
  p.in = in;
  p.vec_ok = 0;
  if (!plan.cols && p.nr == 1 && p.red_stride[0] == 1 && vec > 1 &&
      reinterpret_cast<uintptr_t>(in) % 16 == 0) {
    bool ok = true;
    for (int d = 0; d < p.nk; ++d) ok = ok && (p.keep_stride[d] % vec == 0);
    p.vec_ok = ok ? 1 : 0;
  }
  const bool two_stage = plan.split > 1;
  if (two_stage) {
    const size_t need = (size_t)p.n_keep * (size_t)plan.split * (size_t)acc_itemsize;
    if (!workspace || workspace_bytes < need)
      return fail(AB_ERR_INVALID, "CAReduce workspace too small: need %zu bytes, have %zu", need,
                  workspace_bytes);
  }
  if (plan.cols) {
    dim3 grid((unsigned)((p.n_keep + 255) / 256), (unsigned)plan.split);
    p.out = two_stage ? workspace : out;
    rc = launch(m, two_stage ? Module::RED_COLS_P : Module::RED_COLS, p, grid, st);
    if (rc || !two_stage) return rc;
    RedParamsHost f{};
    f.in = workspace; f.out = out; f.n_keep = p.n_keep; f.n_red = plan.split;
    f.nk = 1; f.nr = 1; f.keep_shape[0] = p.n_keep; f.keep_stride[0] = 1;
    f.red_shape[0] = plan.split; f.red_stride[0] = p.n_keep; f.split = 1; f.slice = plan.split;
    return launch(m, Module::RED_COLS_F, f, dim3(grid.x, 1), st);
  }
  if (p.n_keep > 2147483647LL) return fail(AB_ERR_UNSUPPORTED, "too many outputs for the row pattern");
  dim3 grid((unsigned)p.n_keep, (unsigned)plan.split);
  p.out = two_stage ? workspace : out;
  rc = launch(m, two_stage ? Module::RED_ROWS_P : Module::RED_ROWS, p, grid, st);
  if (rc || !two_stage) return rc;
  RedParamsHost f{};
  f.in = workspace; f.out = out; f.n_keep = p.n_keep; f.n_red = plan.split;
  f.nk = 1; f.nr = 1; f.keep_shape[0] = p.n_keep; f.keep_stride[0] = plan.split;
  f.red_shape[0] = plan.split; f.red_stride[0] = 1; f.split = 1; f.slice = plan.split;
  return launch(m, Module::RED_ROWS_F, f, dim3((unsigned)p.n_keep, 1), st);
}
