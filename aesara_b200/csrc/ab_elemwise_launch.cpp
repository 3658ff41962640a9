// ab_elemwise_launch.cpp — host side of the fused Elemwise kernels.
//
// What the reference does per call inside the generated C thunk
// (aesara/tensor/elemwise.py:835-1168): run-time broadcast checks
// (elemwise_cgen.py:72-125), loop-order selection by output strides
// (make_reordered_loop, elemwise_cgen.py:305-462) and a contiguous fast path
// (elemwise.py:1103-1167).  Here the same decisions pick a kernel flavour:
//   1. drop size-1 dims, order dims by the first output's stride (largest first),
//      merge neighbours that are jointly contiguous for every operand;
//   2. one merged dim with strides in {0,1}            -> ab_ew_flat[_vec]
//      two merged dims with inner strides in {0,1}     -> ab_ew_rows[_vec]
//      [batch,] rows x cols, every operand contiguous
//      along rows or along columns (transposed views)  -> ab_ew_tile
//      otherwise                                       -> ab_ew_nd.
#include <algorithm>
#include <cstdlib>
#include <vector>

#include "ab_common.h"

using namespace ab;

namespace {

struct EwParamsHost {
  // mirrors AbEwParams in ab_elemwise.cuh for a given operand count
  std::vector<unsigned char> buf;
  int nops;
  explicit EwParamsHost(int nops_) : buf(8 + 8 + 8 * AB_MAX_DIMS + (size_t)nops_ * 8 +
                                         (size_t)nops_ * 8 * AB_MAX_DIMS, 0), nops(nops_) {}
  long long& n() { return *reinterpret_cast<long long*>(&buf[0]); }
  int& ndim() { return *reinterpret_cast<int*>(&buf[8]); }
  int& pad() { return *reinterpret_cast<int*>(&buf[12]); }
  long long* shape() { return reinterpret_cast<long long*>(&buf[16]); }
  void** ptr() { return reinterpret_cast<void**>(&buf[16 + 8 * AB_MAX_DIMS]); }
  long long* stride(int k) {
    return reinterpret_cast<long long*>(&buf[16 + 8 * AB_MAX_DIMS + (size_t)nops * 8 +
                                            (size_t)k * 8 * AB_MAX_DIMS]);
  }
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

}  // namespace

extern "C" int ab_elemwise_launch(ab_module* mod, int n_in, int n_out, int ndim,
                                  const int64_t* shape, void* const* ptrs,
                                  const int64_t* strides, const int32_t* itemsizes, int vec,
                                  int unroll, void* stream) {
  Module* m = reinterpret_cast<Module*>(mod);
  const int nops = n_in + n_out;
  if (!m) return fail(AB_ERR_INVALID, "null module");
  if (nops <= 0 || nops > AB_MAX_OPERANDS || n_out <= 0)
    return fail(AB_ERR_INVALID, "bad operand count %d in / %d out", n_in, n_out);
  if (ndim < 0 || ndim > AB_MAX_RAW_DIMS) return fail(AB_ERR_INVALID, "bad ndim %d", ndim);
  if (vec < 1 || unroll < 1) return fail(AB_ERR_INVALID, "bad vec/unroll");

  // 1. squeeze
  std::vector<int64_t> shp;
  std::vector<std::vector<int64_t>> st(nops);
  long long total = 1;
  for (int d = 0; d < ndim; ++d) {
    if (shape[d] < 0) return fail(AB_ERR_INVALID, "negative dimension");
    total *= shape[d];
  }
  if (total == 0) return AB_OK;  // nothing to compute (elemwise.py:738-746)
  for (int d = 0; d < ndim; ++d) {
    if (shape[d] == 1) continue;
    shp.push_back(shape[d]);
    for (int k = 0; k < nops; ++k) st[k].push_back(strides[(size_t)k * ndim + d]);
  }
  int nd = (int)shp.size();
  // outputs must not be broadcast
  for (int k = n_in; k < nops; ++k)
    for (int d = 0; d < nd; ++d)
      if (st[k][d] == 0) return fail(AB_ERR_INVALID, "output operand %d has a broadcast stride", k - n_in);

  // 2. order dims by |stride| of the first output, largest first (stable)
  if (nd > 1) {
    std::vector<int> perm(nd);
    for (int d = 0; d < nd; ++d) perm[d] = d;
    const std::vector<int64_t>& os = st[n_in];
    std::stable_sort(perm.begin(), perm.end(),
                     [&](int a, int b) { return std::llabs(os[a]) > std::llabs(os[b]); });
    std::vector<int64_t> shp2(nd);
    std::vector<std::vector<int64_t>> st2(nops, std::vector<int64_t>(nd));
    for (int d = 0; d < nd; ++d) {
      shp2[d] = shp[perm[d]];
      for (int k = 0; k < nops; ++k) st2[k][d] = st[k][perm[d]];
    }
    shp.swap(shp2);
    st.swap(st2);
  }
  // 3. merge neighbours (d, d+1) when stride[d] == stride[d+1]*shape[d+1] for all operands
  for (int d = nd - 2; d >= 0; --d) {
    bool ok = true;
    for (int k = 0; k < nops && ok; ++k) ok = (st[k][d] == st[k][d + 1] * shp[d + 1]);
    if (ok) {
      shp[d] *= shp[d + 1];
      shp.erase(shp.begin() + d + 1);
      for (int k = 0; k < nops; ++k) {
        st[k][d] = st[k][d + 1];
        st[k].erase(st[k].begin() + d + 1);
      }
      --nd;
    }
  }
  if (nd > AB_MAX_DIMS)
    return fail(AB_ERR_UNSUPPORTED, "Elemwise over %d non-mergeable dims (max %d)", nd, AB_MAX_DIMS);
  if (nd == 0) {  // a single element
    nd = 1;
    shp.assign(1, 1);
    for (int k = 0; k < nops; ++k) st[k].assign(1, k < n_in ? 0 : 1);
  }

  EwParamsHost P(nops);
  P.n() = total;
  P.ndim() = nd;
  for (int d = 0; d < nd; ++d) P.shape()[d] = shp[d];
  for (int k = 0; k < nops; ++k) {
    P.ptr()[k] = ptrs[k];
    for (int d = 0; d < nd; ++d) P.stride(k)[d] = st[k][d];
  }

  auto inner_unit = [&](int d) {
    for (int k = 0; k < nops; ++k)
      if (st[k][d] != 0 && st[k][d] != 1) return false;
    return true;
  };
  auto aligned = [&](int k, int64_t extra_stride_elems) {
    const size_t bytes = (size_t)itemsizes[k] * vec;
    if (reinterpret_cast<uintptr_t>(ptrs[k]) % bytes) return false;
    if (extra_stride_elems % vec) return false;
    return true;
  };

  const int sms = sm_count();
  const unsigned threads = 256;
  int which;
  dim3 grid(1, 1, 1);
  if (nd == 1 && inner_unit(0)) {
    bool v = vec > 1 && total >= vec;
    for (int k = 0; k < nops && v; ++k)
      if (st[k][0] == 1) v = aligned(k, 0);
    const long long per_block = (long long)threads * (v ? vec * unroll : 4);
    long long blocks = (total + per_block - 1) / per_block;
    blocks = std::max<long long>(1, std::min<long long>(blocks, (long long)sms * 32));
    grid.x = (unsigned)blocks;
    which = v ? Module::EW_FLAT_VEC : Module::EW_FLAT;
  } else if (nd == 2 && inner_unit(1)) {
    bool v = vec > 1 && (shp[1] % vec == 0);
    for (int k = 0; k < nops && v; ++k) {
      if (st[k][1] == 1) v = aligned(k, st[k][0]);
    }
    const long long cvec = v ? shp[1] / vec : shp[1];
    const int u = v ? unroll : 4;
    long long gx = (cvec + threads - 1) / threads;
    if (gx > 2147483647LL) return fail(AB_ERR_UNSUPPORTED, "row too long");
    long long gy = (shp[0] + u - 1) / u;
    const long long target = (long long)sms * 16;
    gy = std::min<long long>(gy, std::max<long long>(1, target / gx));
    gy = std::max<long long>(1, std::min<long long>(gy, 65535));
    grid.x = (unsigned)gx;
    grid.y = (unsigned)gy;
    which = v ? Module::EW_ROWS_VEC : Module::EW_ROWS;
  } else {
    // [batch,] rows x cols with every operand contiguous along the rows OR the columns (a
    // matrix and a DimShuffle{1,0} view in one expression): the tiled kernel turns the
    // row-contiguous inputs through shared memory
    bool tiled = (nd == 2 || nd == 3) && n_in <= 16 && getenv("AB_EW_NO_TILE") == nullptr &&
                 shp[nd - 1] >= 16 && shp[nd - 2] >= 16;
    unsigned colmajor = 0;
    for (int k = 0; k < nops && tiled; ++k) {
      const int64_t sr = st[k][nd - 2], sc = st[k][nd - 1];
      if (itemsizes[k] > 8) tiled = false;
      else if (sc == 0 || sc == 1) continue;                       // read in output order
      else if (k < n_in && (sr == 1 || sr == 0)) colmajor |= 1u << k;  // turned in shared memory
      else tiled = false;
    }
    int max_item = 1, staged = 0;
    for (int k = 0; k < n_in; ++k) {
      max_item = std::max(max_item, (int)itemsizes[k]);
      staged += (colmajor >> k) & 1u;
    }
    // 64 x 65 tiles of the widest input type in 48 KB of static shared memory (ab_ew_tile_slots)
    if (tiled && staged > (48 * 1024) / (64 * 65 * max_item)) tiled = false;
    if (tiled && colmajor) {
      const long long tiles = (nd == 3 ? shp[0] : 1) * ((shp[nd - 2] + 63) / 64) * ((shp[nd - 1] + 63) / 64);
      grid.x = (unsigned)std::max<long long>(1, std::min<long long>(tiles, (long long)sms * 32));
      P.pad() = (int)colmajor;
      which = Module::EW_TILE;
    } else {
      long long blocks = (total + threads - 1) / threads;
      blocks = std::max<long long>(1, std::min<long long>(blocks, (long long)sms * 32));
      grid.x = (unsigned)blocks;
      which = Module::EW_ND;
    }
  }

  cudaKernel_t kern;
  int rc = m->get(which, &kern);
  if (rc) return rc;
  void* args[1] = {P.buf.data()};
  AB_CUDA(cudaLaunchKernel((const void*)kern, grid, dim3(threads), args, 0, as_stream(stream)));
  g_launches.fetch_add(1, std::memory_order_relaxed);
  return AB_OK;
}
