// ab_runtime.cpp — device selection, error reporting, NVRTC JIT, module
// loading, events and raw memory helpers of libaesara_b200.so.
//
// Reference counterparts: the C-linker's module pipeline
// (aesara/link/c/cmodule.py:2482 GCC_compiler.compile_str, ModuleCache) and the
// failure protocol of compiled thunks (aesara/link/c/basic.py:93-124,
// lazylinker_c.c:501-520): integer status + an error message left for the
// Python side to raise through raise_with_op.
#include <nvrtc.h>

#include <cstdlib>
#include <mutex>
#include <vector>

#include "ab_common.h"

namespace ab {

std::string& last_error() {
  static thread_local std::string err;
  return err;
}

int fail(int code, const char* fmt, ...) {
  char buf[4096];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof(buf), fmt, ap);
  va_end(ap);
  last_error() = buf;
  return code;
}

std::atomic<uint64_t> g_launches{0};

static const char* kKernelNames[Module::N_KERNELS] = {
    "ab_ew_flat_vec", "ab_ew_flat", "ab_ew_rows_vec", "ab_ew_rows", "ab_ew_nd", "ab_ew_tile",
    "ab_red_rows",    "ab_red_rows_p", "ab_red_rows_f", "ab_red_cols", "ab_red_cols_p",
    "ab_red_cols_f"};

int Module::get(int which, cudaKernel_t* out) {
  if (!tried[which]) {
    tried[which] = true;
    cudaKernel_t kern = nullptr;
    cudaError_t e = cudaLibraryGetKernel(&kern, lib, kKernelNames[which]);
    if (e != cudaSuccess) {
      cudaGetLastError();
      k[which] = nullptr;
    } else {
      k[which] = kern;
    }
  }
  if (!k[which])
    return fail(AB_ERR_INVALID, "module has no kernel %s", kKernelNames[which]);
  *out = k[which];
  return AB_OK;
}

}  // namespace ab

using namespace ab;

extern "C" {

const char* ab_version(void) { return "aesara_b200 0.1 (sm_90a)"; }

const char* ab_last_error(void) { return last_error().c_str(); }

int ab_init(int device_ordinal) {
  int n = 0;
  cudaError_t e = cudaGetDeviceCount(&n);
  if (e != cudaSuccess || n == 0) {
    cudaGetLastError();
    return fail(AB_ERR_NO_DEVICE, "no CUDA device available (%s)",
                e == cudaSuccess ? "device count is 0" : cudaGetErrorString(e));
  }
  if (device_ordinal < 0 || device_ordinal >= n)
    return fail(AB_ERR_INVALID, "device ordinal %d out of range [0,%d)", device_ordinal, n);
  AB_CUDA(cudaSetDevice(device_ordinal));
  AB_CUDA(cudaFree(0));  // force context creation
  return AB_OK;
}

int ab_get_device_info(int device_ordinal, ab_device_info* out) {
  if (!out) return fail(AB_ERR_INVALID, "null ab_device_info");
  cudaDeviceProp p;
  AB_CUDA(cudaGetDeviceProperties(&p, device_ordinal));
  memset(out, 0, sizeof(*out));
  out->sm_count = p.multiProcessorCount;
  out->cc_major = p.major;
  out->cc_minor = p.minor;
  out->total_mem = p.totalGlobalMem;
  out->l2_bytes = (size_t)p.l2CacheSize;
  out->max_smem_per_block_optin = (int)p.sharedMemPerBlockOptin;
  strncpy(out->name, p.name, sizeof(out->name) - 1);
  return AB_OK;
}

int ab_stream_synchronize(void* stream) {
  AB_CUDA(cudaStreamSynchronize(as_stream(stream)));
  return AB_OK;
}

int ab_device_synchronize(void) {
  AB_CUDA(cudaDeviceSynchronize());
  return AB_OK;
}

int ab_malloc(void** dptr, size_t bytes, void* stream) {
  if (!dptr) return fail(AB_ERR_INVALID, "null out pointer");
  AB_CUDA(cudaMallocAsync(dptr, bytes ? bytes : 1, as_stream(stream)));
  return AB_OK;
}

int ab_free(void* dptr, void* stream) {
  if (dptr) AB_CUDA(cudaFreeAsync(dptr, as_stream(stream)));
  return AB_OK;
}

int ab_memcpy_h2d(void* dst, const void* src, size_t bytes, void* stream) {
  AB_CUDA(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyHostToDevice, as_stream(stream)));
  return AB_OK;
}

int ab_memcpy_d2h(void* dst, const void* src, size_t bytes, void* stream) {
  AB_CUDA(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToHost, as_stream(stream)));
  return AB_OK;
}

int ab_memset(void* dst, int value, size_t bytes, void* stream) {
  AB_CUDA(cudaMemsetAsync(dst, value, bytes, as_stream(stream)));
  return AB_OK;
}

int ab_event_create(void** ev) {
  cudaEvent_t e;
  AB_CUDA(cudaEventCreate(&e));
  *ev = e;
  return AB_OK;
}

int ab_event_record(void* ev, void* stream) {
  AB_CUDA(cudaEventRecord((cudaEvent_t)ev, as_stream(stream)));
  return AB_OK;
}

int ab_event_elapsed_ms(void* start, void* stop, float* ms) {
  AB_CUDA(cudaEventSynchronize((cudaEvent_t)stop));
  AB_CUDA(cudaEventElapsedTime(ms, (cudaEvent_t)start, (cudaEvent_t)stop));
  return AB_OK;
}

int ab_event_destroy(void* ev) {
  AB_CUDA(cudaEventDestroy((cudaEvent_t)ev));
  return AB_OK;
}

// ---------------------------------------------------------------- NVRTC ------
int ab_nvrtc_compile(const char* src, const char* name, const char* const* extra_opts,
                     int n_extra_opts, void** cubin, size_t* cubin_size) {
  if (!src || !cubin || !cubin_size) return fail(AB_ERR_INVALID, "null argument");
  nvrtcProgram prog;
  nvrtcResult r = nvrtcCreateProgram(&prog, src, name ? name : "ab_module.cu", 0, nullptr, nullptr);
  if (r != NVRTC_SUCCESS) return fail(AB_ERR_NVRTC, "nvrtcCreateProgram: %s", nvrtcGetErrorString(r));
  std::vector<const char*> opts = {"--gpu-architecture=sm_90a", "--std=c++17", "-lineinfo",
                                   "-default-device"};
  for (int i = 0; i < n_extra_opts; ++i) opts.push_back(extra_opts[i]);
  r = nvrtcCompileProgram(prog, (int)opts.size(), opts.data());
  if (r != NVRTC_SUCCESS) {
    size_t logsz = 0;
    nvrtcGetProgramLogSize(prog, &logsz);
    std::string log(logsz, '\0');
    if (logsz) nvrtcGetProgramLog(prog, &log[0]);
    nvrtcDestroyProgram(&prog);
    if (log.size() > 3500) log.resize(3500);
    return fail(AB_ERR_NVRTC, "NVRTC compilation of %s failed:\n%s", name ? name : "module",
                log.c_str());
  }
  size_t sz = 0;
  r = nvrtcGetCUBINSize(prog, &sz);
  if (r != NVRTC_SUCCESS || sz == 0) {
    nvrtcDestroyProgram(&prog);
    return fail(AB_ERR_NVRTC, "nvrtcGetCUBINSize: %s", nvrtcGetErrorString(r));
  }
  void* buf = malloc(sz);
  r = nvrtcGetCUBIN(prog, (char*)buf);
  nvrtcDestroyProgram(&prog);
  if (r != NVRTC_SUCCESS) {
    free(buf);
    return fail(AB_ERR_NVRTC, "nvrtcGetCUBIN: %s", nvrtcGetErrorString(r));
  }
  *cubin = buf;
  *cubin_size = sz;
  return AB_OK;
}

int ab_nvrtc_version(int* major, int* minor) {
  if (!major || !minor) return fail(AB_ERR_INVALID, "null argument");
  nvrtcResult r = nvrtcVersion(major, minor);
  if (r != NVRTC_SUCCESS) return fail(AB_ERR_NVRTC, "nvrtcVersion: %s", nvrtcGetErrorString(r));
  return AB_OK;
}

void ab_buffer_free(void* p) { free(p); }

int ab_module_load(const void* cubin, size_t cubin_size, ab_module** out) {
  if (!cubin || !out) return fail(AB_ERR_INVALID, "null argument");
  (void)cubin_size;
  cudaLibrary_t lib;
  AB_CUDA(cudaLibraryLoadData(&lib, cubin, nullptr, nullptr, 0, nullptr, nullptr, 0));
  Module* m = new Module();
  m->lib = lib;
  *out = reinterpret_cast<ab_module*>(m);
  return AB_OK;
}

int ab_kernel_launch(ab_module* mod, const char* name, unsigned grid_x, unsigned block_x,
                     size_t smem_bytes, void** args, void* stream) {
  Module* m = reinterpret_cast<Module*>(mod);
  if (!m || !name || !args) return fail(AB_ERR_INVALID, "null argument");
  if (grid_x == 0 || block_x == 0) return AB_OK;
  cudaKernel_t kern = nullptr;
  auto it = m->named.find(name);
  if (it == m->named.end()) {
    cudaError_t e = cudaLibraryGetKernel(&kern, m->lib, name);
    if (e != cudaSuccess) {
      cudaGetLastError();
      return fail(AB_ERR_INVALID, "module has no kernel %s", name);
    }
    m->named[name] = kern;
  } else {
    kern = it->second;
  }
  AB_CUDA(cudaLaunchKernel((const void*)kern, dim3(grid_x), dim3(block_x), args, smem_bytes,
                           as_stream(stream)));
  g_launches++;
  return AB_OK;
}

int ab_module_unload(ab_module* mod) {
  Module* m = reinterpret_cast<Module*>(mod);
  if (!m) return AB_OK;
  cudaError_t e = cudaLibraryUnload(m->lib);
  delete m;
  if (e != cudaSuccess) return fail(AB_ERR_CUDA, "cudaLibraryUnload: %s", cudaGetErrorString(e));
  return AB_OK;
}

uint64_t ab_launch_count(void) { return g_launches.load(); }

}  // extern "C"
