"""ctypes binding of ``libaesara_b200.so`` (the C ABI in ``include/aesara_b200.h``).

There is no CPU fallback: if the shared library is missing this module raises
``RuntimeError`` at import of the product path.
"""

from __future__ import annotations

import ctypes as C
import hashlib
import os
import threading

from .. import build as _build

_lib = None
_lock = threading.Lock()

c_i64p = C.POINTER(C.c_int64)
c_i32p = C.POINTER(C.c_int32)
c_voidpp = C.POINTER(C.c_void_p)


class AbError(RuntimeError):
    def __init__(self, code, msg):
        super().__init__(msg)
        self.code = code


class DeviceInfo(C.Structure):
    _fields_ = [
        ("sm_count", C.c_int),
        ("cc_major", C.c_int),
        ("cc_minor", C.c_int),
        ("total_mem", C.c_size_t),
        ("l2_bytes", C.c_size_t),
        ("max_smem_per_block_optin", C.c_int),
        ("name", C.c_char * 128),
    ]


# name -> (restype, argtypes); must list every symbol include/aesara_b200.h declares
SIGNATURES = {
    "ab_init": (C.c_int, [C.c_int]),
    "ab_get_device_info": (C.c_int, [C.c_int, C.POINTER(DeviceInfo)]),
    "ab_last_error": (C.c_char_p, []),
    "ab_version": (C.c_char_p, []),
    "ab_stream_synchronize": (C.c_int, [C.c_void_p]),
    "ab_device_synchronize": (C.c_int, []),
    "ab_malloc": (C.c_int, [c_voidpp, C.c_size_t, C.c_void_p]),
    "ab_free": (C.c_int, [C.c_void_p, C.c_void_p]),
    "ab_memcpy_h2d": (C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]),
    "ab_memcpy_d2h": (C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]),
    "ab_memset": (C.c_int, [C.c_void_p, C.c_int, C.c_size_t, C.c_void_p]),
    "ab_event_create": (C.c_int, [c_voidpp]),
    "ab_event_record": (C.c_int, [C.c_void_p, C.c_void_p]),
    "ab_event_elapsed_ms": (C.c_int, [C.c_void_p, C.c_void_p, C.POINTER(C.c_float)]),
    "ab_event_destroy": (C.c_int, [C.c_void_p]),
    "ab_nvrtc_compile": (
        C.c_int,
        [C.c_char_p, C.c_char_p, C.POINTER(C.c_char_p), C.c_int, c_voidpp, C.POINTER(C.c_size_t)],
    ),
    "ab_nvrtc_version": (C.c_int, [c_i32p, c_i32p]),
    "ab_buffer_free": (None, [C.c_void_p]),
    "ab_module_load": (C.c_int, [C.c_void_p, C.c_size_t, c_voidpp]),
    "ab_module_unload": (C.c_int, [C.c_void_p]),
    "ab_elemwise_launch": (
        C.c_int,
        [C.c_void_p, C.c_int, C.c_int, C.c_int, c_i64p, c_voidpp, c_i64p, c_i32p, C.c_int,
         C.c_int, C.c_void_p],
    ),
    "ab_elemwise_path_count": (C.c_uint64, [C.c_int]),
    "ab_careduce_workspace_bytes": (
        C.c_int, [C.c_int, c_i64p, c_i32p, C.c_int, C.POINTER(C.c_size_t)]
    ),
    "ab_careduce_launch": (
        C.c_int,
        [C.c_void_p, C.c_int, c_i64p, c_i64p, c_i32p, C.c_void_p, C.c_void_p, C.c_void_p,
         C.c_size_t, C.c_int, C.c_int, C.c_int, C.c_void_p],
    ),
    "ab_gemv": (
        C.c_int,
        [C.c_int, C.c_int64, C.c_int64, C.c_double, C.c_void_p, C.c_int64, C.c_int64,
         C.c_void_p, C.c_int64, C.c_double, C.c_void_p, C.c_int64, C.c_void_p, C.c_size_t,
         C.c_void_p],
    ),
    "ab_gemv_workspace_bytes": (
        C.c_int, [C.c_int, C.c_int64, C.c_int64, C.c_int64, C.c_int64, C.POINTER(C.c_size_t)]
    ),
    "ab_ger": (
        C.c_int,
        [C.c_int, C.c_int64, C.c_int64, C.c_double, C.c_void_p, C.c_int64, C.c_void_p,
         C.c_int64, C.c_void_p, C.c_int64, C.c_int64, C.c_void_p],
    ),
    "ab_gemm": (
        C.c_int,
        [C.c_int, C.c_int, C.c_int64, C.c_int64, C.c_int64, C.c_double, C.c_void_p, C.c_int64,
         C.c_int64, C.c_void_p, C.c_int64, C.c_int64, C.c_double, C.c_void_p, C.c_int64,
         C.c_int64, C.c_void_p, C.c_size_t, C.c_void_p],
    ),
    "ab_gemm_workspace_bytes": (
        C.c_int,
        [C.c_int, C.c_int, C.c_int64, C.c_int64, C.c_int64, C.c_int64, C.c_int64, C.c_int64,
         C.c_int64, C.POINTER(C.c_size_t)],
    ),
    "ab_ravel_index": (
        C.c_int,
        [C.c_int, C.POINTER(C.c_void_p), C.POINTER(C.c_int64), C.POINTER(C.c_int64), C.c_int64,
         C.c_void_p, C.c_int, C.c_void_p],
    ),
    "ab_cumulative": (
        C.c_int,
        [C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_int64, C.c_int64, C.c_int64, C.c_void_p],
    ),
    "ab_arange": (
        C.c_int,
        [C.c_int, C.c_double, C.c_double, C.c_int64, C.c_int64, C.c_int64, C.c_void_p, C.c_void_p],
    ),
    "ab_kernel_launch": (
        C.c_int,
        [C.c_void_p, C.c_char_p, C.c_uint, C.c_uint, C.c_size_t, C.POINTER(C.c_void_p), C.c_void_p],
    ),
    "ab_gemm_pack_bytes": (
        C.c_int, [C.c_int, C.c_int64, C.c_int64, C.c_int64, C.c_int64, C.POINTER(C.c_size_t)]
    ),
    "ab_gemm_pack": (
        C.c_int,
        [C.c_int, C.c_void_p, C.c_int64, C.c_int64, C.c_int64, C.c_int64, C.c_void_p, C.c_size_t,
         C.c_void_p, C.c_void_p],
    ),
    "ab_gemm_pack_kmajor_bytes": (
        C.c_int, [C.c_int, C.c_int64, C.c_int64, C.c_int64, C.c_int64, C.POINTER(C.c_size_t)]
    ),
    "ab_gemm_pack_kmajor": (
        C.c_int,
        [C.c_int, C.c_void_p, C.c_int64, C.c_int64, C.c_int64, C.c_int64, C.c_void_p, C.c_size_t,
         C.c_void_p, C.c_void_p],
    ),
    "ab_gemm_packed": (
        C.c_int,
        [C.c_int, C.c_int64, C.c_int64, C.c_int64, C.c_double, C.c_void_p, C.c_void_p, C.c_double,
         C.c_void_p, C.c_int64, C.c_int64, C.c_void_p, C.c_int64, C.c_int64, C.c_void_p, C.c_size_t,
         C.c_void_p],
    ),
    "ab_gemm_packed_fused": (
        C.c_int,
        [C.c_int, C.c_int64, C.c_int64, C.c_int64, C.c_double, C.c_void_p, C.c_void_p, C.c_double,
         C.c_void_p, C.c_int64, C.c_int64, C.c_void_p, C.c_int64, C.c_int64, C.c_void_p, C.c_void_p],
    ),
    "ab_gemm_packed_workspace_bytes": (
        C.c_int, [C.c_int, C.c_int64, C.c_int64, C.c_int64, C.POINTER(C.c_size_t)]
    ),
    "ab_gemm_tensorcore_eligible": (C.c_int, [C.c_int64, C.c_int64, C.c_int64]),
    "ab_gemm_max_clusters": (C.c_int, [C.c_int, C.c_int, C.POINTER(C.c_int)]),
    "ab_gemm_fused_layout": (C.c_int, [C.c_int64, C.c_int64, C.POINTER(C.c_int64), C.POINTER(C.c_int64)]),
    "ab_softmax": (
        C.c_int,
        [C.c_int, C.c_int, C.c_int64, C.c_int64, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p,
         C.c_void_p],
    ),
    "ab_max_and_argmax": (
        C.c_int,
        [C.c_int, C.c_int64, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p],
    ),
    "ab_random": (
        C.c_int,
        [C.c_int, C.c_int, C.c_uint64, C.c_int, c_i64p, C.c_int, c_voidpp, c_i64p, C.c_void_p, C.c_int,
         C.c_void_p],
    ),
    "ab_linalg_status_reset": (C.c_int, [C.c_void_p, C.c_void_p]),
    "ab_linalg_status_check": (C.c_int, [C.c_void_p, C.c_void_p]),
    "ab_linalg_update_count": (C.c_uint64, [C.c_int]),
    "ab_cholesky_workspace_bytes": (C.c_int, [C.c_int, C.c_int64, C.POINTER(C.c_size_t)]),
    "ab_cholesky": (
        C.c_int,
        [C.c_int, C.c_int64, C.c_void_p, C.c_int64, C.c_int64, C.c_int, C.c_int, C.c_int, C.c_void_p,
         C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p],
    ),
    "ab_trsm_workspace_bytes": (C.c_int, [C.c_int, C.c_int64, C.c_int64, C.POINTER(C.c_size_t)]),
    "ab_trsm": (
        C.c_int,
        [C.c_int, C.c_int64, C.c_int64, C.c_void_p, C.c_int64, C.c_int64, C.c_int, C.c_int, C.c_int,
         C.c_void_p, C.c_int64, C.c_int64, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_size_t,
         C.c_void_p],
    ),
    "ab_take_rows": (
        C.c_int,
        [C.c_int, C.c_int, C.c_void_p, C.c_int64, C.c_int64, C.c_int64, C.c_void_p, C.c_int64,
         C.c_int64, C.c_void_p, C.c_int, C.c_void_p],
    ),
    "ab_scatter_rows_workspace_bytes": (C.c_int, [C.c_int, C.c_int64, C.POINTER(C.c_size_t)]),
    "ab_scatter_rows": (
        C.c_int,
        [C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_int64, C.c_int64, C.c_int64, C.c_void_p,
         C.c_int64, C.c_int64, C.c_void_p, C.c_int64, C.c_int64, C.c_void_p, C.c_size_t, C.c_int,
         C.c_void_p],
    ),
    "ab_cell_scan_supported": (C.c_int, [C.c_int, C.c_int, C.c_int64, C.c_int64, C.c_int64]),
    "ab_cell_scan_workspace_bytes": (C.c_int, [C.c_int, C.c_int64, C.c_int64, C.POINTER(C.c_size_t)]),
    "ab_cell_scan": (
        C.c_int,
        [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int64, C.c_int64, C.c_int64, C.c_void_p, C.c_int64,
         C.c_int64, C.c_void_p, C.c_int64, C.c_int64, C.POINTER(C.c_void_p), C.POINTER(C.c_int64),
         C.POINTER(C.c_int64), C.c_void_p, C.c_size_t, C.c_void_p],
    ),
    "ab_lstm_scan_supported": (C.c_int, [C.c_int64, C.c_int64, C.c_int64]),
    "ab_lstm_scan_workspace_bytes": (C.c_int, [C.c_int64, C.c_int64, C.POINTER(C.c_size_t)]),
    "ab_lstm_scan": (
        C.c_int,
        [C.c_int64, C.c_int64, C.c_int64, C.c_void_p, C.c_int64, C.c_int64, C.c_void_p, C.c_int64,
         C.c_int64, C.c_void_p, C.c_int64, C.c_int64, C.c_void_p, C.c_int64, C.c_int64, C.c_void_p,
         C.c_size_t, C.c_void_p],
    ),
    "ab_launch_count": (C.c_uint64, []),
}


class GemmOperand(C.Structure):
    _fields_ = [
        ("plane0", C.c_void_p),
        ("plane1", C.c_void_p),
        ("rows", C.c_int64),
        ("k", C.c_int64),
        ("pitch", C.c_int64),
        ("mn_major", C.c_int32),
        ("precision", C.c_int32),
    ]


class GemmEpilogue(C.Structure):
    _fields_ = [
        ("module", C.c_void_p),
        ("n_operands", C.c_int32),
        ("ptr", C.c_void_p * 4),
        ("rs", C.c_int64 * 4),
        ("cs", C.c_int64 * 4),
        ("n_outputs", C.c_int32),
        ("out_f32", C.c_void_p * 3),
        ("out_rs", C.c_int64 * 3),
        ("shadow_bf16", C.c_void_p * 3),
        ("shadow_pitch", C.c_int64 * 3),
        ("colsum_ws", C.c_void_p),
        ("fullsum_ws", C.c_void_p),
        ("shadow_t_bf16", C.c_void_p),
        ("shadow_t_pitch", C.c_int64),
    ]


def load():
    """Return the loaded library (building it first if the tree has none)."""
    global _lib
    if _lib is not None:
        return _lib
    with _lock:
        if _lib is not None:
            return _lib
        path = _build.lib_path()
        if not os.path.exists(path):
            try:
                _build.build_library()
            except Exception as e:  # pragma: no cover
                raise RuntimeError(
                    f"libaesara_b200.so is missing and could not be built ({e}); the GPU "
                    "backend has no CPU fallback"
                ) from e
        # The library binds the first libnvrtc.so.12 in the process.  Importing torch first
        # makes that torch's bundled NVRTC in every process, build() included: the cubins
        # build() caches are then keyed (compile_cubin) on the NVRTC the tests and the bench
        # use, instead of the toolkit's one, which no later process would find.
        import torch  # noqa: F401

        lib = C.CDLL(path, mode=C.RTLD_GLOBAL)
        for name, (res, args) in SIGNATURES.items():
            try:
                fn = getattr(lib, name)
            except AttributeError:
                raise RuntimeError(f"{path} does not export {name}; rebuild with "
                                   "`python -m aesara_b200.build --force`") from None
            fn.restype = res
            fn.argtypes = args
        _lib = lib
    return _lib


def check(rc):
    if rc != 0:
        msg = load().ab_last_error().decode(errors="replace")
        raise AbError(rc, msg)


# ---------------------------------------------------------------------------
# JIT kernel cache: source hash -> cubin on disk -> loaded module handle
# ---------------------------------------------------------------------------
_cache_dir = {}


def cache_dir():
    env = os.environ.get("AESARA_B200_CACHE")
    if env not in _cache_dir:
        _cache_dir[env] = _find_cache_dir(env)
    return _cache_dir[env]


def _find_cache_dir(d):
    import threading

    if not d:
        d = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "_kcache")
    try:
        os.makedirs(d, exist_ok=True)
        probe = os.path.join(d, f".w{os.getpid()}_{threading.get_ident()}")
        with open(probe, "w"):
            pass
        os.remove(probe)
    except OSError:  # a read-only tree: the cubins go to a temporary directory
        import tempfile

        d = os.path.join(tempfile.gettempdir(), f"aesara_b200_kernels_{os.getuid()}")
        os.makedirs(d, exist_ok=True)
    return d


def nvrtc_version() -> tuple:
    """(major, minor) of the NVRTC that compiles the generated kernels: the libnvrtc.so.12
    loaded first in this process (torch's bundled one once torch is imported)."""
    major, minor = C.c_int32(), C.c_int32()
    check(load().ab_nvrtc_version(C.byref(major), C.byref(minor)))
    return major.value, minor.value


def compile_cubin(src: str, name: str = "ab_module") -> bytes:
    """NVRTC-compile ``src`` for sm_90a (disk-cached).  Needs no GPU.  The cache key holds the
    library version and the NVRTC version: two NVRTC versions make different code from one
    source."""
    lib = load()
    nvrtc = "nvrtc %d.%d\n" % nvrtc_version()
    key = hashlib.sha256((lib.ab_version().decode() + nvrtc + src).encode()).hexdigest()[:40]
    path = os.path.join(cache_dir(), f"{name}_{key}.cubin")
    if os.path.exists(path):
        try:
            os.utime(path)  # mark as used: prune_cache() drops what no build touched
        except OSError:
            pass
        with open(path, "rb") as f:
            return f.read()
    out = C.c_void_p()
    size = C.c_size_t()
    check(lib.ab_nvrtc_compile(src.encode(), (name + ".cu").encode(), None, 0,
                               C.byref(out), C.byref(size)))
    try:
        data = C.string_at(out, size.value)
    finally:
        lib.ab_buffer_free(out)
    import threading

    tmp = path + f".tmp{os.getpid()}_{threading.get_ident()}"
    with open(tmp, "wb") as f:
        f.write(data)
    os.replace(tmp, path)
    return data


def prune_cache(older_than: float) -> int:
    """Delete cached cubins that were neither compiled nor used since ``older_than`` (a
    time.time() value): every kernel revision leaves its cubins behind otherwise, and the
    cache travels with the tree to the GPU box."""
    n = 0
    d = cache_dir()
    for name in os.listdir(d):
        path = os.path.join(d, name)
        try:
            if name.endswith(".cubin") and os.path.getmtime(path) < older_than:
                os.remove(path)
                n += 1
        except OSError:
            pass
    return n


_modules = {}


def load_module(src: str, name: str = "ab_module"):
    """Compile (cached) and load a module on the current device; returns the
    opaque ``ab_module*`` as an int."""
    key = hashlib.sha256(src.encode()).hexdigest()
    h = _modules.get(key)
    if h is not None:
        return h[0]
    cubin = compile_cubin(src, name)
    lib = load()
    out = C.c_void_p()
    buf = C.create_string_buffer(cubin, len(cubin))
    check(lib.ab_module_load(buf, len(cubin), C.byref(out)))
    _modules[key] = (out.value, buf)  # keep the image alive with the module
    return out.value
