"""Build ``libaesara_b200.so`` in-tree with nvcc for sm_90a (H100).

``python -m aesara_b200.build`` (or ``__graft_entry__.build()``).  nvcc
cross-compiles without a GPU; the resulting ``.so`` is git-ignored but travels
with the tree.
"""

from __future__ import annotations

import hashlib
import os
import shutil
import subprocess
import sys

PKG = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(PKG, "csrc")
LIBDIR = os.path.join(PKG, "lib")
LIBNAME = "libaesara_b200.so"
CUDA_HOME = os.environ.get("CUDA_HOME", "/usr/local/cuda")

ARCH_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a"]
COMMON = ["-O3", "-std=c++17", "-lineinfo", "-Xcompiler", "-fPIC", "-Xcompiler", "-Wall",
          "-Xcompiler", "-Wno-unused-function"]


def _sources():
    out = []
    for fn in sorted(os.listdir(CSRC)):
        if fn.endswith((".cpp", ".cu")):
            out.append(os.path.join(CSRC, fn))
    return out


def _stamp():
    h = hashlib.sha256()
    for fn in sorted(os.listdir(CSRC)):
        if fn.endswith((".cpp", ".cu", ".h", ".cuh")):
            with open(os.path.join(CSRC, fn), "rb") as f:
                h.update(fn.encode())
                h.update(f.read())
    with open(os.path.join(os.path.dirname(PKG), "include", "aesara_b200.h"), "rb") as f:
        h.update(f.read())
    h.update(" ".join(ARCH_FLAGS + COMMON).encode())
    return h.hexdigest()


def lib_path():
    return os.path.join(LIBDIR, LIBNAME)


def is_current():
    stamp = os.path.join(LIBDIR, "build.stamp")
    if not (os.path.exists(lib_path()) and os.path.exists(stamp)):
        return False
    with open(stamp) as f:
        return f.read().strip() == _stamp()


def build_library(force=False, verbose=True):
    """Compile every source under csrc/ into lib/libaesara_b200.so."""
    if not force and is_current():
        return lib_path()
    nvcc = shutil.which("nvcc") or os.path.join(CUDA_HOME, "bin", "nvcc")
    if not os.path.exists(nvcc):
        raise RuntimeError("nvcc not found; cannot build libaesara_b200.so")
    os.makedirs(LIBDIR, exist_ok=True)
    objdir = os.path.join(LIBDIR, "obj")
    os.makedirs(objdir, exist_ok=True)
    objs = []
    procs = []
    for src in _sources():
        obj = os.path.join(objdir, os.path.basename(src) + ".o")
        cmd = [nvcc, "-c", src, "-o", obj] + ARCH_FLAGS + COMMON
        if src.endswith(".cu"):
            cmd += ["-Xptxas", "-v"]
        else:
            cmd += ["-x", "cu"]
        procs.append((src, obj, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT)))
        objs.append(obj)
    log = []
    for src, obj, p in procs:
        out = p.communicate()[0].decode()
        log.append(f"== {os.path.basename(src)}\n{out}")
        if p.returncode != 0:
            raise RuntimeError(f"nvcc failed on {src}:\n{out}")
    link = [nvcc, "-shared", "-o", lib_path()] + objs + ARCH_FLAGS + [
        "-lnvrtc", "-ldl", "-lpthread",
        "-Xlinker", f"-rpath,{os.path.join(CUDA_HOME, 'lib64')}",
    ]
    r = subprocess.run(link, stdout=subprocess.PIPE, stderr=subprocess.STDOUT)
    if r.returncode != 0:
        raise RuntimeError("link failed:\n" + r.stdout.decode())
    with open(os.path.join(LIBDIR, "build.log"), "w") as f:
        f.write("\n".join(log))
    with open(os.path.join(LIBDIR, "build.stamp"), "w") as f:
        f.write(_stamp())
    if verbose:
        print(f"built {lib_path()}", file=sys.stderr)
    return lib_path()


if __name__ == "__main__":
    build_library(force="--force" in sys.argv)
