"""CPU: the wgmma main loop of the tensor-core GEMM keeps a k-block in flight.

Each MMA warpgroup commits one wgmma group per k-block and waits with ``wait_group 1``, so
that the tensor core works on k-block i while k-block i + 1 is issued; only the end of a K
segment drains the pipe (``wait_group 0``) before the segment is folded into the total.  Two
things have broken that without changing any result, and both are visible in the SASS:

* a branch around a k-block's wgmmas (an operand layout chosen at run time): ptxas closes a
  group at the end of each branch, and the commit after the join becomes an empty group
  (``HGMMA.64x8x16.F16 RZ``) that ``wait_group 1`` then lets through, instead of the k-block;
* a non-wgmma definition of accumulator registers inside the pipeline stage (ptxas C7515):
  every wgmma is serialised, with a ``WARPGROUP.DEPBAR.LE gsb0, 0x0`` after each HGMMA.

Checked on the ahead-of-time kernels of the built library (nvcc) and on the fused-epilogue
kernels of the cfg3 regions, compiled by NVRTC in this process -- which has imported torch, as
every user of the library has, and so uses the libnvrtc bundled with torch.  The fused
module has one entry point per MMA-loop layout; each keeps a stack frame of at most 128 bytes
(four loops in one kernel made that ptxas spill in the epilogue path).
"""
import os
import re
import shutil
import subprocess
import tempfile

import pytest

import torch  # noqa: F401  (first: its bundled NVRTC is the one production compiles with)

pytestmark = pytest.mark.skipif(shutil.which("cuobjdump") is None, reason="cuobjdump is not installed")

EMPTY_GROUP = "HGMMA.64x8x16.F16 RZ"
# the fused-epilogue module's entry points, one per MMA-loop layout (csrc/ab_gemm_tc_kernel.cuh)
EP_KERNELS = ["ab_gemm_ep_tf32", "ab_gemm_ep_tf32_1p", "ab_gemm_ep_f16", "ab_gemm_ep_f16_km",
              "ab_gemm_ep_f16_mk", "ab_gemm_ep_f16_mm"]


def sass_functions(sass):
    """function name -> the wgmma events of its SASS, in order: 'H' (an HGMMA that closes a
    group, i.e. carries gsb0), 'h' (any other HGMMA), 'E' (an empty group), 'W0' / 'W1'
    (WARPGROUP.DEPBAR.LE gsb0, 0x0 / 0x1)."""
    out, cur = {}, None
    for line in sass.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            cur = out.setdefault(m.group(1), [])
            continue
        if cur is None:
            continue
        if EMPTY_GROUP in line:
            cur.append("E")
        elif "HGMMA." in line:
            cur.append("H" if "gsb0" in line else "h")
        elif "WARPGROUP.DEPBAR.LE gsb0, 0x0" in line:
            cur.append("W0")
        elif "WARPGROUP.DEPBAR.LE gsb0, 0x1" in line:
            cur.append("W1")
    return out


def check_pipelined(name, ev):
    """The assertions of the module docstring on one kernel's event list."""
    assert "E" not in ev, f"{name}: empty wgmma group ({EMPTY_GROUP}): wait_group 1 waits for the real k-block"
    assert ev.count("H") + ev.count("h") >= 4, f"{name}: no wgmma main loop found"
    assert "W1" in ev, f"{name}: no wait_group 1: no k-block is kept in flight"
    for i, e in enumerate(ev):
        if e == "W0":
            # a segment drain: the k-block loop's last wait_group 1, then wait_group 0
            assert i > 0 and ev[i - 1] == "W1", \
                f"{name}: wait_group 0 right after an HGMMA (serialised wgmma, ptxas C7515): {ev}"
    assert ev.count("W0") <= ev.count("W1"), f"{name}: more full waits than pipelined ones: {ev}"


def cubin_sass(data: bytes) -> str:
    with tempfile.NamedTemporaryFile(suffix=".cubin") as tf:
        tf.write(data)
        tf.flush()
        return subprocess.run(["cuobjdump", "-sass", tf.name], capture_output=True, text=True, check=True).stdout


def test_ahead_of_time_gemm_kernels_keep_a_kblock_in_flight():
    from aesara_b200 import build
    from aesara_b200.runtime import lib

    lib.load()
    sass = subprocess.run(["cuobjdump", "-sass", build.lib_path()], capture_output=True, text=True, check=True).stdout
    kernels = {n: ev for n, ev in sass_functions(sass).items() if "gemm_tc_kernel" in n}
    assert len(kernels) == 4, sorted(kernels)  # {tf32, bf16} x {single CTA, cluster of 4}
    for name, ev in kernels.items():
        check_pipelined(name, ev)


@pytest.mark.parametrize("precision", [2, 0])
def test_fused_epilogue_gemm_kernels_keep_a_kblock_in_flight(precision, monkeypatch):
    from aesara_b200.runtime import lib
    from aesara_b200.runtime.vm import ProgramExecutor
    from tests._cases import load_case

    monkeypatch.setenv("AB_GEMM_FUSE_FP32", "1")  # the regions exist under precision 0 only with it
    prog, _, _ = load_case("cfg3_mlp")
    regions = ProgramExecutor(prog, precision=precision)._fusions
    assert len(regions) == 3
    nvrtc = "%d.%d" % lib.nvrtc_version()
    for f in regions:
        cubin = lib.compile_cubin(f.source(), "gemm_ep")
        kernels = {n: ev for n, ev in sass_functions(cubin_sass(cubin)).items() if n.startswith("ab_gemm_ep_")
                   and "marker" not in n}
        assert sorted(kernels) == sorted(EP_KERNELS)
        for name, ev in kernels.items():
            check_pipelined(f"{name} (region {f.g}, precision {precision}, NVRTC {nvrtc})", ev)
        # one MMA loop per entry point keeps the epilogue path free of spills
        with tempfile.NamedTemporaryFile(suffix=".cubin") as tf:
            tf.write(cubin)
            tf.flush()
            res = subprocess.run(["cuobjdump", "-res-usage", tf.name], capture_output=True, text=True).stdout
        for name, stack in re.findall(r"Function (ab_gemm_ep_\w+):\s*\n\s*REG:\d+ STACK:(\d+)", res):
            assert int(stack) <= 128, f"{name} (region {f.g}, precision {precision}): {stack}-byte stack frame"


def test_kernel_cache_is_keyed_on_the_nvrtc_version(tmp_path, monkeypatch):
    """A cubin compiled by one NVRTC is not served to a process that compiles with another."""
    from aesara_b200.runtime import lib

    major, minor = lib.nvrtc_version()
    assert major >= 12
    monkeypatch.setenv("AESARA_B200_CACHE", str(tmp_path))
    src = 'extern "C" __global__ void ab_probe_kernel(float* x) { x[threadIdx.x] *= 2.0f; }\n'
    lib.compile_cubin(src, "probe")
    lib.compile_cubin(src, "probe")
    assert len(os.listdir(tmp_path)) == 1
    monkeypatch.setattr(lib, "nvrtc_version", lambda: (major, minor + 1))
    lib.compile_cubin(src, "probe")
    assert len(os.listdir(tmp_path)) == 2
