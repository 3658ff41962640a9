"""NVRTC-compile (no GPU needed) every kernel the committed fixtures use, so the
cubins in aesara_b200/_kcache/ travel with the tree."""
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from concurrent.futures import ThreadPoolExecutor

from aesara_b200.runtime.vm import ProgramExecutor
from aesara_b200.runtime import kernels as K
from aesara_b200.runtime import lib as _lib
from tests._cases import case_names, load_case


def main():
    t = time.time()
    had = os.environ.get("AB_GEMM_FUSE_FP32")
    os.environ["AB_GEMM_FUSE_FP32"] = "1"  # also the (opt-in) regions of the fp32-faithful kernels: tests launch them
    try:
        _compile_all(t)
    finally:
        if had is None:
            del os.environ["AB_GEMM_FUSE_FP32"]
        else:
            os.environ["AB_GEMM_FUSE_FP32"] = had


def _compile_all(t):
    exs = [ProgramExecutor(load_case(n)[0]) for n in case_names()]
    # GEMM-epilogue regions are generated per precision policy (float-pair vs float32-tree sums)
    for n in case_names():
        prog = load_case(n)[0]
        if any(nd.op in ("Dot22", "Gemm", "Dot22Scalar") for nd in prog.nodes):
            exs += [ProgramExecutor(prog, precision=pr) for pr in (1, 2)]
    # the reduction signatures the kernel-edge tests cover beyond the fixtures
    from tests.test_gpu_kernel_edges import REDUCE_SIGNATURES

    for sig in REDUCE_SIGNATURES:
        K.CAReduceKernel.get(*sig)
    # the fused-region graphs of tests/test_gpu_fused_regions.py (built with the reference front
    # end, where it is present): every GEMM-epilogue module per policy, every row-region J
    row_modules = []
    from aesara_b200.compat import bootstrap

    if bootstrap.available():
        from tests import _fused_regions as FR

        for name in FR.GEMM:
            exs += [ProgramExecutor(FR.gemm_program(name), precision=pr) for pr in (0, 1, 2)]
        for name in FR.ROW:
            for f in ProgramExecutor(FR.row_program(name))._fusions:
                classes = tuple("scal" if f.program.vars[v].ndim == 0 or f.program.vars[v].const is not None
                                else "row" for v in f.ext)
                by_ptr = tuple(f.program.vars[v].ndim == 0 and f.program.vars[v].const is None for v in f.ext)
                row_modules += [f._module(J, classes, by_ptr)["src"] for J in range(1, 9)]
    kerns = list(K.ElemwiseKernel._by_key.values()) + list(K.CAReduceKernel._by_key.values())
    for dt in ("float32", "float64", "int64", "int32", "int8", "bool"):
        kerns.append(K._identity_kernel(dt))
    fusions = [f for ex in exs for f in ex._fusions]  # row-region / GEMM-epilogue / map-reduce kernels
    with ThreadPoolExecutor(8) as pool:
        list(pool.map(lambda k: k.compile(), kerns))
        list(pool.map(lambda f: f.compile_all(), fusions))
        list(pool.map(lambda src: _lib.compile_cubin(src, "rowfuse"), row_modules))
    print(f"compiled {len(kerns)} modules + {len(fusions) + len(row_modules)} fused regions in {time.time() - t:.1f}s")


if __name__ == "__main__":
    main()
