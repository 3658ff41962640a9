"""Throughput of the Cholesky factorisation and the multi-RHS triangular solve (csrc/ab_linalg.cu).

    python tools/linalg_probe.py [--sizes 4096 8192 16384] [--reps 3]

For each n and dtype, times ``kernels.cholesky`` (n^3/3 useful flops) and ``kernels.trsm`` with
n right-hand sides (n^3 flops) by CUDA events, after one warm-up call, and prints TFLOP/s and
the share of the ceiling: a third of the H100 SXM data-sheet TF32 rate (495 TFLOP/s dense) for
float32, whose updates run as 3xTF32 products, and the data-sheet FP64 rate (67 TFLOP/s) for
float64.  The card's name, power limit and SM clock are read in the same run.  Writes nothing.
"""
import argparse
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

CEILING_TFLOPS = {"float32": 495.0 / 3, "float64": 67.0}


def smi(query):
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={query}", "--format=csv,noheader", "-i", "0"],
                             stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True, timeout=30).stdout
        return out.strip().splitlines()[0]
    except Exception:
        return "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", type=int, nargs="+", default=[4096, 8192, 16384])
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    import numpy as np
    import torch

    from aesara_b200.runtime import kernels as K
    from aesara_b200.runtime import lib
    from aesara_b200.runtime.device import DeviceArray

    lib.check(lib.load().ab_init(0))
    torch.cuda.set_device(0)
    print(f"card: {torch.cuda.get_device_name(0)}, power limit {smi('power.limit')}, "
          f"max SM clock {smi('clocks.max.sm')}")
    print(f"{'op':>8} {'dtype':>8} {'n':>6} {'ms':>9} {'TFLOP/s':>8} {'share':>6}  SM clock after")
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for dt in ("float32", "float64"):
        for n in args.sizes:
            g = torch.Generator(device="cuda").manual_seed(n)
            m = torch.randn(n, n, dtype=getattr(torch, dt), device="cuda", generator=g) / np.sqrt(n)
            spd = m @ m.T + torch.eye(n, dtype=m.dtype, device="cuda")
            a = DeviceArray(spd, spd.data_ptr(), dt, (n, n), (n, 1))
            rhs = torch.randn(n, n, dtype=m.dtype, device="cuda", generator=g)
            b = DeviceArray(rhs, rhs.data_ptr(), dt, (n, n), (n, 1))
            fac = None
            for op, flops in (("cholesky", n ** 3 / 3), ("trsm", float(n) ** 3)):
                def run():
                    st = K.LinalgStatus()
                    if op == "cholesky":
                        out = K.cholesky(a, True, st)
                    else:
                        out = K.trsm(fac, b, True, False, False, st)
                    st.check()
                    return out
                res = run()  # warm-up
                if op == "cholesky":
                    fac = res
                torch.cuda.synchronize()
                best = None
                for _ in range(args.reps):
                    ev0.record()
                    run()
                    ev1.record()
                    ev1.synchronize()
                    ms = ev0.elapsed_time(ev1)
                    best = ms if best is None else min(best, ms)
                tf = flops / (best * 1e-3) / 1e12
                print(f"{op:>8} {dt:>8} {n:>6} {best:9.2f} {tf:8.2f} {tf / CEILING_TFLOPS[dt]:6.1%}  "
                      f"{smi('clocks.sm')}", flush=True)
            del a, b, spd, rhs, m, fac
            torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
