"""Throughput of the random-variable kernels (csrc/ab_random.cu) at 2^28 elements.

    python tools/rng_probe.py [--log2n 28] [--reps 20]

Times uniform f32/f64, normal f32/f64 and Bernoulli (int64) draws with scalar parameters by
CUDA events around ``ab_random`` and prints, per case, the milliseconds, the bytes written
over that time, and that rate as a fraction of the H100 SXM data-sheet HBM3 bandwidth
(3.35 TB/s), with the card's name and power limit.  Writes nothing.
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

DATASHEET_TBPS = 3.35


def power_limit():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                             stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True, timeout=30).stdout
        return out.strip().splitlines()[0]
    except Exception:
        return "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--log2n", type=int, default=28)
    ap.add_argument("--reps", type=int, default=20)
    args = ap.parse_args()
    import numpy as np
    import torch

    from aesara_b200.ir import DTYPE_CODE
    from aesara_b200.runtime import lib
    from aesara_b200.runtime.device import stream_handle

    L = lib.load()
    lib.check(L.ab_init(0))
    torch.cuda.set_device(0)
    n = 1 << args.log2n
    card = torch.cuda.get_device_name(0)
    plim = power_limit()
    cases = [("uniform", 0, "float32"), ("uniform", 0, "float64"), ("normal", 1, "float32"),
             ("normal", 1, "float64"), ("bernoulli", 2, "int64")]
    for name, dist, dt in cases:
        item = np.dtype(dt).itemsize
        out = torch.empty(n * item, dtype=torch.uint8, device="cuda")
        pdt = "float64" if dist == 2 else dt
        vals = [0.5] if dist == 2 else [0.0, 1.0]
        par = [torch.tensor([v], dtype=getattr(torch, pdt), device="cuda") for v in vals]
        ptrs = (C.c_void_p * len(par))(*[p.data_ptr() for p in par])
        strides = (C.c_int64 * len(par))(*([0] * len(par)))
        shape = (C.c_int64 * 1)(n)

        def run(key):
            lib.check(L.ab_random(dist, DTYPE_CODE[dt], key, 1, shape, len(par), ptrs, strides, out.data_ptr(),
                                  0, stream_handle()))

        for k in range(3):
            run(k)
        torch.cuda.synchronize()
        times = []
        for k in range(args.reps):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            run(1000 + k)
            e1.record()
            e1.synchronize()
            times.append(e0.elapsed_time(e1))
        ms = float(np.median(times))
        tbps = n * item / (ms * 1e-3) / 1e12
        print(json.dumps({"case": f"{name}_{dt}", "elements": n, "median_ms": round(ms, 4),
                          "min_ms": round(min(times), 4), "written_TBps": round(tbps, 3),
                          "of_datasheet": round(tbps / DATASHEET_TBPS, 3), "card": card,
                          "power_limit": plim}))
        del out


if __name__ == "__main__":
    main()
