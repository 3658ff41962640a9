"""Tensor-core GEMM throughput at the two cfg3 product shapes, kernel by kernel (run on a GPU).

    python tools/gemm_probe.py                 # every case, >= 1 s timed windows
    python tools/gemm_probe.py --window 2 --repeats 5 --json out.json

Times ``kernels.gemm`` (plain alpha/beta epilogue, operands packed once beforehand, so only the
GEMM kernel is in the window) with CUDA events over windows of at least ``--window`` seconds
after a warm-up, at the shapes of the cfg3 MLP (batch 65536, hidden 4096):

    fwd    65536 x 4096 x 4096   (X @ W: the forward products and dout @ W2.T)
    wgrad  4096 x 4096 x 65536   (X.T @ dpre: the weight gradients, K = batch)

with the operand layouts those products use: K-major (contiguous along K) and MN-major (the
transposed views; bf16 only, TF32 operands are always packed K-major), under the bf16 policy
(precision 2) and the fp32-faithful 3xTF32 policy (precision 0).  This separates the main
loop from the fused epilogue regions that bench.py measures with it.  Prints one JSON line per
case and a header line with the card, its power limit, the SM clock sampled during the timed
windows and the NVRTC version.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
os.environ["AB_GEMM_NO_TPACK"] = "1"  # an MN-major case stays MN-major (no transposing pack)

from aesara_b200.runtime import kernels as K, lib  # noqa: E402
from aesara_b200.runtime.device import DeviceArray  # noqa: E402
from bench import ClockSampler  # noqa: E402

B, H = 65536, 4096
# name, M, N, K, precision, A layout, B layout
CASES = [
    ("fwd", B, H, H, 2, "K", "K"),
    ("fwd", B, H, H, 2, "K", "MN"),
    ("wgrad", H, H, B, 2, "K", "K"),
    ("wgrad", H, H, B, 2, "MN", "MN"),
    ("fwd", B, H, H, 0, "K", "K"),
    ("wgrad", H, H, B, 0, "K", "K"),
]
POLICY = {0: "fp32", 2: "bf16"}


def operand_a(M, Kd, layout, gen):
    """[M, K] operand: K-major = a row-major matrix; MN-major = the transpose of a [K, M] one."""
    if layout == "K":
        return DeviceArray.from_torch(torch.randn(M, Kd, device="cuda", generator=gen))
    return DeviceArray.from_torch(torch.randn(Kd, M, device="cuda", generator=gen)).dimshuffle((1, 0))


def operand_b(Kd, N, layout, gen):
    """[K, N] operand: K-major = the transpose of an [N, K] matrix; MN-major = a row-major one."""
    if layout == "K":
        return DeviceArray.from_torch(torch.randn(N, Kd, device="cuda", generator=gen)).dimshuffle((1, 0))
    return DeviceArray.from_torch(torch.randn(Kd, N, device="cuda", generator=gen))


def time_calls(fn, n):
    start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(n):
        fn()
    stop.record()
    stop.synchronize()
    return start.elapsed_time(stop) / 1e3


def run_case(case, window, repeats, warmup):
    name, M, N, Kd, prec, la, lb = case
    gen = torch.Generator(device="cuda").manual_seed(0)
    A = operand_a(M, Kd, la, gen)
    Bm = operand_b(Kd, N, lb, gen)
    C = DeviceArray.empty((M, N), "float32")
    cache = K.PackCache()

    def call():
        K.gemm(C, 1.0, A, Bm, 0.0, precision=prec, cache=cache)

    call()  # packs the operands (kept in `cache`) and loads the kernel
    torch.cuda.synchronize()
    n, t = 1, time_calls(call, 1)
    while t < warmup:  # warm-up, and the call count of a window of >= `window` seconds
        n *= 2
        t = time_calls(call, n)
    n = max(1, int(np.ceil(n * window / t)))
    clocks = ClockSampler(torch.cuda.current_device())
    clocks.start()
    secs = [time_calls(call, n) for _ in range(repeats)]
    clk = clocks.stop()
    flop = 2.0 * M * N * Kd
    tflops = [flop * n / s / 1e12 for s in secs]
    return {
        "case": f"{name} {M}x{N}x{Kd}", "policy": POLICY[prec], "a": la, "b": lb,
        "calls_per_window": n, "window_s": round(float(np.median(secs)), 3),
        "ms_per_call": round(float(np.median(secs)) / n * 1e3, 4),
        "tflops": round(float(np.median(tflops)), 1),
        "tflops_min": round(min(tflops), 1), "tflops_max": round(max(tflops), 1),
        "sm_mhz": clk.get("sm_mhz"), "clock_reasons": clk.get("reasons"),
    }


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--window", type=float, default=1.0, help="seconds per timed window (>= 1)")
    ap.add_argument("--repeats", type=int, default=3, help="timed windows per case")
    ap.add_argument("--warmup", type=float, default=0.5, help="seconds of warm-up per case")
    ap.add_argument("--policy", choices=["all", "bf16", "fp32"], default="all")
    ap.add_argument("--json", help="also write the results to this file")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("gemm_probe needs a CUDA device")
    lib.check(lib.load().ab_init(0))
    torch.cuda.set_device(0)
    try:
        smi = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit,clocks.max.sm",
                              "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:
        smi = "unavailable"
    head = {"device": torch.cuda.get_device_name(0), "nvidia_smi": smi,
            "nvrtc": "%d.%d" % lib.nvrtc_version(), "library": lib.load().ab_version().decode(),
            "window_s": args.window, "repeats": args.repeats}
    print(json.dumps(head), flush=True)
    rows = []
    for case in CASES:
        if args.policy != "all" and POLICY[case[4]] != args.policy:
            continue
        r = run_case(case, max(args.window, 1.0), args.repeats, args.warmup)
        print(json.dumps(r), flush=True)
        rows.append(r)
        torch.cuda.empty_cache()
        time.sleep(0.5)
    if args.json:
        with open(args.json, "w") as f:
            json.dump({"header": head, "cases": rows}, f, indent=1)


if __name__ == "__main__":
    main()
