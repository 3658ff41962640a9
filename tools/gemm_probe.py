"""Tensor-core GEMM throughput at the two cfg3 product shapes, arm by arm (run on a GPU).

    python tools/gemm_probe.py                 # every case and arm, >= 1 s timed windows
    python tools/gemm_probe.py --window 2 --repeats 5 --json out.json

Times ``kernels.gemm`` (operands packed once beforehand, so only the GEMM kernel is in the
window) with CUDA events over windows of at least ``--window`` seconds after a warm-up, at the
shapes of the cfg3 MLP (batch 65536, hidden 4096):

    fwd    65536 x 4096 x 4096   (X @ W: the forward products and dout @ W2.T)
    wgrad  4096 x 4096 x 65536   (X.T @ dpre: the weight gradients, K = batch)

with the operand layouts those products use: K-major (contiguous along K) and MN-major (the
transposed views; bf16 only, TF32 operands are always packed K-major), under the bf16 policy
(precision 2) and the fp32-faithful 3xTF32 policy (precision 0).

Each case is timed in several arms, which take turns window by window so that a drift of the
clock falls on all of them alike:

    single    the ahead-of-time kernel with the plain alpha/beta epilogue, one CTA per 128 x 128
              tile (AB_GEMM_CLUSTER=1);
    pair      the same kernel on CTA pairs stacked along M that share the B tile by TMA
              multicast (AB_GEMM_CLUSTER=2);
    nvrtc     the fused-epilogue entry point of that layout, built by NVRTC, with the identity
              region (value 0 = alpha * acc + beta * Cin), as gemm_run launches it;
    stages4   ``single`` with a 4-stage operand ring (AB_GEMM_STAGES=4, the fused kernels' ring);
    group8 / group1   ``single`` with tile groups of 8 rows / plain row order (AB_GEMM_GROUP_M;
              square tile grids only);
    pair_group2 / pair_group8   ``pair`` with groups of 2 / 8 pair rows (4 is its default).

Prints one JSON line per case and arm, and a header line with the card, its power limit, the
NVRTC version and how many clusters of 2 and of 4 CTAs of the bf16 kernel can be resident at
once (cudaOccupancyMaxActiveClusters); every line carries the SM clock sampled during its timed
windows.
"""
import argparse
import ctypes
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

from aesara_b200.codegen.gemm_epilogue import gemm_region_source  # noqa: E402
from aesara_b200.runtime import kernels as K, lib  # noqa: E402
from aesara_b200.runtime.device import DeviceArray  # noqa: E402
from aesara_b200.runtime.gemmfuse import EpilogueRequest  # noqa: E402
from bench import ClockSampler  # noqa: E402

B, H = 65536, 4096
# name, M, N, K, precision, A layout, B layout -- the layouts of the cfg3 products:
# X @ W1 (K/K), dW2 = h.T @ dout (both from transposed planes: K/K), dW1 = X.T @ dpre (X read
# MN-major: MN/K), dout @ W2.T with W2 read MN-major (K/MN: B not transposed-packed)
CASES = [
    ("wgrad", H, H, B, 2, "K", "K"),
    ("wgrad", H, H, B, 2, "MN", "K"),
    ("fwd", B, H, H, 2, "K", "K"),
    ("fwd", B, H, H, 2, "K", "MN"),
    ("fwd", B, H, H, 0, "K", "K"),
    ("wgrad", H, H, B, 0, "K", "K"),
]
POLICY = {0: "fp32", 2: "bf16"}
ARMS = {  # arm -> (environment, fused)
    "single": ({"AB_GEMM_CLUSTER": "1"}, False),
    "pair": ({"AB_GEMM_CLUSTER": "2"}, False),
    "nvrtc": ({}, True),
    "stages4": ({"AB_GEMM_CLUSTER": "1", "AB_GEMM_STAGES": "4"}, False),
    "group8": ({"AB_GEMM_CLUSTER": "1", "AB_GEMM_GROUP_M": "8"}, False),
    "group1": ({"AB_GEMM_CLUSTER": "1", "AB_GEMM_GROUP_M": "1"}, False),
    "pair_group2": ({"AB_GEMM_CLUSTER": "2", "AB_GEMM_GROUP_M": "2"}, False),
    "pair_group8": ({"AB_GEMM_CLUSTER": "2", "AB_GEMM_GROUP_M": "8"}, False),
}


class IdentityRegion:
    """A fused-epilogue module whose region yields its input: C = alpha * acc + beta * Cin."""

    def __init__(self, precision):
        merged = {"inputs": ["float32"], "out_dtypes": ["float32"], "outputs": ["i0"], "stmts": [],
                  "name": "identity"}
        self.src = gemm_region_source(merged, 0, cin=False, exact_sums=precision == 0)
        self._handle = None

    def handle(self):
        if self._handle is None:
            self._handle = lib.load_module(self.src, "gemm_ep")
        return self._handle


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


class Env:
    """Sets environment variables for the duration of a with-block."""

    def __init__(self, env):
        self.env, self.old = env, {}

    def __enter__(self):
        for k, v in self.env.items():
            self.old[k] = os.environ.get(k)
            os.environ[k] = v

    def __exit__(self, *exc):
        for k, v in self.old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


def run_case(case, arms, window, repeats, warmup):
    name, M, N, Kd, prec, la, lb = case
    gen = torch.Generator(device="cuda").manual_seed(0)
    A = operand_a(M, Kd, la, gen)
    Bm = operand_b(Kd, N, lb, gen)
    C = DeviceArray.empty((M, N), "float32")
    cache = K.PackCache()
    region = IdentityRegion(prec)
    calls, counts, secs, clks = {}, {}, {a: [] for a in arms}, {}

    def make_call(arm):
        env, fused = ARMS[arm]

        def call():
            with Env(env):
                ep = EpilogueRequest(region, [], [(True, False, False)], False, False) if fused else None
                K.gemm(C, 1.0, A, Bm, 0.0, precision=prec, cache=cache, epilogue=ep)
        return call

    for arm in arms:
        call = calls[arm] = make_call(arm)
        call()  # packs the operands (kept in `cache`) and loads the kernel
        torch.cuda.synchronize()
        n, t = 1, time_calls(call, 1)
        while t < warmup:  # warm-up, and the call count of a window of >= `window` seconds
            n *= 2
            t = time_calls(call, n)
        counts[arm] = max(1, int(np.ceil(n * window / t)))
    clk_rows = {a: [] for a in arms}
    for _ in range(repeats):
        for arm in arms:  # arm by arm, window by window
            clocks = ClockSampler(torch.cuda.current_device())
            clocks.start()
            secs[arm].append(time_calls(calls[arm], counts[arm]))
            clk_rows[arm].append(clocks.stop())
    flop = 2.0 * M * N * Kd
    out = []
    for arm in arms:
        n = counts[arm]
        tflops = [flop * n / s / 1e12 for s in secs[arm]]
        mhz = [c.get("sm_mhz") for c in clk_rows[arm] if c.get("sm_mhz")]
        reasons = sorted({r for c in clk_rows[arm] for r in c.get("reasons", [])})
        out.append({
            "case": f"{name} {M}x{N}x{Kd}", "policy": POLICY[prec], "a": la, "b": lb, "arm": arm,
            "calls_per_window": n, "window_s": round(float(np.median(secs[arm])), 3),
            "ms_per_call": round(float(np.median(secs[arm])) / n * 1e3, 4),
            "tflops": round(float(np.median(tflops)), 1),
            "tflops_min": round(min(tflops), 1), "tflops_max": round(max(tflops), 1),
            "sm_mhz": float(np.median(mhz)) if mhz else None, "clock_reasons": reasons,
        })
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--window", type=float, default=1.0, help="seconds per timed window (>= 1)")
    ap.add_argument("--repeats", type=int, default=3, help="timed windows per case and arm")
    ap.add_argument("--warmup", type=float, default=0.5, help="seconds of warm-up per case and arm")
    ap.add_argument("--policy", choices=["all", "bf16", "fp32"], default="all")
    ap.add_argument("--arms", default=",".join(ARMS), help="comma-separated subset of " + ", ".join(ARMS))
    ap.add_argument("--json", help="also write the results to this file")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("gemm_probe needs a CUDA device")
    want = [a for a in args.arms.split(",") if a]
    if any(a not in ARMS for a in want):
        sys.exit(f"unknown arm in {args.arms!r}; choose from {', '.join(ARMS)}")
    lib.check(lib.load().ab_init(0))
    torch.cuda.set_device(0)
    try:
        smi = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit,clocks.max.sm",
                              "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:
        smi = "unavailable"
    clusters = {}
    for ctas in (2, 4):
        n = ctypes.c_int(0)
        lib.check(lib.load().ab_gemm_max_clusters(2, ctas, ctypes.byref(n)))
        clusters[f"max_clusters_{ctas}"] = n.value
    head = {"device": torch.cuda.get_device_name(0), "nvidia_smi": smi, **clusters,
            "sms": torch.cuda.get_device_properties(0).multi_processor_count,
            "nvrtc": "%d.%d" % lib.nvrtc_version(), "library": lib.load().ab_version().decode(),
            "window_s": args.window, "repeats": args.repeats}
    print(json.dumps(head), flush=True)
    rows = []
    for case in CASES:
        if args.policy != "all" and POLICY[case[4]] != args.policy:
            continue
        tm, tn = -(-case[1] // 128), -(-case[2] // 128)
        arms = [a for a in want if not ("group" in a and tm >= 4 * tn)]  # square grids only
        for r in run_case(case, arms, max(args.window, 1.0), args.repeats, args.warmup):
            print(json.dumps(r), flush=True)
            rows.append(r)
        torch.cuda.empty_cache()
        time.sleep(0.5)
    if args.json:
        with open(args.json, "w") as f:
            json.dump({"header": head, "cases": rows}, f, indent=1)


if __name__ == "__main__":
    main()
