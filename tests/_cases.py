"""Shared helpers: load golden fixtures, compare with the tolerances stated here.

Tolerance policy (BASELINE north star; the reference's own test tolerances are
aesara/tensor/math.py:85-96: f32 rtol=atol=1e-5, f64 rtol=1e-5/atol=1e-8):
  * integer / bool outputs: bit-exact;
  * float outputs of element-wise / reduction graphs: rtol 1e-5 (+ atol 1e-6 f32, 1e-10 f64);
  * float outputs downstream of a dot product: rtol 1e-5 relative to the
    largest magnitude of the output (norm-wise), because the summation order
    differs between BLAS, NumPy and the device kernels.
"""
import glob
import os

import numpy as np

from aesara_b200.ir import Program

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
BLAS_OPS = {"Dot22", "Dot22Scalar", "Gemm", "Gemv", "Ger", "Dot", "Scan"}


def case_names():
    return sorted(os.path.basename(p)[:-5] for p in glob.glob(os.path.join(GOLDEN, "*.json")))


def load_case(name):
    prog = Program.load(os.path.join(GOLDEN, name + ".json"))
    z = np.load(os.path.join(GOLDEN, name + ".npz"))
    ins = [z[f"in_{k}"] for k in range(len(prog.inputs))]
    outs = [z[f"out_{k}"] for k in range(len(prog.outputs))]
    return prog, ins, outs


def uses_blas(prog):
    return any(n.op in BLAS_OPS for n in prog.nodes)


def assert_matches(got, want, blas=False, rtol=1e-5, what=""):
    got = np.asarray(got)
    want = np.asarray(want)
    assert got.shape == want.shape, f"{what}: shape {got.shape} != {want.shape}"
    assert got.dtype == want.dtype, f"{what}: dtype {got.dtype} != {want.dtype}"
    if want.dtype.kind in "biu":
        np.testing.assert_array_equal(got, want, err_msg=what)
        return
    if blas:
        scale = float(np.max(np.abs(want))) if want.size else 1.0
        atol = rtol * max(scale, 1e-30)
        np.testing.assert_allclose(got, want, rtol=rtol, atol=atol, err_msg=what)
    else:
        atol = 1e-6 if want.dtype == np.float32 else 1e-10
        np.testing.assert_allclose(got, want, rtol=rtol, atol=atol, equal_nan=True, err_msg=what)


def fused_vs_plain(fused, plain, what, exact_sums=True):
    """cfg3 outputs [loss, dW1, db1, dW2, db2]: the products see identical operands (the
    epilogue evaluates the same scalar expressions on the same fp32 values; a bf16 plane written
    by the epilogue equals the separate pack), so the weight gradients are BIT-identical.  Loss
    and bias gradients, fp32-faithful policy: float64(-equivalent) sums of identical float32
    terms in a different (still deterministic) order: equal to the last float32 bit or one ulp.
    tf32 / bf16 policies (``exact_sums=False``): the epilogue adds 8 / 32 terms at a time as a
    float32 tree before the float64 stage -- a few 2^-24 of the sum of magnitudes, checked
    norm-wise at 2e-6 (the terms themselves carry 2^-8 from the bf16 operands)."""
    for k, (a, b) in enumerate(zip(fused, plain)):
        if np.ndim(a) == 2:
            np.testing.assert_array_equal(a, b, err_msg=f"{what} output {k}: fused vs node-by-node")
        elif exact_sums:
            np.testing.assert_allclose(a, b, rtol=3e-7, atol=0, err_msg=f"{what} output {k}: fused vs node-by-node")
        else:
            np.testing.assert_allclose(a, b, rtol=0, atol=2e-6 * float(np.max(np.abs(b))),
                                       err_msg=f"{what} output {k}: fused vs node-by-node")


def mlp_inputs(rng, B, H):
    """cfg3 inputs [X, Y, W1, b1, W2, b2] (float32) at batch B and hidden size H."""
    return [rng.standard_normal((B, H)).astype("float32"), rng.standard_normal((B, H)).astype("float32"),
            (rng.standard_normal((H, H)) / np.sqrt(H)).astype("float32"), (rng.standard_normal(H) * 0.1).astype("float32"),
            (rng.standard_normal((H, H)) / np.sqrt(H)).astype("float32"), (rng.standard_normal(H) * 0.1).astype("float32")]


def mlp_truth(ins):
    """cfg3 outputs [loss, dW1, db1, dW2, db2] in float64 (NumPy) for the given inputs."""
    X, Y, W1, b1, W2, b2 = [np.asarray(a, np.float64) for a in ins]
    h = np.tanh(X @ W1 + b1)
    diff = h @ W2 + b2 - Y
    dout = 2.0 * diff / diff.size
    dpre = (dout @ W2.T) * (1.0 - h * h)
    return [np.mean(diff ** 2), X.T @ dpre, dpre.sum(0), h.T @ dout, dout.sum(0)]
