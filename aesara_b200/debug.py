"""Dual-run checker: the B200 path against the reference's own thunks, node by node.

Reference pattern: ``DualLinker`` / ``WrapLinker`` (``aesara/link/c/basic.py:1934-2030``,
``link/basic.py:560-700``) run two linkers over the same ``FunctionGraph`` in lock step and
compare every intermediate value (``DebugMode`` builds on the same idea,
``compile/debugmode.py``).  Here the optimised graph produced for the B200 mode is linked a
second time with the reference's ``PerformLinker`` (Python ``perform``) or ``OpWiseCLinker``
(C thunks); the B200 executor records each node's outputs; the two traces are compared in
schedule order and the first disagreement is reported with the Apply node that produced it.

    from aesara_b200.debug import check_function
    report = check_function([x, y], [out], [xv, yv])      # raises DualRunMismatch on failure
"""

from __future__ import annotations

import copy

import numpy as np

from .compat.bootstrap import load_aesara

load_aesara()


class DualRunMismatch(AssertionError):
    def __init__(self, position, node, out_index, err, message):
        super().__init__(message)
        self.position = position
        self.node = node
        self.out_index = out_index
        self.err = err


def _as_host(v):
    if hasattr(v, "to_numpy") and not isinstance(v, np.ndarray):
        return v.to_numpy()
    return np.asarray(v)


def _compare(got, want, rtol, atol):
    got, want = _as_host(got), np.asarray(want)
    if got.shape != want.shape:
        return f"shape {got.shape} != reference {want.shape}", np.inf
    if got.dtype != want.dtype:
        return f"dtype {got.dtype} != reference {want.dtype}", np.inf
    if want.dtype.kind in "biu":
        bad = int(np.sum(got != want))
        return (f"{bad} integer/bool elements differ" if bad else None), float(bad)
    scale = float(np.max(np.abs(want))) if want.size else 0.0
    tol = atol + rtol * max(scale, 1e-30)
    with np.errstate(invalid="ignore"):
        diff = np.abs(got.astype(np.float64) - want.astype(np.float64))
    diff = np.where(np.isnan(got) & np.isnan(want), 0.0, diff)
    diff = np.where(np.isinf(want) & (got == want), 0.0, diff)
    err = float(np.nanmax(diff)) if diff.size else 0.0
    if not np.isfinite(err) or err > tol:
        return f"max |diff| {err:.3g} > {tol:.3g} (norm-wise rtol {rtol}, atol {atol})", err
    return None, err


def check_function(inputs, outputs, values, mode=None, reference_linker="py", rtol=1e-5, atol=1e-6,
                   updates=None, raise_on_mismatch=True):
    """Compile ``inputs -> outputs`` for the B200 mode, run it, and compare every node's
    outputs with the reference linker's thunks on the SAME optimised graph.

    Returns a list of ``(position, node, max_error)``; raises ``DualRunMismatch`` at the first
    node whose outputs disagree (unless ``raise_on_mismatch=False``: then the entry carries
    the message instead of the error)."""
    import aesara
    from aesara.link.basic import PerformLinker
    from aesara.link.c.basic import OpWiseCLinker

    from . import linker as L

    mode = mode or L.mode()
    f = aesara.function(inputs, outputs, mode=mode, updates=updates, on_unused_input="ignore")
    fgraph = f.maker.fgraph
    vm = f.vm
    order = vm.nodes

    # reference thunks over the same fgraph, nothing garbage-collected
    ref_linker = (PerformLinker(allow_gc=False) if reference_linker == "py"
                  else OpWiseCLinker(allow_gc=False)).accept(fgraph)
    ref_linker.schedule = lambda fg, _o=order: list(_o)
    ref_fn, ref_in, ref_out, ref_thunks, ref_order = ref_linker.make_all()
    assert list(ref_order) == list(order)
    # B200 trace: every node's outputs, copied to the host when the node has run
    for c, v in zip(vm.input_storage, values):
        c[0] = np.array(_as_host(v), copy=True) if not np.isscalar(v) else v
    # a Generator (random variables) is copied as it is before the B200 run advances it
    all_inputs = [copy.deepcopy(c[0]) if isinstance(c[0], np.random.Generator)
                  else np.array(_as_host(c[0]), copy=True) for c in vm.input_storage]
    for c, v in zip(ref_in, all_inputs):  # explicit inputs first, then shared variables
        c.storage[0] = v
    trace = {}
    ex = vm.executor
    prev = getattr(ex, "trace", None)
    ex.trace = trace
    try:
        vm()
    finally:
        ex.trace = prev

    program = getattr(vm.executor, "program", None)
    report = []
    for pos, (node, thunk) in enumerate(zip(order, ref_thunks)):
        if program is not None and program.nodes[pos].op == "RandomVariable" and pos in trace:
            # the device does not draw the reference's NumPy stream: its sample is checked
            # against the NumPy restatement of the device stream, then handed to the
            # reference's cells so that the nodes downstream are compared like for like
            msg, err = _check_random(program.nodes[pos], thunk, trace[pos])
            thunk()
            thunk.outputs[0][0] = copy.deepcopy(trace[pos][0])
            thunk.outputs[1][0] = trace[pos][1]
            if msg is not None:
                text = f"node {pos} {node} output 1: {msg}"
                if raise_on_mismatch:
                    raise DualRunMismatch(pos, node, 1, err, text)
                report.append((pos, node, text))
            else:
                report.append((pos, node, err))
            continue
        thunk()
        if pos not in trace:
            continue  # executed inside a fused region: compared at the region's outputs
        if type(node.op).__name__ == "AllocEmpty":
            continue  # uninitialised memory by definition (tensor/basic.py:3833)
        for k, (cell, got) in enumerate(zip(thunk.outputs, trace[pos])):
            if got is None:
                continue
            msg, err = _compare(got, cell[0], rtol, atol)
            if msg is not None:
                text = f"node {pos} {node} output {k}: {msg}"
                if raise_on_mismatch:
                    raise DualRunMismatch(pos, node, k, err, text)
                report.append((pos, node, text))
                break
        else:
            report.append((pos, node, 0.0 if not thunk.outputs else err))
    return report


# float32 / float64 Box-Muller draws against the long-double truth from the same words: the
# device's logf / sqrtf / sincospif and their float64 twins, plus the affine step
_NORMAL_TOL = {"float32": 4e-6, "float64": 1e-14}


def _check_random(pnode, thunk, traced):
    """(message or None, error) of a RandomVariable node's device sample: uniform and
    Bernoulli draws must equal the NumPy restatement of the stream (oracle/random_np.py) bit
    for bit, normal draws must lie within ``_NORMAL_TOL * (1 + |truth|)`` of it.  The key is
    the one the device drew: one full-range uint64 from the node's input Generator."""
    from oracle.random_np import random_sample, random_shape

    p = pnode.params
    rng, size, _dtype, *params = [c[0] for c in thunk.inputs]
    params = params[-1:] if p["dist"] == "bernoulli" else params
    key = int(copy.deepcopy(rng).integers(0, 2 ** 64, dtype=np.uint64))
    want = random_sample(p["dist"], p["dtype"], key, random_shape(size, params), params)
    got = np.asarray(traced[1])
    if got.shape != want.shape or got.dtype != np.dtype(p["dtype"]):
        return f"sample {got.dtype}{got.shape} != {p['dtype']}{want.shape}", np.inf
    state = traced[0].bit_generator.state
    g = copy.deepcopy(rng)
    g.integers(0, 2 ** 64, dtype=np.uint64)
    if state != g.bit_generator.state:
        return "the Generator did not advance by exactly one 64-bit draw", np.inf
    if p["dist"] == "normal":
        with np.errstate(invalid="ignore"):
            err = np.abs(got.astype(np.float64) - want) / (1 + np.abs(want))
        err = float(np.nanmax(err)) if err.size else 0.0
        if not err <= _NORMAL_TOL[p["dtype"]]:
            return f"normal draws off the stream by {err:.3g} (bound {_NORMAL_TOL[p['dtype']]:.0e})", err
        return None, err
    bad = int(np.sum(~((got == want) | (np.isnan(got) & np.isnan(want))) if got.dtype.kind == "f"
                     else got != want))
    return (f"{bad} draws differ from the stream" if bad else None), float(bad)
