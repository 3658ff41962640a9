"""Host-side evaluation of *metadata* scalar expressions.

About half of a dynamically-shaped optimised graph is int64 shape arithmetic
(``Shape_i`` → ``ScalarFromTensor`` → scalar ``Composite`` → ``Assert`` →
``AllocEmpty``; SURVEY.md F5/a9).  Those values decide allocations and launch
geometry, so they must be known on the host before any kernel is launched;
they are a handful of integers, not tensor work.  This evaluator covers the
operator subset such graphs use; anything else on ≤1-element operands is sent
to the device kernel instead (never the other way round for real tensors).
"""

from __future__ import annotations

import numpy as np

MAX_HOST_ELEMS = 64


def _np(x):
    return np.asarray(x)


def _div_int(x, y):
    # in the operands' upcast type, as the device casts both (uint64 // bool stays uint64)
    t = np.result_type(x, y)
    x, y = x.astype(t), y.astype(t)
    y_safe = np.where(y == 0, t.type(1), y)
    return np.where(y == 0, t.type(0), np.floor_divide(x, y_safe))


def _mod_int(x, y):
    t = np.result_type(x, y)
    x, y = x.astype(t), y.astype(t)
    y_safe = np.where(y == 0, t.type(1), y)
    return np.where(y == 0, t.type(0), np.mod(x, y_safe))


def _c_type(dt):
    """C's integer promotion of an operand type: bool, 8- and 16-bit integers become int."""
    dt = np.dtype(dt)
    if dt.kind in "iub" and dt.itemsize < 4:
        return np.dtype(np.int32)
    return dt


def _c_common(a, b):
    """C's usual arithmetic conversions of two operand types (the device bodies write
    ``x < y``, ``x + y``, ``c ? x : y`` on the typed operands).  They differ from NumPy's
    promotion for mixed signedness (int32 with uint32 is uint32, int64 with uint64 is uint64)
    and for integers with float32 (float32, not float64)."""
    a, b = _c_type(a), _c_type(b)
    if a.kind == "f" or b.kind == "f":
        return np.dtype(np.float64) if np.dtype(np.float64) in (a, b) else np.dtype(np.float32)
    if a == b:
        return a
    if a.kind == b.kind:
        return a if a.itemsize > b.itemsize else b
    s, u = (a, b) if a.kind == "i" else (b, a)
    # an unsigned type at least as wide wins; otherwise int64 holds every uint32
    return u if u.itemsize >= s.itemsize else s


def _c_args(x, y):
    t = _c_common(x.dtype, y.dtype)
    return x.astype(t), y.astype(t)


def _c(fn):
    return lambda x, y: fn(*_c_args(_np(x), _np(y)))


def _true_div(x, y):
    if x.dtype.kind in "biu" and y.dtype.kind in "biu":
        return x.astype(np.float64) / y
    return _c(np.true_divide)(x, y)


def _switch(c, x, y):
    return np.where(c != 0, *_c_args(x, y))


def _clip(x, lo, hi):  # x < lo ? lo : (x > hi ? hi : x)
    inner = _switch(_c(np.greater)(x, hi), hi, x)
    return _switch(_c(np.less)(x, lo), lo, inner)


_OPS = {
    "add": lambda a, out: _fold(a, np.logical_or if out == np.bool_ else _c(np.add)),
    "mul": lambda a, out: _fold(a, np.logical_and if out == np.bool_ else _c(np.multiply)),
    "sub": lambda a, out: _c(np.subtract)(a[0], a[1]),
    "neg": lambda a, out: -a[0],
    "abs": lambda a, out: np.abs(a[0]),
    "sqr": lambda a, out: a[0] * a[0],
    "identity": lambda a, out: a[0],
    "second": lambda a, out: np.broadcast_to(a[1], np.broadcast_shapes(a[0].shape, a[1].shape)),
    "true_divide": lambda a, out: _true_div(a[0], a[1]),
    "int_div": lambda a, out: _div_int(a[0], a[1]) if out.kind in "biu" else np.floor(a[0] / a[1]),
    "mod": lambda a, out: _mod_int(a[0], a[1]) if out.kind in "biu" else np.mod(a[0], a[1]),
    "lt": lambda a, out: _c(np.less)(a[0], a[1]),
    "gt": lambda a, out: _c(np.greater)(a[0], a[1]),
    "le": lambda a, out: _c(np.less_equal)(a[0], a[1]),
    "ge": lambda a, out: _c(np.greater_equal)(a[0], a[1]),
    "eq": lambda a, out: _c(np.equal)(a[0], a[1]),
    "neq": lambda a, out: _c(np.not_equal)(a[0], a[1]),
    "switch": lambda a, out: _switch(*a),
    "maximum": lambda a, out: np.maximum(a[0], a[1]),
    "minimum": lambda a, out: np.minimum(a[0], a[1]),
    "and": lambda a, out: _c(np.bitwise_and)(a[0], a[1]),
    "or": lambda a, out: _c(np.bitwise_or)(a[0], a[1]),
    "xor": lambda a, out: _c(np.bitwise_xor)(a[0], a[1]),
    "invert": lambda a, out: np.logical_not(a[0]) if out == np.bool_ else np.invert(a[0]),
    "clip": lambda a, out: _clip(*a),
    "sgn": lambda a, out: np.sign(a[0]),
    "cast": lambda a, out: (a[0] != 0) if out == np.bool_ else a[0].astype(out),
    "ceil": lambda a, out: np.ceil(a[0].astype(out)),
    "floor": lambda a, out: np.floor(a[0].astype(out)),
    "reciprocal": lambda a, out: 1.0 / a[0].astype(out),
    "sqrt": lambda a, out: np.sqrt(a[0].astype(out)),
}


def _fold(args, fn):
    r = args[0]
    for x in args[1:]:
        r = fn(r, x)
    return r


def supports(expr):
    for st in expr["stmts"]:
        if st["op"] not in _OPS:
            return False
        # float IntDiv / Mod follow branchy C formulas in the reference (basic.py:2083-2121,
        # :2207-2236) that only the device bodies reproduce: never evaluate them here
        if st["op"] in ("int_div", "mod") and np.dtype(st["dtype"]).kind not in "biu":
            return False
    return True


def eval_expr(expr, inputs):
    """Evaluate an IR scalar expression on small host values."""
    temps = []
    inputs = [_np(x) for x in inputs]

    def ref(r):
        if isinstance(r, dict):
            return np.asarray(r["const"], dtype=r["dtype"])
        if r[0] == "i":
            return inputs[int(r[1:])]
        return temps[int(r[1:])]

    with np.errstate(all="ignore"):
        for st in expr["stmts"]:
            out = np.dtype(st["dtype"])
            val = _OPS[st["op"]]([ref(r) for r in st["args"]], out)
            temps.append(np.asarray(val).astype(out, copy=False))
    return [ref(r) for r in expr["outputs"]]
