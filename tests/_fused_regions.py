"""Graphs of the executor-level fused regions, built with the reference front end, and their
NumPy truths.

GEMM-epilogue regions (runtime/gemmfuse.py): a ``Dot22`` / ``Dot22Scalar`` / ``Gemm`` node and
the ``Elemwise`` / ``Sum`` nodes that consume it.  Row regions (runtime/rowfuse.py):
``Gemv(X, w)`` -> per-row ``Elemwise`` -> ``Sum`` / ``Gemv(X.T, r)``.

Every graph is written once, as ``fn(o, v) -> outputs`` over an ops namespace ``o`` and a dict
``v`` of its inputs, and evaluated twice: symbolically (``aesara.tensor``) and on float64 NumPy
arrays (the truth).  The exact graphs use only add / sub / mul of small integers, maximum,
minimum, clip, abs, switch and scaling by powers of two.  With integer operands in [-4, 4], the
right operands of products in {-1, 0, 1} with a few non-zeros per column (the GPU suite's inputs)
and K <= 2048, every value read as a bf16 plane is a small integer, so every value, every plane
of it and every product of such a plane is exact, and float64 is the truth bit for bit.

``GEMM[name].expect`` is what region detection must find: the ``#define``s of the generated
module (``AB_EP_*``), the member node ops and, where the region must shrink, the members left out.
"""
import functools
from collections import namedtuple

import numpy as np

F32 = np.float32

# inputs: name -> (kind, shape in the symbols M, N, K, P, D, NR)
#   kinds: "mat" fmatrix, "vec" fvector, "col" fcol, "scal" fscalar, "ivec" ivector, "bvec" bool
GCase = namedtuple("GCase", "name inputs fn expect exact")
RCase = namedtuple("RCase", "name inputs fn expect")


class _SymOps:
    def __init__(self, at):
        self.at = at
        for f in ("maximum", "minimum", "tanh", "exp", "sigmoid", "softplus", "switch", "abs", "sqr",
                  "lt", "gt", "ge", "dot"):
            setattr(self, f, getattr(at, f))

    def clip(self, v, lo=-64, hi=64):
        return self.at.clip(v, F32(lo), F32(hi))

    def sum(self, v, axis=None):
        return self.at.sum(v, axis=axis)

    def cast32(self, v):
        return self.at.cast(v, "float32")

    def rowsum(self, v):
        return self.at.sum(v, axis=1, keepdims=True)


class _NpOps:
    maximum, minimum, tanh, exp = (staticmethod(f) for f in (np.maximum, np.minimum, np.tanh, np.exp))
    abs, lt, gt, ge, switch = (staticmethod(f) for f in (np.abs, np.less, np.greater, np.greater_equal, np.where))

    @staticmethod
    def sqr(v):
        return v * v

    @staticmethod
    def dot(a, b):
        return np.asarray(a, np.float64) @ np.asarray(b, np.float64)

    @staticmethod
    def clip(v, lo=-64, hi=64):
        return np.clip(v, lo, hi)

    @staticmethod
    def sum(v, axis=None):
        return np.sum(v, axis=axis)

    @staticmethod
    def cast32(v):
        return np.asarray(v, np.float64)

    @staticmethod
    def rowsum(v):
        return np.sum(v, axis=1, keepdims=True)

    @staticmethod
    def sigmoid(v):
        with np.errstate(over="ignore"):
            return 1.0 / (1.0 + np.exp(-v))

    @staticmethod
    def softplus(v):
        return np.logaddexp(0.0, v)


def _xw(o, v):
    return o.dot(v["X"], v["W"])


XW = {"X": ("mat", "MK"), "W": ("mat", "KN")}
DEF = {"AB_EP_NOPS": 0, "AB_EP_NOUT": 1, "AB_EP_COLSUM": -1, "AB_EP_FULLSUM": -1, "AB_EP_CIN": 0,
       "AB_EP_PRE_OP": -1, "AB_EP_TPLANE": -1, "AB_EP_ROWMASK": 0}


def _g(name, extra, fn, exact=True, ops="Dot22 Elemwise", left_out=0, **defs):
    """``defs``: the ``#define``s that differ from ``DEF``; ``ops``: the member ops in schedule
    order (``left_out``: member candidates a legal region must leave to run node by node)."""
    d = dict(DEF)
    d.update({("AB_EP_" + k.upper()): v for k, v in defs.items()})
    return GCase(name, dict(XW, **extra), fn, {"defines": d, "ops": ops.split(), "left_out": left_out}, exact)


MAT = ("mat", "MN")
VEC = ("vec", "N")
SCAL = ("scal", "")


def _acc2(o, v):
    return o.dot(v["X2"], v["W2"])


GEMM = {c.name: c for c in [
    # ---- operands: 0..4 of them, every kind and run-time path
    _g("ops0", {}, lambda o, v: [o.abs(_xw(o, v))]),
    _g("scalar", {"s": SCAL}, lambda o, v: [o.maximum(_xw(o, v), v["s"])], nops=1),
    _g("bias_static", {"b": VEC}, lambda o, v: [_xw(o, v) + v["b"]], nops=1, rowmask=1),
    # a [1, N] row only known at run time: read by shuffle when it is not the read-ahead operand
    _g("row_runtime", {"Y": MAT, "r": ("mat", "1N")},
       lambda o, v: [o.maximum(_xw(o, v), v["Y"]) * v["r"]], nops=2, pre_op=0),
    _g("row_runtime_pre", {"r": ("mat", "1N")}, lambda o, v: [_xw(o, v) * v["r"]], nops=1, pre_op=0),
    _g("col", {"c": ("col", "M1")}, lambda o, v: [_xw(o, v) * v["c"]], nops=1, pre_op=0),
    _g("mn_op0", {"Y": MAT}, lambda o, v: [o.maximum(_xw(o, v), v["Y"])], nops=1, pre_op=0),
    _g("mn_op1", {"b": VEC, "Y": MAT}, lambda o, v: [(_xw(o, v) + v["b"]) * v["Y"]], nops=2, pre_op=1, rowmask=1),
    _g("mn_ld8", {"Y": MAT, "Z": MAT}, lambda o, v: [o.maximum(_xw(o, v), v["Y"]) * v["Z"]], nops=2, pre_op=0),
    _g("mn_strided", {"Yt": ("mat", "NM")}, lambda o, v: [o.maximum(_xw(o, v), v["Yt"].T)], nops=1, pre_op=0),
    _g("mn_reversed", {"Y": MAT, "Z": MAT},
       lambda o, v: [o.maximum(_xw(o, v), v["Y"]) * v["Z"][::-1]], nops=2, pre_op=0),
    _g("mn_reversed_pre", {"Y": MAT}, lambda o, v: [o.maximum(_xw(o, v), v["Y"][::-1])], nops=1, pre_op=0),
    _g("ops4", {"s": SCAL, "b": VEC, "Y": MAT, "Z": MAT},
       lambda o, v: [o.minimum(o.maximum(_xw(o, v), v["s"]) + v["b"], v["Y"]) * v["Z"]],
       nops=4, pre_op=2, rowmask=2),
    # ---- more than a region takes: it shrinks to its largest legal prefix
    _g("shrink_ops5", {"s": SCAL, "b": VEC, "Y": MAT, "Z": MAT, "c": ("col", "M1")},
       lambda o, v: (lambda h: [h, (h * v["Y"] - v["Z"]) * v["c"]])(o.maximum(_xw(o, v), v["s"]) + v["b"]),
       nops=2, rowmask=2, left_out=1),
    _g("shrink_nout4", {"b": VEC, "Y": MAT},
       lambda o, v: (lambda h1: (lambda h2: (lambda h3: [h1, h2, h3, o.abs(h3) - h1])(h2 * h2))(h1 * v["Y"]))(
           _xw(o, v) + v["b"]),
       nops=2, rowmask=1, pre_op=1, nout=3, ops="Dot22 Elemwise Elemwise Elemwise", left_out=1),
    # a second column sum: the region keeps the first one
    _g("shrink_colsum2", {"b": VEC, "Y": MAT},
       lambda o, v: (lambda h1: [h1, o.sum(h1, axis=0), o.sum(h1 * v["Y"], axis=0)])(_xw(o, v) + v["b"]),
       nops=2, rowmask=1, pre_op=1, nout=2, colsum=0, ops="Dot22 Elemwise CAReduce Elemwise", left_out=1),
    # ---- values and reductions
    _g("nout2", {"b": VEC, "Y": MAT},
       lambda o, v: (lambda h: [h, h * v["Y"]])(_xw(o, v) + v["b"]),
       nops=2, rowmask=1, pre_op=1, nout=2, ops="Dot22 Elemwise Elemwise"),
    _g("nout3", {"b": VEC, "Y": MAT, "Z": MAT},
       lambda o, v: (lambda h: (lambda h2: [h, h2, o.maximum(h2, v["Z"])])(h * v["Y"]))(_xw(o, v) + v["b"]),
       nops=3, rowmask=1, pre_op=1, nout=3, ops="Dot22 Elemwise Elemwise Elemwise"),
    _g("colsum_v0", {"b": VEC}, lambda o, v: [o.sum(_xw(o, v) + v["b"], axis=0)],
       nops=1, rowmask=1, colsum=0, ops="Dot22 Elemwise CAReduce"),
    _g("colsum_v1", {"b": VEC, "Y": MAT},
       lambda o, v: (lambda h: [h, o.sum(h * v["Y"], axis=0)])(_xw(o, v) + v["b"]),
       nops=2, rowmask=1, pre_op=1, nout=2, colsum=1, ops="Dot22 Elemwise Elemwise CAReduce"),
    _g("colsum_v2", {"b": VEC, "Y": MAT},
       lambda o, v: (lambda h: (lambda h2: [h, h2, o.sum(o.abs(h2) - h, axis=0)])(h * v["Y"]))(_xw(o, v) + v["b"]),
       nops=2, rowmask=1, pre_op=1, nout=3, colsum=2, ops="Dot22 Elemwise Elemwise Elemwise CAReduce"),
    _g("total_only", {}, lambda o, v: [o.sum(o.abs(_xw(o, v)))], fullsum=0, ops="Dot22 Elemwise CAReduce"),
    _g("col_full_same", {"Y": MAT, "Z": MAT},
       lambda o, v: (lambda h: [h, o.sum(h, axis=0), o.sum(h)])(o.maximum(_xw(o, v), v["Y"]) * v["Z"]),
       nops=2, pre_op=0, colsum=0, fullsum=0, ops="Dot22 Elemwise CAReduce CAReduce"),
    _g("col_full_diff", {"b": VEC, "Y": MAT},
       lambda o, v: (lambda h: [h, o.sum(h, axis=0), o.sum(h * v["Y"])])(_xw(o, v) + v["b"]),
       nops=2, rowmask=1, pre_op=1, nout=2, colsum=0, fullsum=1, ops="Dot22 Elemwise CAReduce Elemwise CAReduce"),
    # ---- plans: values read by downstream products (bf16 planes under the bf16 policy)
    _g("plane_nat", {"b": VEC, "W2": ("mat", "NP")},
       lambda o, v: [o.dot(o.abs(_xw(o, v) + v["b"]), v["W2"])], nops=1, rowmask=1),
    _g("plane_nat_stored", {"b": VEC, "W2": ("mat", "NP")},
       lambda o, v: (lambda h: [h, o.dot(h, v["W2"])])(o.abs(_xw(o, v) + v["b"])), nops=1, rowmask=1),
    # (Gt @ h contracts over the rows of h; Gt exists before the region runs, so h needs no
    # float32 copy)
    _g("plane_t_colsum", {"b": VEC, "Gt": ("mat", "PM")},
       lambda o, v: (lambda h: [o.sum(h, axis=0), o.dot(v["Gt"], h)])(_xw(o, v) + v["b"]),
       nops=1, rowmask=1, tplane=0, colsum=0, ops="Dot22 Elemwise CAReduce"),
    # a transposed plane without column sums (its natural plane too)
    _g("plane_both", {"b": VEC, "W2": ("mat", "NP"), "Gt": ("mat", "PM")},
       lambda o, v: (lambda h: [o.dot(h, v["W2"]), o.dot(v["Gt"], h)])(_xw(o, v) + v["b"]),
       nops=1, rowmask=1, tplane=0),
    # ---- products
    _g("dot22scalar", {"Y": MAT}, lambda o, v: [o.maximum(_xw(o, v) * F32(0.5), v["Y"])],
       nops=1, pre_op=0, ops="Dot22Scalar Elemwise"),
    _g("gemm_beta", {"Y": MAT, "Z": MAT}, lambda o, v: [o.maximum(v["Y"] * F32(0.25) + _xw(o, v), v["Z"])],
       nops=1, pre_op=0, cin=1, ops="Gemm Elemwise"),
    # Dot22 -> Gemm{inplace}(h, ...) -> Elemwise{inplace}: t reuses h's memory, and h's packs
    # (made for h @ W4) must not serve t @ W3
    GCase("gemm_inplace", {"X": ("mat", "MK"), "W": ("mat", "KN"), "X2": ("mat", "MK"), "W2": ("mat", "KN"),
                           "W3": ("mat", "NP"), "W4": ("mat", "NP")},
          lambda o, v: (lambda h: [o.dot(o.abs(h + _acc2(o, v)), v["W3"]), o.dot(h, v["W4"])])(_xw(o, v)),
          {"defines": dict(DEF, AB_EP_CIN=1), "ops": ["Gemm", "Elemwise"], "left_out": 0}, True),
    # ---- operand layouts of the product (with sums)
    GCase("layout_xt", {"Xt": ("mat", "KM"), "W": ("mat", "KN"), "b": VEC},
          lambda o, v: (lambda h: [h, o.sum(h, axis=0), o.sum(h)])(o.dot(v["Xt"].T, v["W"]) + v["b"]),
          {"defines": dict(DEF, AB_EP_NOPS=1, AB_EP_ROWMASK=1, AB_EP_COLSUM=0, AB_EP_FULLSUM=0),
           "ops": ["Dot22", "Elemwise", "CAReduce", "CAReduce"], "left_out": 0}, True),
    # ---- misaligned operands (the fused launch is refused at run time)
    _g("mn_misaligned", {"Yw": ("mat", "MN+")}, lambda o, v: [o.maximum(_xw(o, v), v["Yw"][:, 1:])], nops=1, pre_op=0),
    _g("gemm_z_misaligned", {"Yw": ("mat", "MN+"), "Z": MAT},
       lambda o, v: [o.maximum(v["Yw"][:, 1:] * F32(0.5) + _xw(o, v), v["Z"])], nops=1, pre_op=0, cin=1,
       ops="Gemm Elemwise"),
    # ---- an operand computed by another node (a [1, 1] factor from a shape)
    _g("late_operand", {"Y": MAT},
       lambda o, v: [o.maximum(_xw(o, v), v["Y"]) * o.cast32(v["Y"].shape[0])], nops=2, pre_op=0),
    # ---- transcendental programs: bit-identical to the node-by-node kernels, ulps vs float64
    GCase("transc", {"X": ("mat", "MK"), "W": ("mat", "KN"), "b": VEC},
          lambda o, v: (lambda h: [o.tanh(h), o.sigmoid(h) * o.exp(h * F32(-0.125)), o.softplus(h)])(
              _xw(o, v) * F32(0.0625) + v["b"]),
          {"defines": None, "ops": None, "left_out": 0}, False),
]}


def _rz(o, v):
    return o.clip(o.dot(v["X"], v["w"]), -8, 8)


XWV = {"X": ("mat", "ND"), "w": ("vec", "D")}


def _r(name, extra, fn, sums):
    return RCase(name, dict(XWV, **extra), fn, {"sums": sums})


# Row regions: z = clip(X @ w, -8, 8) per row, a per-row step r, then X.T @ r and 0..2 sums of
# per-row values.  X in [-4, 4], w in [-2, 2]: every per-row value is an integer, |X.T @ r| and
# the sums stay far below 2**24.
ROW = {c.name: c for c in [
    _r("sums0", {"y": ("vec", "N")}, lambda o, v: [o.dot(v["X"].T, _rz(o, v) * v["y"])], 0),
    _r("sums1", {"y": ("vec", "N")},
       lambda o, v: (lambda r: [o.dot(v["X"].T, r), o.sum(r)])(_rz(o, v) * v["y"]), 1),
    _r("sums2", {"y": ("vec", "N")},
       lambda o, v: (lambda r: [o.dot(v["X"].T, r), o.sum(r), o.sum(r * v["y"])])(_rz(o, v) * v["y"]), 2),
    # a per-row vector as a strided view, an int32 and a bool per-row vector
    _r("strided", {"yy": ("vec", "2N")},
       lambda o, v: (lambda r: [o.dot(v["X"].T, r), o.sum(r)])(_rz(o, v) * v["yy"][::2]), 1),
    _r("int32", {"i": ("ivec", "N")},
       lambda o, v: (lambda r: [o.dot(v["X"].T, r), o.sum(r)])(_rz(o, v) * o.cast32(v["i"])), 1),
    _r("bool", {"m": ("bvec", "N")},
       lambda o, v: (lambda r: [o.dot(v["X"].T, r), o.sum(r)])(o.switch(v["m"], _rz(o, v), -_rz(o, v) - 1)), 1),
    # a scalar argument (uploaded: read by pointer) next to the clip bounds (constants: by value)
    _r("scalar", {"y": ("vec", "N"), "s": SCAL},
       lambda o, v: (lambda r: [o.dot(v["X"].T, r), o.sum(r)])(_rz(o, v) * v["y"] + v["s"]), 1),
    # a transcendental step
    _r("sigmoid", {"y": ("vec", "N")},
       lambda o, v: (lambda r: [o.dot(v["X"].T, r), o.sum(r)])(o.sigmoid(o.dot(v["X"], v["w"]) * F32(0.125)) - v["y"]), 1),
]}


@functools.lru_cache(maxsize=None)
def row_program(name):
    from aesara_b200.graphs import _at, optimized_program

    aesara, at = _at()
    case = ROW[name]
    v = {k: _sym(at, k, kind) for k, (kind, _) in case.inputs.items()}
    outs = case.fn(_SymOps(at), v)
    prog, _ = optimized_program(list(v.values()), outs, name=f"rowregion_{name}", linker="py")
    return prog


@functools.lru_cache(maxsize=None)
def gemm_program(name):
    """Lowered program of GEMM case ``name``; inputs in ``GEMM[name].inputs`` order."""
    from aesara_b200.graphs import _at, optimized_program

    aesara, at = _at()
    case = GEMM[name]
    v = {k: _sym(at, k, kind) for k, (kind, _) in case.inputs.items()}
    outs = case.fn(_SymOps(at), v)
    prog, _ = optimized_program(list(v.values()), outs, name=f"region_{name}", linker="py")
    return prog


def _sym(at, name, kind):
    return {"mat": at.fmatrix, "vec": at.fvector, "col": at.fcol, "scal": at.fscalar,
            "ivec": at.ivector, "bvec": lambda n: at.vector(n, dtype="bool")}[kind](name)


def int_inputs(case, dims, seed=0, lo=-4, hi=4):
    """Integer operands in [lo, hi] at the symbolic dims ``dims`` ({"M": .., "N": .., ...})."""
    rng = np.random.default_rng(seed)
    out = {}
    for k, (kind, shape) in case.inputs.items():
        if shape == "2N":
            shp = (2 * dims["N"],)
        else:
            shp = tuple(int(ch) if ch.isdigit() else dims[ch] for ch in shape.replace("+", ""))
        if shape.endswith("+"):  # one column more (sliced at column 1)
            shp = shp[:-1] + (shp[-1] + 1,)
        dt = {"ivec": np.int32, "bvec": np.bool_}.get(kind, F32)
        out[k] = rng.integers(lo, hi + 1, shp).astype(dt)
    return out


def truth(case, vals):
    """float64 evaluation of the outputs."""
    v = {k: np.asarray(a, np.float64) if a.dtype != np.bool_ else a for k, a in vals.items()}
    with np.errstate(all="ignore"):
        return [np.asarray(o, np.float64) for o in case.fn(_NpOps, v)]


def defines(src):
    """The ``#define AB_EP_*`` values of a generated module's own header (integers)."""
    out = {}
    for line in src.split("\n"):
        parts = line.split()
        if len(parts) == 3 and parts[0] == "#define" and parts[1].startswith("AB_EP_") and parts[1] not in out:
            try:
                out[parts[1]] = int(parts[2].strip("()"))
            except ValueError:
                pass
        if line.startswith("#define AB_EP_EVAL"):
            break
    return out
