"""Lower an optimised Aesara ``FunctionGraph`` to an :class:`aesara_b200.ir.Program`.

This is the only module (besides ``linker.py``) that touches Aesara objects.
It walks ``fgraph.toposort()`` (``aesara/graph/fg.py:766``) exactly like
``VMLinker.make_all`` does (``aesara/link/vm.py:1236-1252``) and emits one
program node per ``Apply``.  Ops with no device implementation raise
``NotImplementedError`` naming the Op — there is deliberately no CPU fallback
for tensor work (BASELINE north star).
"""

from __future__ import annotations

from typing import Dict, List

import numpy as np

from .ir import Node, Program, Var

_LOWERERS = {}


def lowers(*names):
    def deco(fn):
        for n in names:
            _LOWERERS[n] = fn
        return fn

    return deco


class UnsupportedOp(NotImplementedError):
    pass


# ---------------------------------------------------------------------------
# scalar expressions
# ---------------------------------------------------------------------------
# aesara scalar Op class name -> IR op name (semantics: aesara/scalar/basic.py
# c_code of each class; see aesara_b200/codegen/scalar_cuda.py for the table)
_SCALAR_OPS = {
    "LT": "lt", "GT": "gt", "LE": "le", "GE": "ge", "EQ": "eq", "NEQ": "neq",
    "IsNan": "isnan", "IsInf": "isinf", "Switch": "switch",
    "OR": "or", "XOR": "xor", "AND": "and", "Invert": "invert",
    "ScalarMaximum": "maximum", "ScalarMinimum": "minimum", "MulWithoutZeros": "mul_without_zeros",
    "Add": "add", "Mul": "mul", "Sub": "sub", "TrueDivide": "true_divide",
    "IntDiv": "int_div", "FloorDivide": "int_div", "Mod": "mod", "Pow": "pow",
    "Clip": "clip", "Second": "second", "Identity": "identity", "Cast": "cast",
    "Abs": "abs", "Sgn": "sgn", "Ceil": "ceil", "Floor": "floor", "Trunc": "trunc",
    "RoundHalfToEven": "round_half_to_even",
    "RoundHalfAwayFromZero": "round_half_away_from_zero",
    "Neg": "neg", "Reciprocal": "reciprocal", "Log": "log", "Log2": "log2",
    "Log10": "log10", "Log1p": "log1p", "Exp": "exp", "Exp2": "exp2",
    "Expm1": "expm1", "Sqr": "sqr", "Sqrt": "sqrt", "Deg2Rad": "deg2rad",
    "Rad2Deg": "rad2deg", "Cos": "cos", "ArcCos": "arccos", "Sin": "sin",
    "ArcSin": "arcsin", "Tan": "tan", "ArcTan": "arctan", "ArcTan2": "arctan2",
    "Cosh": "cosh", "ArcCosh": "arccosh", "Sinh": "sinh", "ArcSinh": "arcsinh",
    "Tanh": "tanh", "ArcTanh": "arctanh",
    "Sigmoid": "sigmoid", "Softplus": "softplus", "Log1mexp": "log1mexp",
    "Erf": "erf", "Erfc": "erfc", "Erfinv": "erfinv", "Erfcinv": "erfcinv",
    "Erfcx": "erfcx", "Gamma": "gamma", "GammaLn": "gammaln",
    "InRange": "inrange", "Mean": "mean",
}


def _scalar_const(v):
    data = np.asarray(v.data)
    val = data.item()
    if isinstance(val, complex):
        raise UnsupportedOp("complex scalar constants are not supported on device")
    return {"const": val, "dtype": data.dtype.name}


def lower_scalar_op(scalar_op, in_dtypes=None):
    """Return the IR scalar expression of a scalar Op applied to inputs of the
    given dtypes (``Composite`` graphs are inlined, recursively)."""
    stmts: List[dict] = []

    def emit(op, arg_refs, arg_dtypes, out_dtypes):
        """Append statements for ``op`` and return refs of its outputs."""
        cls = type(op).__name__
        if cls == "Composite":
            fg = op.fgraph
            env = {}
            for k, iv in enumerate(fg.inputs):
                env[iv] = arg_refs[k]
            for node in fg.toposort():
                refs, dts = [], []
                for iv in node.inputs:
                    if iv in env:
                        refs.append(env[iv])
                    elif hasattr(iv, "data"):
                        refs.append(_scalar_const(iv))
                    else:
                        raise UnsupportedOp(f"free scalar variable {iv} in {op}")
                    dts.append(iv.type.dtype)
                outs = emit(node.op, refs, dts, [o.type.dtype for o in node.outputs])
                for ov, r in zip(node.outputs, outs):
                    env[ov] = r
            res = []
            for ov in fg.outputs:
                if ov in env:
                    res.append(env[ov])
                elif hasattr(ov, "data"):
                    res.append(_scalar_const(ov))
                else:
                    raise UnsupportedOp(f"unbound Composite output {ov}")
            return res
        name = _SCALAR_OPS.get(cls)
        if name is None:
            raise UnsupportedOp(f"scalar op {cls} ({op}) has no device expression")
        st = {"op": name, "args": list(arg_refs), "dtype": out_dtypes[0],
              "in_dtypes": list(arg_dtypes)}
        if name == "inrange":
            st["openlow"], st["openhi"] = bool(op.openlow), bool(op.openhi)
        if len(out_dtypes) != 1:
            raise UnsupportedOp(f"multi-output scalar op {cls}")
        stmts.append(st)
        return [f"t{len(stmts) - 1}"]

    if in_dtypes is None:
        in_dtypes = [i.type.dtype for i in scalar_op.fgraph.inputs]
    # output dtypes via the op's own type inference
    from aesara.scalar.basic import get_scalar_type

    out_types = scalar_op.output_types([get_scalar_type(dt) for dt in in_dtypes])
    outs = emit(
        scalar_op,
        [f"i{k}" for k in range(len(in_dtypes))],
        list(in_dtypes),
        [t.dtype for t in out_types],
    )
    # an output may be an input or a constant directly (identity Composite)
    final = []
    for r, t in zip(outs, out_types):
        if isinstance(r, str) and r.startswith("t"):
            final.append(r)
        else:
            dt = t.dtype
            stmts.append({"op": "identity", "args": [r], "dtype": dt,
                          "in_dtypes": [dt if not isinstance(r, dict) else r["dtype"]]})
            final.append(f"t{len(stmts) - 1}")
    return {
        "inputs": list(in_dtypes),
        "stmts": stmts,
        "outputs": final,
        "out_dtypes": [t.dtype for t in out_types],
        "name": str(scalar_op),
    }


# ---------------------------------------------------------------------------
# graph lowering
# ---------------------------------------------------------------------------
class _Ctx:
    def __init__(self):
        self.vars: List[Var] = []
        self.ids: Dict[object, int] = {}

    def var_id(self, v):
        vid = self.ids.get(v)
        if vid is not None:
            return vid
        self.ids[v] = vid = len(self.vars)
        self.vars.append(_make_var(v))
        return vid


def _make_var(v):
    from aesara.graph.basic import Constant
    from aesara.scalar.basic import ScalarType
    from aesara.tensor.type import TensorType

    t = v.type
    name = getattr(v, "name", None)
    if isinstance(t, TensorType):
        var = Var(dtype=t.dtype, ndim=t.ndim, kind="tensor",
                  static_shape=tuple(t.shape), name=name)
        if isinstance(v, Constant):
            var.const = np.asarray(v.data, dtype=t.dtype)
        return var
    if isinstance(t, ScalarType):
        var = Var(dtype=t.dtype, ndim=0, kind="scalar", name=name)
        if isinstance(v, Constant):
            var.const = np.asarray(v.data, dtype=t.dtype)
        return var
    # NoneConst, slices, etc.
    var = Var(dtype=None, ndim=0, kind="other", name=name)
    if isinstance(v, Constant):
        data = v.data
        if data is None:
            var.const_other = {"none": True}
        elif isinstance(data, slice):
            var.const_other = {"slice": [data.start, data.stop, data.step]}
        else:
            raise UnsupportedOp(f"constant of type {t} is not supported")
    return var


def lower_fgraph(fgraph, name=None, order=None) -> Program:
    ctx = _Ctx()
    prog = Program(name=name)
    for iv in fgraph.inputs:
        prog.inputs.append(ctx.var_id(iv))
    if order is None:
        order = fgraph.toposort()
    for apply in order:
        node = lower_apply(apply, ctx)
        prog.nodes.append(node)
    for ov in fgraph.outputs:
        prog.outputs.append(ctx.var_id(ov))
    upd = getattr(fgraph, "update_mapping", None) or {}
    prog.updates = sorted((int(o), int(i)) for o, i in upd.items())
    prog.vars = ctx.vars
    return prog


def lower_apply(apply, ctx) -> Node:
    op = apply.op
    cls = type(op).__name__
    fn = None
    for klass in type(op).__mro__:
        fn = _LOWERERS.get(klass.__name__)
        if fn is not None:
            break
    if fn is None:
        raise UnsupportedOp(
            f"B200 backend: no device implementation for Op {cls} in node {apply}; "
            "there is no CPU fallback for tensor work"
        )
    ins = [ctx.var_id(v) for v in apply.inputs]
    outs = [ctx.var_id(v) for v in apply.outputs]
    opname, params = fn(op, apply)
    # generic destroy_map (graph/op.py: "destroy_map {out: [in]}"): which inputs this node
    # overwrites — the executor invalidates cached GEMM operand planes of those buffers and
    # refuses to defer a fused region across such a node (runtime/vm.py)
    dm = getattr(op, "destroy_map", None) or {}
    destroyed = sorted({int(i) for v in dm.values() for i in v})
    if destroyed:
        params = dict(params)
        params["destroy"] = destroyed
    return Node(op=opname, inputs=ins, outputs=outs, params=params, label=str(apply)[:200])


# -- elementwise / layout ------------------------------------------------------
@lowers("Elemwise")
def _l_elemwise(op, apply):
    expr = lower_scalar_op(op.scalar_op, [v.type.dtype for v in apply.inputs])
    want = [o.type.dtype for o in apply.outputs]
    if expr["out_dtypes"] != want:
        raise UnsupportedOp(
            f"Elemwise dtype inference mismatch {expr['out_dtypes']} vs {want} in {apply}"
        )
    return "Elemwise", {
        "expr": expr,
        "inplace": {str(int(o)): int(i) for o, i in (op.inplace_pattern or {}).items()},
    }


@lowers("DimShuffle")
def _l_dimshuffle(op, apply):
    return "DimShuffle", {"new_order": [x if x == "x" else int(x) for x in op.new_order]}


@lowers("CAReduce")
def _l_careduce(op, apply):
    sop = type(op.scalar_op).__name__
    name = _SCALAR_OPS.get(sop)
    if name not in ("add", "mul", "maximum", "minimum", "and", "or", "xor", "mul_without_zeros"):
        raise UnsupportedOp(f"CAReduce over scalar op {sop}")
    in_dtype = apply.inputs[0].type.dtype
    out_dtype = apply.outputs[0].type.dtype
    ndim = apply.inputs[0].type.ndim
    axis = op.axis
    if axis is None:
        axis = list(range(ndim))
    axis = sorted(int(a) % ndim if ndim else int(a) for a in axis)
    acc = getattr(op, "acc_dtype", None)
    if hasattr(op, "_acc_dtype"):
        acc_dtype = op._acc_dtype(in_dtype)
    else:
        acc_dtype = acc or out_dtype
    return "CAReduce", {
        "scalar_op": name, "axis": axis, "acc_dtype": str(acc_dtype),
        "in_dtype": in_dtype, "out_dtype": out_dtype,
    }


# -- row ops (SURVEY §8f N1) -------------------------------------------------------
def _axis_or_none(op):
    return None if op.axis is None else int(op.axis)


@lowers("Softmax")
def _l_softmax(op, apply):
    return "Softmax", {"axis": _axis_or_none(op), "mode": 0}


@lowers("LogSoftmax")
def _l_logsoftmax(op, apply):
    return "Softmax", {"axis": _axis_or_none(op), "mode": 1}


@lowers("SoftmaxGrad")
def _l_softmaxgrad(op, apply):
    return "Softmax", {"axis": _axis_or_none(op), "mode": 2}


@lowers("MaxAndArgmax")
def _l_maxandargmax(op, apply):
    ndim = apply.inputs[0].type.ndim
    axis = op.axis
    axes = list(range(ndim)) if axis is None else sorted(int(a) % ndim for a in axis)
    return "MaxAndArgmax", {"axes": axes}


@lowers("Argmax")
def _l_argmax(op, apply):
    ndim = apply.inputs[0].type.ndim
    axis = op.axis
    axes = list(range(ndim)) if axis is None else sorted(int(a) % ndim for a in axis)
    return "MaxAndArgmax", {"axes": axes, "argmax_only": True}


# -- BLAS family -----------------------------------------------------------------
@lowers("Dot22")
def _l_dot22(op, apply):
    return "Dot22", {}


@lowers("Dot22Scalar")
def _l_dot22scalar(op, apply):
    return "Dot22Scalar", {}


@lowers("Gemm")
def _l_gemm(op, apply):
    return "Gemm", {"inplace": bool(op.inplace)}


@lowers("Gemv", "CGemv")
def _l_gemv(op, apply):
    return "Gemv", {"inplace": bool(op.inplace)}


@lowers("Ger", "CGer")
def _l_ger(op, apply):
    return "Ger", {"inplace": bool(op.destructive)}


@lowers("Dot")
def _l_dot(op, apply):
    return "Dot", {}


# -- allocation / copies -----------------------------------------------------------
@lowers("AllocEmpty")
def _l_allocempty(op, apply):
    return "AllocEmpty", {"dtype": op.dtype}


@lowers("Alloc")
def _l_alloc(op, apply):
    return "Alloc", {}


@lowers("BroadcastTo")
def _l_broadcast_to(op, apply):
    # tensor/extra_ops.py:1613 BroadcastTo: a (read-only) broadcast VIEW of input 0
    # (view_map {0: [0]}) -- stride-0 dims on device
    return "BroadcastTo", {}


@lowers("DeepCopyOp")
def _l_deepcopy(op, apply):
    return "DeepCopy", {}


@lowers("ViewOp", "Unbroadcast", "SpecifyShape", "OutputGuard")
def _l_view(op, apply):
    return "View", {}


@lowers("Reshape")
def _l_reshape(op, apply):
    return "Reshape", {"ndim": int(op.ndim)}


# -- host-side metadata (SURVEY a9) --------------------------------------------------
@lowers("Shape_i")
def _l_shape_i(op, apply):
    return "Shape_i", {"i": int(op.i)}


@lowers("Shape")
def _l_shape(op, apply):
    return "Shape", {}


@lowers("ScalarFromTensor")
def _l_sft(op, apply):
    return "ScalarFromTensor", {}


@lowers("TensorFromScalar")
def _l_tfs(op, apply):
    return "TensorFromScalar", {}


@lowers("MakeVector")
def _l_makevector(op, apply):
    return "MakeVector", {"dtype": op.dtype}


@lowers("CheckAndRaise")
def _l_assert(op, apply):
    return "Assert", {"msg": str(op.msg), "exc": op.exc_type.__name__}


@lowers("ScalarOp")
def _l_scalarop(op, apply):
    # a scalar Op applied directly to ScalarType variables (shape arithmetic)
    expr = lower_scalar_op(op, [v.type.dtype for v in apply.inputs])
    return "ScalarOp", {"expr": expr}


# -- indexing -------------------------------------------------------------------------
def _idx_list_json(idx_list):
    from aesara.graph.type import Type

    def elem(e):
        if e is None:
            return None
        if isinstance(e, Type):
            return "in"
        return int(e)

    out = []
    for entry in idx_list:
        if isinstance(entry, slice):
            out.append({"slice": [elem(entry.start), elem(entry.stop), elem(entry.step)]})
        else:
            out.append({"index": elem(entry)})
    return out


@lowers("Subtensor")
def _l_subtensor(op, apply):
    return "Subtensor", {"idx_list": _idx_list_json(op.idx_list)}


@lowers("IncSubtensor")
def _l_incsubtensor(op, apply):
    return "IncSubtensor", {
        "idx_list": _idx_list_json(op.idx_list),
        "inplace": bool(op.inplace),
        "set": bool(op.set_instead_of_inc),
    }


@lowers("AdvancedSubtensor1")
def _l_advsub1(op, apply):
    return "AdvancedSubtensor1", {}


@lowers("AdvancedIncSubtensor1")
def _l_advincsub1(op, apply):
    return "AdvancedIncSubtensor1", {"inplace": bool(op.inplace), "set": bool(op.set_instead_of_inc)}


def _int_vector_indices(apply, first):
    """AdvancedSubtensor / AdvancedIncSubtensor are lowered for the integer-array form only:
    one integer vector (or 0-d integer) per leading dimension of x, no slices / newaxis /
    boolean masks (subtensor.py:2577-2805)."""
    for v in apply.inputs[first:]:
        t = v.type
        if not hasattr(t, "dtype") or not hasattr(t, "ndim") or str(t.dtype)[:3] not in ("int", "uin") or t.ndim > 1:
            raise UnsupportedOp(
                f"B200 backend: {apply.op} is implemented for integer index vectors only "
                f"(got an index of type {t}); there is no CPU fallback for tensor work")
    return len(apply.inputs) - first


@lowers("AdvancedSubtensor")
def _l_advsub(op, apply):
    return "AdvancedSubtensor", {"n_idx": _int_vector_indices(apply, 1)}


@lowers("AdvancedIncSubtensor")
def _l_advincsub(op, apply):
    return "AdvancedIncSubtensor", {"n_idx": _int_vector_indices(apply, 2), "inplace": bool(op.inplace),
                                    "set": bool(op.set_instead_of_inc),
                                    "ignore_duplicates": bool(getattr(op, "ignore_duplicates", False))}


@lowers("BatchedDot")
def _l_batched_dot(op, apply):
    # tensor/blas.py:2232 BatchedDot: z[b] = dot(x[b], y[b]) for 2-D / 3-D operands
    return "BatchedDot", {}


@lowers("IfElse")
def _l_ifelse(op, apply):
    # aesara/ifelse.py:44: outputs = the `then` values if the condition is true, else the
    # `else` values.  The reference VM evaluates only the taken branch (lazy thunk); this
    # executor runs nodes in schedule order, so both branches exist by the time the node
    # runs and it only selects (same values, no laziness).
    return "IfElse", {"n_outs": int(op.n_outs), "as_view": bool(op.as_view)}


@lowers("CumOp")
def _l_cumop(op, apply):
    return "CumOp", {"axis": None if op.axis is None else int(op.axis), "mode": str(op.mode)}


@lowers("ExtractDiag")
def _l_extract_diag(op, apply):
    # tensor/basic.py:3480 ExtractDiag: ndarray.diagonal(offset, axis1, axis2) — a view of the
    # input when op.view, else a copy
    return "ExtractDiag", {"offset": int(op.offset), "axis1": int(op.axis1), "axis2": int(op.axis2),
                           "view": bool(op.view)}


@lowers("AllocDiag")
def _l_alloc_diag(op, apply):
    # tensor/basic.py:3600 AllocDiag (the gradient of ExtractDiag): a zero matrix with the
    # input vector on its `offset` diagonal; lowered for vector inputs
    if apply.inputs[0].type.ndim != 1 or (int(op.axis1), int(op.axis2)) != (0, 1):
        raise UnsupportedOp("B200 backend: AllocDiag is implemented for vector inputs only; "
                            "there is no CPU fallback for tensor work")
    return "AllocDiag", {"offset": int(op.offset)}


@lowers("Tri")
def _l_tri(op, apply):
    return "Tri", {"dtype": str(op.dtype)}


@lowers("Eye")
def _l_eye(op, apply):
    return "Eye", {"dtype": str(op.dtype)}


@lowers("ARange")
def _l_arange(op, apply):
    return "ARange", {"dtype": str(op.dtype)}


@lowers("Join")
def _l_join(op, apply):
    return "Join", {}


@lowers("Split")
def _l_split(op, apply):
    return "Split", {"len_splits": int(op.len_splits)}


# -- random variables ------------------------------------------------------------------
# RandomVariable (aesara/tensor/random/op.py:344 perform): inputs (rng, size, dtype, *params),
# outputs (rng_out, sample).  The device draws from its own Philox stream keyed by one 64-bit
# draw of the node's Generator (runtime/vm.py, csrc/ab_random.cu); the Generator stays a host
# value.  Distribution class -> (device distribution, output dtypes it draws).
_RV_DISTS = {
    "UniformRV": ("uniform", ("float32", "float64")),
    "NormalRV": ("normal", ("float32", "float64")),
    "BernoulliRV": ("bernoulli", ("int64",)),
    "BinomialRV": ("bernoulli", ("int64",)),
}


@lowers("RandomVariable")
def _l_random_variable(op, apply):
    from aesara.graph.basic import Constant
    from aesara.tensor.random.type import RandomGeneratorType

    cls = type(op).__name__
    name = getattr(op, "name", cls)
    what = f"B200 backend: random variable {name} ({cls})"
    hit = _RV_DISTS.get(cls)
    if hit is None:
        raise UnsupportedOp(f"{what} has no device implementation (device draws: uniform, normal, "
                            "bernoulli, binomial with n = 1); there is no CPU fallback for tensor work")
    if not isinstance(apply.inputs[0].type, RandomGeneratorType):
        raise UnsupportedOp(f"{what}: the rng is a {apply.inputs[0].type}; the device draws from "
                            "numpy Generator rngs only (RandomStream, not RandomState)")
    dist, dtypes = hit
    out_dtype = apply.outputs[1].type.dtype
    if out_dtype not in dtypes:
        raise UnsupportedOp(f"{what}: no device draw of dtype {out_dtype}")
    if cls == "BinomialRV":
        n = apply.inputs[3]
        if not (isinstance(n, Constant) and np.all(np.asarray(n.data) == 1)):
            raise UnsupportedOp(f"{what}: the device draws binomial variables with the constant n = 1 "
                                "(Bernoulli) only")
    return "RandomVariable", {"dist": dist, "dtype": out_dtype, "inplace": bool(op.inplace)}


# -- dense linear algebra ----------------------------------------------------------------
# aesara/tensor/slinalg.py.  Registered by concrete class: every other SolveBase subclass (and
# every other slinalg / nlinalg Op) has no device implementation.
_LINALG_DTYPES = ("float32", "float64")


def _linalg_out_dtype(op, apply):
    dt = apply.outputs[0].type.dtype
    if dt not in _LINALG_DTYPES:
        raise UnsupportedOp(f"B200 backend: {type(op).__name__} with output dtype {dt} has no device "
                            "implementation (float32, float64)")
    return dt


@lowers("Cholesky")
def _l_cholesky(op, apply):
    dt = apply.inputs[0].type.dtype
    if dt not in _LINALG_DTYPES:
        raise UnsupportedOp(f"B200 backend: Cholesky of a {dt} matrix has no device implementation: the "
                            "reference casts the factor back to the input dtype, which for integers "
                            "truncates it; the device factors float32 and float64 matrices")
    return "Cholesky", {"lower": bool(op.lower), "on_error": str(op.on_error)}


_TRANS = {0: 0, 1: 1, 2: 1, "N": 0, "T": 1, "C": 1}  # 2 / "C" (conjugate transpose) is 1 for real data


@lowers("SolveTriangular")
def _l_solve_triangular(op, apply):
    _linalg_out_dtype(op, apply)
    if op.trans not in _TRANS:
        raise UnsupportedOp(f"B200 backend: SolveTriangular with trans={op.trans!r}")
    return "SolveTriangular", {"lower": bool(op.lower), "trans": _TRANS[op.trans],
                               "unit_diagonal": bool(op.unit_diagonal), "check_finite": bool(op.check_finite)}


@lowers("CholeskySolve")
def _l_cholesky_solve(op, apply):
    _linalg_out_dtype(op, apply)
    return "CholeskySolve", {"lower": bool(op.lower), "check_finite": bool(op.check_finite)}


@lowers("Solve")
def _l_solve(op, apply):
    if op.assume_a != "pos":
        raise UnsupportedOp(f"B200 backend: Solve(assume_a={op.assume_a!r}) has no device implementation: "
                            "the device solves positive definite systems (assume_a='pos') by Cholesky; "
                            "the LU / LDL^T factorisations of 'gen', 'sym' and 'her' are not implemented")
    _linalg_out_dtype(op, apply)
    return "Solve", {"lower": bool(op.lower), "check_finite": bool(op.check_finite)}


# -- Scan --------------------------------------------------------------------------------
def optimized_inner_fgraph(op):
    """The inner graph of a ``Scan`` as the reference would *execute* it.

    ``op.fgraph`` as stored in the outer graph is the raw inner function: the reference
    rewrites it only when ``Scan.fn`` is first touched (``scan/op.py:1431-1459``:
    ``pfunc(..., mode=self.mode_instance, fgraph=self.fgraph)`` mutates it in place with the
    protections ``prepare_fgraph`` sets up, ``:1300-1428``).  Lowering must not depend on
    whether some other linker happened to trigger that side effect, so the same compilation
    is run here on a *clone* of the Op with a linker that links nothing: what comes back is
    the rewritten graph (``Dot`` -> ``Gemm``, fused ``Composite``s, in-place ops where the
    Supervisor allows them, ``DeepCopyOp`` on outputs that alias inputs)."""
    from aesara.compile.mode import Mode

    if getattr(op, "_fn", None) is not None:
        # the reference already compiled this Op (a C-linker function over the same graph,
        # debug.check_function): op.fgraph IS the rewritten graph
        return op.fgraph
    op2 = op.clone()  # copy(op) + fgraph.clone()  (scan/op.py:1469-1472)
    op2._fn = None
    inner_mode = op.mode_instance
    op2.mode_instance = Mode(linker=_LinkNothing(), optimizer=inner_mode.provided_optimizer,
                             db=inner_mode.optdb)
    op2.fn  # noqa: B018  -- compiles: rewrites op2.fgraph in place
    return op2.fgraph


def _link_nothing_cls():
    from aesara.link.basic import Container, LocalLinker
    from aesara.link.utils import map_storage

    class LinkNothing(LocalLinker):
        """A linker that only allocates the storage cells ``Function`` wants to see."""

        def __init__(self):
            super().__init__()
            self.fgraph = None

        def accept(self, fgraph, no_recycling=None, profile=None):
            if self.fgraph is not None and self.fgraph is not fgraph:
                return type(self)().accept(fgraph, no_recycling, profile)
            self.fgraph = fgraph
            self.no_recycling = no_recycling or []
            return self

        def make_all(self, input_storage=None, output_storage=None, storage_map=None):
            fgraph = self.fgraph
            order = self.schedule(fgraph)
            input_storage, output_storage, storage_map = map_storage(
                fgraph, order, input_storage, output_storage, storage_map)

            def fn():
                raise RuntimeError("this inner function exists for its rewritten graph only")

            fn.allow_gc = False
            fn.storage_map = storage_map
            return (fn, [Container(i, s) for i, s in zip(fgraph.inputs, input_storage)],
                    [Container(o, s, readonly=True) for o, s in zip(fgraph.outputs, output_storage)],
                    [], order)

    return LinkNothing


_LINK_NOTHING = None


def _LinkNothing():
    global _LINK_NOTHING
    if _LINK_NOTHING is None:
        _LINK_NOTHING = _link_nothing_cls()
    return _LINK_NOTHING()


@lowers("Scan")
def _l_scan(op, apply):
    info = op.info
    inner = lower_fgraph(optimized_inner_fgraph(op), name=f"scan_inner:{getattr(op, 'name', None)}")
    return "Scan", {
        "info": {
            "n_seqs": info.n_seqs,
            "mit_mot_in_slices": [list(x) for x in info.mit_mot_in_slices],
            "mit_mot_out_slices": [list(x) for x in info.mit_mot_out_slices],
            "mit_sot_in_slices": [list(x) for x in info.mit_sot_in_slices],
            "sit_sot_in_slices": [list(x) for x in info.sit_sot_in_slices],
            "n_nit_sot": info.n_nit_sot,
            "n_shared_outs": info.n_shared_outs,
            "n_non_seqs": info.n_non_seqs,
            "as_while": bool(info.as_while),
        },
        "inner": inner,
        "destroy_map": {str(k): list(v) for k, v in (op.destroy_map or {}).items()},
    }
