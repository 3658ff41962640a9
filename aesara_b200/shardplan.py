"""Which graphs shard over their leading ("row") axis, and how their outputs combine.

SURVEY.md §8e, the general rule: *a graph input axis is shardable iff every consumer treats it
as a broadcast-free Elemwise axis, the M axis of Gemm/Gemv/Dot22, a Scan batch axis, or reduces
it with a CAReduce (-> partial + combine).  Otherwise replicas only.*  The reference has no
notion of this (it has no parallelism at all, SURVEY F2); the ops whose semantics the rule
walks are ``Elemwise`` (``tensor/elemwise.py:304``), ``CAReduce`` (``:1221``), ``Dot22`` /
``Gemm`` (``tensor/blas.py:1659/872``), ``Gemv`` (``:231``), ``DimShuffle`` (``elemwise.py:39``)
and the int64 shape arithmetic around them (``Shape_i`` ``tensor/shape.py:189`` ...).

This module is pure host logic over the lowered program: it propagates one label per variable

    ("rep",)          identical on every rank (weights, constants, shapes of unsharded dims)
    ("scal", q)       a host scalar proportional to (local row count)**q — what ``x.shape[0]``
                      of a sharded ``x`` is, and what ``mean`` divides by
    ("vec", qs)       a small shape vector, element i proportional to rows**qs[i]
    ("rows", a, p)    sharded along its axis ``a``: the unsharded value restricted to this
                      rank's rows equals local * (n_r / N)**p   (p != 0 after dividing by a
                      local row count, e.g. the ``2*diff/n`` of an MSE gradient)
    ("part", p)       a partial result of a reduction / contraction over the sharded axis: the
                      unsharded value is  sum_r (n_r / N)**p * local_r

and derives, per function output, how the ranks' results combine: ``sum`` (p = 0), ``mean``
(p = 1: weights n_r / N), ``concat`` along an axis, or ``rep``.  Whatever it cannot prove raises
``ReplicasOnly`` naming the node — never a silently wrong combination.
"""

from __future__ import annotations

from dataclasses import dataclass
from typing import Dict, List, Optional, Sequence, Tuple

REP = ("rep",)


class ReplicasOnly(ValueError):
    """The graph is not a row-wise batch map (plus batch reductions): run replicas instead."""


@dataclass
class ShardPlan:
    sharded_inputs: List[Optional[int]]      # per function input: sharded axis or None
    outputs: List[Tuple]                     # per output: ("sum",) ("mean",) ("concat", axis) ("rep",)
    labels: Dict[int, Tuple]                 # every variable's label (for inspection / tests)

    def reductions(self):
        return [k for k, o in enumerate(self.outputs) if o[0] in ("sum", "mean")]


# ---------------------------------------------------------------------------- scalar algebra
_NONLINEAR_OK = ("rep",)
_CMP = {"lt", "gt", "le", "ge", "eq", "neq", "isnan", "isinf", "and", "or", "xor", "invert", "inrange"}
_LINEAR_UNARY = {"neg", "identity", "cast"}


def _fail(node, why):
    raise ReplicasOnly(f"replicas only: {node.label or node.op}: {why}")


def _mul(a, b, node):
    ka, kb = a[0], b[0]
    if ka == "rep":
        return b
    if kb == "rep":
        return a
    if ka == "scal" and kb == "scal":
        return ("scal", a[1] + b[1])
    if ka == "scal":
        a, b, ka, kb = b, a, kb, ka
    if kb == "scal":  # multiplying by rows**q lowers the (n_r/N) power by q
        if ka == "rows":
            return ("rows", a[1], a[2] - b[1])
        if ka == "part":
            return ("part", a[1] - b[1])
    if ka == "rows" and kb == "rows":
        if a[1] != b[1]:
            _fail(node, "product of values sharded along different axes")
        return ("rows", a[1], a[2] + b[2])
    _fail(node, f"product of {a} and {b}")


def _div(a, b, node):
    kb = b[0]
    if kb == "rep":
        return a
    if kb == "scal":
        if a[0] == "rep":
            return ("scal", -b[1])
        if a[0] == "scal":
            return ("scal", a[1] - b[1])
        if a[0] == "rows":
            return ("rows", a[1], a[2] + b[1])
        if a[0] == "part":
            return ("part", a[1] + b[1])
    if kb == "rows" and b[2] == 0 and a[0] in ("rep", "rows"):
        if a[0] == "rows" and a[1] != b[1]:
            _fail(node, "quotient of values sharded along different axes")
        return ("rows", b[1], a[2] if a[0] == "rows" else 0)
    _fail(node, f"quotient of {a} and {b}")


def _add(labels, node):
    out = labels[0]
    for b in labels[1:]:
        a = out
        if a == b:
            continue
        if a[0] == "rows" and b[0] == "rows":
            _fail(node, f"sum of {a} and {b}")
        if a[0] == "rep" and b[0] == "rows" and b[2] == 0:
            out = b
        elif b[0] == "rep" and a[0] == "rows" and a[2] == 0:
            out = a
        else:
            _fail(node, f"sum of {a} and {b}")
    return out


def _nonlinear(labels, node, op):
    kinds = {l[0] for l in labels}
    if kinds <= {"rep"}:
        return REP
    if kinds <= {"rep", "rows"}:
        axes = {l[1] for l in labels if l[0] == "rows"}
        if len(axes) == 1 and all(l[2] == 0 for l in labels if l[0] == "rows"):
            return ("rows", axes.pop(), 0)
    if kinds <= {"rep", "scal"}:
        if op in _CMP:
            return REP  # shape checks (Assert conditions) are local decisions
        if op in ("switch", "maximum", "minimum", "abs"):
            # broadcast resolution of a dimension (`max(switch(d == 1, -1, d), ...)`): the row
            # count of the sharded operands, whatever the replicated (size 1) ones say
            qs = {l[1] for l in labels if l[0] == "scal"}
            if len(qs) == 1:
                return ("scal", qs.pop())
    _fail(node, f"{op} of {labels} is not a batch map")


def eval_expr_labels(expr, in_labels, node):
    """Propagate labels through a scalar expression (one label per temporary)."""
    temps = []

    def ref(r):
        if isinstance(r, dict):
            return REP
        return in_labels[int(r[1:])] if r[0] == "i" else temps[int(r[1:])]

    for st in expr["stmts"]:
        a = [ref(r) for r in st["args"]]
        op = st["op"]
        if op in _LINEAR_UNARY:
            if op == "cast" and a[0][0] in ("rows", "part") and not st["dtype"].startswith("float"):
                out = _nonlinear(a, node, op)
            else:
                out = a[0]
        elif op == "mul":
            out = a[0]
            for b in a[1:]:
                out = _mul(out, b, node)
        elif op == "true_divide":
            out = _div(a[0], a[1], node)
        elif op in ("add", "sub"):
            out = _add(a, node)
        elif op == "sqr":
            out = _mul(a[0], a[0], node)
        elif op == "second":
            out = a[1] if a[0][0] == "rep" else _nonlinear(a, node, op)
        elif op == "switch" and a[0][0] == "rep" and a[1] == a[2]:
            out = a[1]
        else:
            out = _nonlinear(a, node, op)
        temps.append(out)
    return [ref(r) for r in expr["outputs"]]


# ---------------------------------------------------------------------------- node rules
def _matmul(x, y, node):
    """x [m, k] @ y [k, n]."""
    kx, ky = x[0], y[0]
    if kx == "rep" and ky == "rep":
        return REP
    if kx == "rows" and ky == "rep" and x[1] == 0:
        return ("rows", 0, x[2])
    if kx == "rep" and ky == "rows" and y[1] == 1:
        return ("rows", 1, y[2])
    if kx == "rows" and ky == "rows" and x[1] == 1 and y[1] == 0:
        return ("part", x[2] + y[2])          # contraction over the sharded axis
    _fail(node, f"product of {x} and {y} (the sharded axis must be M, N or the whole of K)")


def _scale(lab, s, node):
    return _mul(lab, s, node) if s[0] != "rep" else lab


def _spans_axis(program, vid, axis):
    """True unless variable ``vid`` is known (statically) to have extent 1 along ``axis`` —
    a replicated operand that spans the sharded axis of its partner would have the GLOBAL row
    count there: not a batch map (and a shape error at run time)."""
    v = program.vars[vid]
    if v.ndim == 0 or axis >= v.ndim:
        return False
    if v.const is not None:
        return v.const.shape[axis] != 1
    ss = v.static_shape
    return ss is None or ss[axis] != 1


def _check_rep_operands(program, n, ins, var_ids=None):
    axes = {l[1] for l in ins if l[0] == "rows"}
    if not axes:
        return
    a = next(iter(axes))
    for v, l in zip(var_ids if var_ids is not None else n.inputs, ins):
        if l == REP and _spans_axis(program, v, a):
            _fail(n, f"replicated operand {program.vars[v].name or v} spans the sharded axis {a}")


def analyse(program, sharded_inputs: Sequence[Optional[int]], _inner=False) -> ShardPlan:
    """``sharded_inputs[i]``: the axis along which function input i is split (usually 0), or
    None for a replicated input."""
    L: Dict[int, Tuple] = {}
    for vid, v in enumerate(program.vars):
        if v.const is not None or v.const_other is not None:
            L[vid] = REP
    if len(sharded_inputs) != len(program.inputs):
        raise ValueError("one entry per function input")
    for vid, ax in zip(program.inputs, sharded_inputs):
        if ax is None:
            L[vid] = REP
        else:
            if program.vars[vid].kind != "tensor" or not 0 <= ax < program.vars[vid].ndim:
                raise ValueError(f"input {program.vars[vid].name or vid} has no axis {ax}")
            L[vid] = ("rows", int(ax), 0)

    for n in program.nodes:
        ins = [L[v] for v in n.inputs]
        op = n.op
        outs = None
        if op == "RandomVariable":
            # each rank would draw its own key from its own copy of the Generator: neither
            # a row block of one sample nor one shared update of the rng
            _fail(n, "a random variable draws from host Generator state")
        if op in ("Cholesky", "SolveTriangular", "CholeskySolve", "Solve"):
            # every element of a factor or a solution depends on every row of the matrix
            _fail(n, "a factorisation or triangular solve is not a row-wise batch map")
        if all(l == REP for l in ins) and op != "Scan":
            outs = [REP] * len(n.outputs)
        elif op == "Elemwise" or op == "ScalarOp":
            # operands sharded along an axis must agree on it (equal ndim inside an Elemwise);
            # replicated ones must broadcast along it
            if op == "Elemwise":
                _check_rep_operands(program, n, ins)
            outs = eval_expr_labels(n.params["expr"], ins, n)
        elif op == "DimShuffle":
            (x,) = ins
            if x[0] == "rows":
                order = list(n.params["new_order"])
                if x[1] not in order:
                    _fail(n, "drops the sharded axis")
                outs = [("rows", order.index(x[1]), x[2])]
            elif x[0] in ("scal", "part"):
                outs = [x]
            else:
                _fail(n, f"DimShuffle of {x}")
        elif op in ("Dot22", "Dot"):
            x, y = ins
            if op == "Dot" and (program.vars[n.inputs[0]].ndim != 2 or program.vars[n.inputs[1]].ndim != 2):
                xv, yv = program.vars[n.inputs[0]].ndim, program.vars[n.inputs[1]].ndim
                outs = [_dot_vec(x, y, xv, yv, n)]
            else:
                outs = [_matmul(x, y, n)]
        elif op == "Dot22Scalar":
            outs = [_scale(_matmul(ins[0], ins[1], n), ins[2], n)]
        elif op == "Gemm":
            z, a, x, y, b = ins
            prod = _scale(_matmul(x, y, n), a, n)
            zz = _scale(z, b, n)
            if _is_zero_const(program, n.inputs[4]):
                outs = [prod]
            else:
                _check_rep_operands(program, n, [zz, prod], [n.inputs[0], n.outputs[0]])
                outs = [_add([zz, prod], n)]
        elif op == "Gemv":
            y0, a, A, x, b = ins
            if A[0] == "rows" and A[1] == 0 and x[0] == "rep":
                prod = ("rows", 0, A[2])
            elif A[0] == "rows" and A[1] == 1 and x[0] == "rows" and x[1] == 0:
                prod = ("part", A[2] + x[2])
            elif A[0] == "rep" and x[0] == "rep":
                prod = REP
            else:
                _fail(n, f"Gemv of {A} and {x}")
            prod = _scale(prod, a, n)
            if _is_zero_const(program, n.inputs[4]):
                outs = [prod]       # beta == 0: y is not read (blas_c.py:418-430)
            else:
                outs = [_add([_scale(y0, b, n), prod], n)]
        elif op == "CAReduce":
            (x,) = ins
            axes = list(n.params["axis"] or [])
            nd = program.vars[n.inputs[0]].ndim
            if not axes:
                axes = list(range(nd)) if n.params["axis"] is None else []
            if x[0] == "rows":
                if x[1] in axes:
                    if n.params["scalar_op"] != "add":
                        _fail(n, "only sums reduce the sharded axis")
                    outs = [("part", x[2])]
                else:
                    outs = [("rows", x[1] - sum(1 for a in axes if a < x[1]), x[2])]
            elif x[0] == "part" and n.params["scalar_op"] == "add":
                outs = [x]
            else:
                _fail(n, f"reduction of {x}")
        elif op == "Shape_i":
            (x,) = ins
            outs = [("scal", 1) if (x[0] == "rows" and x[1] == n.params["i"]) else REP]
        elif op in ("ScalarFromTensor", "TensorFromScalar", "View", "DeepCopy", "Unbroadcast"):
            outs = [ins[0]]
        elif op == "Assert":
            outs = [ins[0]]
        elif op == "MakeVector":
            if any(l[0] not in ("rep", "scal") for l in ins):
                _fail(n, "vector of sharded values")
            outs = [("vec", tuple(l[1] if l[0] == "scal" else 0 for l in ins))]
        elif op == "Subtensor":
            x = ins[0]
            idx = n.params["idx_list"]
            if x[0] == "vec":
                k = None
                if len(idx) == 1 and "index" in idx[0]:
                    k = idx[0]["index"]
                    if k == "in":  # run-time index input: usable when it is a constant
                        c = program.vars[n.inputs[1]].const if len(n.inputs) > 1 else None
                        k = None if c is None else int(c)
                if k is None:
                    _fail(n, "slicing a shape vector of a sharded value")
                q = x[1][int(k)]
                outs = [("scal", q) if q else REP]
            elif x[0] == "rows":
                if any(l != REP for l in ins[1:]):
                    _fail(n, "index depends on a local shape")
                a = x[1]
                if a < len(idx):
                    e = idx[a]
                    if "slice" not in e or any(s is not None for s in e["slice"]):
                        _fail(n, "indexes into the sharded axis")
                dropped = sum(1 for e in idx[:a] if "index" in e)
                outs = [("rows", a - dropped, x[2])]
            else:
                _fail(n, f"Subtensor of {x}")
        elif op == "IncSubtensor":
            x, y = ins[0], ins[1]
            idx = n.params["idx_list"]
            if any(l != REP for l in ins[2:]):
                _fail(n, "index depends on a local shape")
            if x[0] != "rows" or x[2] != 0:
                _fail(n, f"writes into {x}")
            a = x[1]
            if a < len(idx) and ("slice" not in idx[a] or any(e is not None for e in idx[a]["slice"])):
                _fail(n, "writes along the sharded axis")
            dropped = sum(1 for e in idx[:a] if "index" in e)
            xnd = program.vars[n.inputs[0]].ndim - sum(1 for e in idx if "index" in e)
            ynd = program.vars[n.inputs[1]].ndim
            if y[0] == "rows":
                if y[2] != 0 or y[1] + (xnd - ynd) != a - dropped:
                    _fail(n, "value is sharded along another axis than its destination")
            elif y != REP or _spans_axis(program, n.inputs[1], a - dropped - (xnd - ynd)):
                _fail(n, f"value {y} written into a sharded buffer")
            outs = [x]
        elif op in ("AllocEmpty", "Alloc", "BroadcastTo"):
            shape = ins if op == "AllocEmpty" else ins[1:]
            if op != "AllocEmpty" and ins[0] != REP:
                _fail(n, "fills with a sharded value")
            axes = [k for k, l in enumerate(shape) if l[0] == "scal"]
            if len(axes) != 1 or shape[axes[0]][1] != 1 or any(l[0] not in ("rep", "scal") for l in shape):
                _fail(n, "allocation shape mixes local row counts")
            outs = [("rows", axes[0], 0)]
        elif op == "Softmax":
            # Softmax / LogSoftmax (mode 0 / 1) of x; SoftmaxGrad (mode 2) of (dy, sm): linear in dy
            x = ins[-1]
            ax = n.params["axis"]
            nd = program.vars[n.inputs[-1]].ndim
            if not (x[0] == "rows" and x[2] == 0 and ax is not None and ax % nd != x[1]):
                _fail(n, "softmax over the sharded axis")
            if n.params["mode"] == 2:
                dy = ins[0]
                if dy[0] != "rows" or dy[1] != x[1]:
                    _fail(n, f"SoftmaxGrad of {dy} and {x}")
                outs = [dy]
            else:
                outs = [x]
        elif op == "MaxAndArgmax":
            (x,) = ins
            axes = list(n.params["axes"])
            if not (x[0] == "rows" and x[2] == 0 and x[1] not in axes):
                _fail(n, "maximum over the sharded axis")
            outs = [("rows", x[1] - sum(1 for a in axes if a < x[1]), 0)] * len(n.outputs)
        elif op == "Reshape":
            _fail(n, "reshape of a sharded value")
        elif op == "Scan":
            outs = _scan(program, n, ins)
        else:
            _fail(n, "no sharding rule for this op")
        if len(outs) != len(n.outputs):
            outs = list(outs) + [outs[-1]] * (len(n.outputs) - len(outs))
        for v, l in zip(n.outputs, outs):
            L[v] = l

    out_modes = []
    for k, v in enumerate(program.outputs):
        l = L[v]
        if l[0] == "rep":
            out_modes.append(("rep",))
        elif l[0] == "part" and l[1] == 0:
            out_modes.append(("sum",))
        elif l[0] == "part" and l[1] == 1:
            out_modes.append(("mean",))
        elif l[0] == "rows" and l[2] == 0:
            out_modes.append(("concat", l[1]))
        elif _inner:
            out_modes.append(l)
        else:
            raise ReplicasOnly(f"replicas only: output {k} is {l}: no combination rule")
    return ShardPlan([a if a is None else int(a) for a in sharded_inputs], out_modes, L)


def _is_zero_const(program, vid):
    c = program.vars[vid].const
    return c is not None and float(c) == 0.0


def _dot_vec(x, y, xnd, ynd, node):
    if xnd == 2 and ynd == 1:
        if x[0] == "rows" and x[1] == 0 and y[0] == "rep":
            return ("rows", 0, x[2])
        if x[0] == "rows" and x[1] == 1 and y[0] == "rows":
            return ("part", x[2] + y[2])
    if xnd == 1 and ynd == 2:
        if x[0] == "rows" and y[0] == "rows" and y[1] == 0:
            return ("part", x[2] + y[2])
        if x[0] == "rep" and y[0] == "rows" and y[1] == 1:
            return ("rows", 0, y[2])
    if xnd == 1 and ynd == 1 and x[0] == "rows" and y[0] == "rows":
        return ("part", x[2] + y[2])
    _fail(node, f"Dot of {x} and {y}")


def _scan(program, n, ins):
    """A Scan whose sequences [T, B, ...] and states [k, B, ...] are sharded along axis 1 (the
    batch axis) is a batch map iff its inner function is one along axis 0 (``scan/op.py:1673``:
    the loop hands row t of each buffer to the inner function)."""
    info = n.params["info"]
    inner = n.params["inner"]
    n_seqs = info["n_seqs"]
    taps = list(info["mit_mot_in_slices"]) + list(info["mit_sot_in_slices"]) + list(info["sit_sot_in_slices"])
    if info["mit_mot_in_slices"] or info["n_shared_outs"] or info["n_nit_sot"] or info.get("as_while"):
        _fail(n, "Scan with mit-mot / shared / nit-sot outputs or a while condition")
    if ins[0] != REP:
        _fail(n, "number of steps depends on a local shape")
    pos = 1
    inner_labels = []
    for s in range(n_seqs):
        l = ins[pos + s]
        if l[0] == "rows":
            if l[1] != 1 or l[2] != 0:
                _fail(n, "sequence sharded along an axis other than the batch axis")
            inner_labels.append(("rows", 0, 0))
        elif l == REP:
            inner_labels.append(REP)
        else:
            _fail(n, f"sequence {l}")
    pos += n_seqs
    state_labels = []
    for t, tp in enumerate(taps):
        l = ins[pos + t]
        if l[0] == "rows":
            if l[1] != 1 or l[2] != 0:
                _fail(n, "state sharded along an axis other than the batch axis")
            il = ("rows", 0, 0)
        elif l == REP:
            il = REP
        else:
            _fail(n, f"state {l}")
        state_labels.append(il)
        inner_labels += [il] * len(tp)
    pos += len(taps)
    for l in ins[pos:]:
        if l != REP:
            _fail(n, "sharded non-sequence")
        inner_labels.append(REP)
    sub = analyse(inner, [None if l == REP else l[1] for l in inner_labels], _inner=True)
    outs = []
    for k, (mode, sl) in enumerate(zip(sub.outputs, state_labels)):
        want = ("concat", 0) if sl != REP else ("rep",)
        if mode != want:
            _fail(n, f"inner output {k} is {mode}, its state is {sl}")
        outs.append(("rows", 1, 0) if sl != REP else REP)
    return outs


def infer_sharded_inputs(program, candidates=None):
    """Largest set of function inputs (by default: every tensor input with at least one
    dimension that no ``updates=`` writes) that can be split along axis 0 so that the graph is
    a batch map; among equally large sets the one with the earlier inputs.  Weights drop out
    because they meet the batch on the K axis of a product; a data input cannot be left out
    because a replicated operand must broadcast along the sharded axis."""
    if candidates is None:
        updated = {i for _, i in program.updates}
        candidates = [k for k, v in enumerate(program.inputs)
                      if program.vars[v].kind == "tensor" and program.vars[v].ndim >= 1 and k not in updated]
    def attempt(cand):
        spec = [0 if k in cand else None for k in range(len(program.inputs))]
        plan = analyse(program, spec)
        if all(o[0] == "rep" for o in plan.outputs):
            raise ReplicasOnly("replicas only: no output depends on a sharded input")
        return plan

    import itertools

    cand = list(candidates)
    if len(cand) > 12:
        raise ReplicasOnly("replicas only: too many candidate inputs to infer; pass shard_inputs explicitly")
    last = None
    for size in range(len(cand), 0, -1):
        for sub in itertools.combinations(cand, size):
            try:
                return attempt(sub)
            except ReplicasOnly as e:
                last = last or e
    raise last or ReplicasOnly("replicas only: no tensor input to shard")
