"""GPU: the fused Elemwise kernels at every launch flavour, and every device scalar op.

``ab_elemwise_launch`` squeezes, orders and merges the dims of one Elemwise call and picks one
of six kernels (``flat_vec``, ``flat``, ``rows_vec``, ``rows``, ``tile``, ``nd``).  Part A
lands on each side of those decisions on purpose, and ``ab_elemwise_path_count`` confirms the
flavour the case id names.  Operands make every output exact (integers or integer-valued
floats), so a wrong index, tail or tile fails by equality, and every output is written into
the middle of a buffer filled with a sentinel that must survive outside the view.

Part B checks the scalar op table (``codegen/scalar_cuda.py`` over ``csrc/ab_types.cuh``)
that every fused Elemwise, CAReduce pre-map, row region and GEMM epilogue shares: integer ops
exactly against C's promotions and conversions restated on Python integers; the correctly
rounded float ops bit for bit against NumPy in the same dtype (so ``-ftz``, fast math or
approximate division would fail); the transcendental ops in ulps against float64
NumPy / SciPy (float32 results) and 100-bit mpmath (float64 results).  Part C runs the same
bodies as a CAReduce pre-map and behind ``copy_into`` / ``add_into``.  Part D checks that the
host evaluator of small operands and the device give one answer.
"""
import itertools
import math
import os
import zlib

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

FLAVOURS = ["flat_vec", "flat", "rows_vec", "rows", "nd", "tile"]  # Module::EW_* order
REACHED = set()

INTS = ["int8", "int16", "int32", "int64", "uint8", "uint16", "uint32", "uint64"]
DISCRETE = ["bool"] + INTS
FLOATS = ["float32", "float64"]


@pytest.fixture(scope="module")
def L():
    import torch

    from aesara_b200.runtime import lib

    lib.check(lib.load().ab_init(0))
    torch.cuda.set_device(0)
    return lib.load()


def _kernel(expr):
    from aesara_b200.runtime.kernels import ElemwiseKernel

    return ElemwiseKernel.get(expr)


def _st(op, args, dtype, in_dtypes, **kw):
    return dict(op=op, args=list(args), dtype=dtype, in_dtypes=list(in_dtypes), **kw)


def _sum_expr(in_dts, out_dt):
    """o0 = i0 + i1 + ... (C addition; exact on the small integers used here)."""
    args = [f"i{k}" for k in range(len(in_dts))]
    if len(args) == 1:
        stmts = [_st("identity", args, out_dt, in_dts)]
    else:
        stmts = [_st("add", args, out_dt, in_dts)]
    return {"inputs": list(in_dts), "out_dtypes": [out_dt], "outputs": ["t0"], "stmts": stmts,
            "name": "sum_" + "_".join(in_dts)}


def _counts(L):
    return [L.ab_elemwise_path_count(k) for k in range(len(FLAVOURS))]


def _launch(L, expr, shape, ins, outs):
    """Launch once; return the flavour that ran (None if nothing launched)."""
    from aesara_b200.runtime.device import DeviceArray  # noqa: F401

    before = _counts(L)
    _kernel(expr).launch(tuple(shape), ins, outs)
    diff = [a - b for a, b in zip(_counts(L), before)]
    assert sum(diff) <= 1, diff
    if sum(diff) == 0:
        return None
    ran = FLAVOURS[diff.index(1)]
    REACHED.add(ran)
    return ran


# ------------------------------------------------------------------------------------------
# strided placement with sentinels
# ------------------------------------------------------------------------------------------
def _sentinel(dt):
    dt = np.dtype(dt)
    if dt.kind == "f":
        return dt.type(-12345.0)
    if dt.kind == "b":
        return True
    return np.iinfo(dt).max if dt.kind == "u" else dt.type(-77)


class Placed:
    """A logical array stored at element strides ``strides`` inside a sentinel-filled buffer
    (``misalign`` extra elements in front shift it off 16-byte alignment)."""

    def __init__(self, a, strides=None, misalign=0, pad=32):
        from aesara_b200.runtime.device import DeviceArray, c_strides

        a = np.asarray(a)
        self.dtype = a.dtype
        self.shape = a.shape
        strides = tuple(c_strides(a.shape) if strides is None else strides)
        neg = sum((n - 1) * -s for n, s in zip(a.shape, strides) if s < 0 and n > 0)
        pos = sum((n - 1) * s for n, s in zip(a.shape, strides) if s > 0 and n > 0)
        self.offset = pad + misalign + neg
        size = self.offset + pos + 1 + pad
        idx = np.full(a.shape, self.offset, dtype=np.int64)
        for d, s in enumerate(strides):
            sh = [1] * a.ndim
            sh[d] = a.shape[d]
            idx = idx + (np.arange(a.shape[d]) * s).reshape(sh)
        self.idx = idx
        buf = np.full(size, _sentinel(a.dtype), dtype=a.dtype)
        buf[idx] = a
        self.host = buf
        self.base = DeviceArray.from_numpy(buf)
        self.view = self.base.view(a.shape, strides, self.offset)

    def result(self):
        """(values in the view, True if every element outside it still holds the sentinel)."""
        buf = self.base.to_numpy()
        mask = np.ones(buf.shape, bool)
        mask[self.idx.reshape(-1)] = False
        outside = buf[mask]
        same = np.array_equal(outside.view(np.uint8), self.host[mask].view(np.uint8))
        return buf[self.idx], same


def _t_strides(shape):
    """Strides of the transpose of the last two dims of a C-contiguous buffer (a column-major
    view: unit stride along rows)."""
    from aesara_b200.runtime.device import c_strides

    sw = list(shape)
    sw[-1], sw[-2] = sw[-2], sw[-1]
    st = list(c_strides(sw))
    st[-1], st[-2] = st[-2], st[-1]
    return tuple(st)


def _ints(shape, dt, rng, lo=-20, hi=21):
    dt = np.dtype(dt)
    if dt.kind == "u":
        lo = 0
    if dt.kind == "b":
        return rng.random(shape) < 0.5
    return rng.integers(lo, hi, shape).astype(dt)


def _run_case(L, in_specs, out_dt, shape, out_strides=None, out_misalign=0, env=None):
    """in_specs: list of (logical array, strides or None, misalign).  Returns (flavour, got,
    want, sentinel intact)."""
    ins = [Placed(a, st, mis) for a, st, mis in in_specs]
    want = np.zeros(shape, np.int64 if np.dtype(out_dt).kind != "f" else np.float64)
    for a, _, _ in in_specs:
        want = want + a.astype(want.dtype)
    want = want.astype(out_dt)
    out = Placed(np.zeros(shape, out_dt), out_strides, out_misalign)
    expr = _sum_expr([str(p.dtype) for p in ins], out_dt)
    old = {}
    for k, v in (env or {}).items():
        old[k] = os.environ.get(k)
        os.environ[k] = v
    try:
        ran = _launch(L, expr, shape, [p.view for p in ins], [out.view])
    finally:
        for k, v in old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v
    got, intact = out.result()
    return ran, got, want, intact


def _sms():
    import torch

    return torch.cuda.get_device_properties(0).multi_processor_count


def _case(name, rng):
    """-> (flavour, in_specs, out dtype, shape, out strides, extra)."""
    i32 = "int32"
    flavour, _, rest = name.partition("-")
    if flavour == "flat_vec":
        if rest.startswith("tail"):  # int32 and int8: n % VEC = t
            dt, t = rest[4:].split("_")
            v = 16 // np.dtype(dt).itemsize
            n = 5 * v + int(t)
            return [(_ints(n, dt, rng), None, 0), (_ints(n, dt, rng), None, 0)], dt, (n,), None, {}
        if rest == "mixed_int8_f64":  # VEC = 16 / 8 = 2, odd n
            n = 1001
            return [(_ints(n, "int8", rng), None, 0),
                    (_ints(n, "float64", rng), None, 0)], "float64", (n,), None, {}
        if rest == "bcast_scalar":
            n = 4099
            return [(_ints(n, i32, rng), None, 0), (_ints(1, i32, rng), None, 0)], i32, (n,), None, {}
        if rest == "beyond_grid":  # more vectors than 32 x SMs blocks of 256 threads cover
            n = 32 * _sms() * 256 * 4 * 3 + 3
            return [(_ints(n, i32, rng), None, 0), (_ints(n, i32, rng), None, 0)], i32, (n,), None, {}
        if rest == "fortran_out":  # F-contiguous inputs: F-order output, one merged run
            a = np.asfortranarray(_ints((37, 41), i32, rng))
            return [(a, (1, 37), 0), (a * 2, (1, 37), 0)], i32, (37, 41), (1, 37), {}
    if flavour == "flat":
        if rest == "misaligned":
            n = 1003
            return [(_ints(n, i32, rng), None, 1), (_ints(n, i32, rng), None, 0)], i32, (n,), None, {}
        if rest == "below_vec":
            return [(_ints(3, i32, rng), None, 0), (_ints(3, i32, rng), None, 0)], i32, (3,), None, {}
        if rest == "single":
            return [(_ints(1, i32, rng), None, 0), (_ints(1, i32, rng), None, 0)], i32, (1,), None, {}
        if rest == "zero_d":
            return [(_ints((), i32, rng), (), 0), (_ints((), i32, rng), (), 0)], i32, (), (), {}
        if rest == "all_ones":
            s = (1, 1, 1)
            return [(_ints(s, i32, rng), None, 0), (_ints(s, i32, rng), None, 0)], i32, s, None, {}
    if flavour in ("rows_vec", "rows"):
        R, C = 37, 64
        if rest == "bcast_1C":
            return [(_ints((R, C), i32, rng), None, 0), (_ints((1, C), i32, rng), None, 0)], i32, (R, C), None, {}
        if rest == "bcast_R1":
            return [(_ints((R, C), i32, rng), None, 0), (_ints((R, 1), i32, rng), None, 0)], i32, (R, C), None, {}
        if rest == "colslice_pitch_odd":  # row stride C + 3: not a multiple of VEC
            return [(_ints((R, C), i32, rng), (C + 3, 1), 0), (_ints((R, C), i32, rng), None, 0)], \
                i32, (R, C), None, {}
        if rest == "cols_mod_vec":
            return [(_ints((R, 63), i32, rng), None, 0), (_ints((1, 63), i32, rng), None, 0)], \
                i32, (R, 63), None, {}
        if rest == "neg_rowstride":
            return [(_ints((R, C), i32, rng), (-C, 1), 0), (_ints((1, C), i32, rng), None, 0)], \
                i32, (R, C), None, {}
        if rest == "many_rows":  # more rows than 65535 x unroll (grid.y clamp)
            R = 65535 * (1 if flavour == "rows_vec" else 4) + 7
            C = 4 if flavour == "rows_vec" else 3
            return [(_ints((R, C), i32, rng), None, 0), (_ints((1, C), i32, rng), None, 0)], \
                i32, (R, C), None, {}
        if rest == "strided_out":  # output row pitch C + 8 (a column slice of a wider matrix)
            return [(_ints((R, C), i32, rng), None, 0), (_ints((1, C), i32, rng), None, 0)], \
                i32, (R, C), (C + 8, 1), {}
    if flavour == "tile":
        if rest.startswith("2d_"):
            R, C = map(int, rest[3:].split("x"))
            a = _ints((R, C), i32, rng)
            return [(a, None, 0), (_ints((R, C), i32, rng), _t_strides((R, C)), 0)], i32, (R, C), None, {}
        if rest == "3d":
            s = (3, 65, 70)
            return [(_ints(s, i32, rng), None, 0), (_ints(s, i32, rng), _t_strides(s), 0)], i32, s, None, {}
        if rest.startswith("slots_"):  # staged inputs of one width: 1, several, the maximum
            dt, k = rest[6:].split("_")
            k = int(k)
            s = (70, 66)
            specs = [(_ints(s, dt, rng, 0, 5), _t_strides(s), 0) for _ in range(k)]
            specs.append((_ints(s, dt, rng, 0, 5), None, 0))
            return specs, dt, s, None, {}
        if rest == "bcast_rows_colstride2":  # [1, C] read at column stride 2: staged
            R, C = 40, 50
            return [(_ints((R, C), i32, rng), None, 0), (_ints((1, C), i32, rng), (0, 2), 0)], \
                i32, (R, C), None, {}
        if rest == "bcast_batch":
            s = (4, 33, 70)
            return [(_ints(s, i32, rng), None, 0), (_ints((1,) + s[1:], i32, rng), _t_strides((1,) + s[1:]), 0)], \
                i32, s, None, {}
    if flavour == "nd":
        if rest.startswith("slots_over_"):
            dt = rest[11:]
            k = {"int8": 11, "int16": 5, "int32": 2, "int64": 1}[dt] + 1
            s = (70, 66)
            return [(_ints(s, dt, rng, 0, 5), _t_strides(s), 0) for _ in range(k)], dt, s, None, {}
        if rest == "15x15":
            s = (15, 15)
            return [(_ints(s, i32, rng), None, 0), (_ints(s, i32, rng), _t_strides(s), 0)], i32, s, None, {}
        if rest == "no_tile_env":
            s = (65, 70)
            return [(_ints(s, i32, rng), None, 0), (_ints(s, i32, rng), _t_strides(s), 0)], i32, s, None, \
                {"AB_EW_NO_TILE": "1"}
        if rest == "neg_inner":
            s = (33, 40)
            return [(_ints(s, i32, rng), (40, -1), 0), (_ints(s, i32, rng), None, 0)], i32, s, None, {}
        if rest == "bcast_middle":
            s = (5, 17, 33)
            return [(_ints(s, i32, rng), None, 0), (_ints((5, 1, 33), i32, rng), None, 0)], i32, s, None, {}
        if rest == "eight_dims":  # an F-order input against a C-order output: nothing merges
            s = (2, 3, 2, 3, 2, 3, 2, 3)
            from aesara_b200.runtime.device import f_strides

            return [(_ints(s, i32, rng), f_strides(s), 0), (_ints(s, i32, rng), None, 0)], i32, s, None, {}
        if rest == "strided_out":  # output at column stride 2
            s = (20, 30)
            return [(_ints(s, i32, rng), None, 0), (_ints(s, i32, rng), None, 0)], i32, s, (60, 2), {}
    raise KeyError(name)


GEOMETRY_CASES = (
    [f"flat_vec-tail{dt}_{t}" for dt, ts in (("int32", (1, 2, 3)), ("int8", (1, 7, 15))) for t in ts]
    + ["flat_vec-mixed_int8_f64", "flat_vec-bcast_scalar", "flat_vec-beyond_grid", "flat_vec-fortran_out",
       "flat-misaligned", "flat-below_vec", "flat-single", "flat-zero_d", "flat-all_ones",
       "rows_vec-bcast_1C", "rows_vec-bcast_R1", "rows_vec-neg_rowstride", "rows_vec-many_rows",
       "rows_vec-strided_out",
       "rows-colslice_pitch_odd", "rows-cols_mod_vec", "rows-many_rows"]
    + [f"tile-2d_{r}x{c}" for r, c in ((16, 16), (63, 65), (64, 64), (65, 1000), (1000, 63))]
    + ["tile-3d", "tile-bcast_rows_colstride2", "tile-bcast_batch"]
    + [f"tile-slots_{dt}_{k}" for dt, ks in (("int8", (1, 4, 11)), ("int16", (1, 3, 5)),
                                             ("int32", (1, 2)), ("int64", (1,))) for k in ks]
    + [f"nd-slots_over_{dt}" for dt in ("int8", "int16", "int32", "int64")]
    + ["nd-15x15", "nd-no_tile_env", "nd-neg_inner", "nd-bcast_middle", "nd-eight_dims",
       "nd-strided_out"]
)


@pytest.mark.parametrize("name", GEOMETRY_CASES)
def test_launch_geometry(L, name):
    rng = np.random.default_rng(zlib.crc32(name.encode()))
    specs, out_dt, shape, out_st, env = _case(name, rng)
    ran, got, want, intact = _run_case(L, specs, out_dt, shape, out_st, env=env)
    assert ran == name.split("-")[0], f"{name}: ran {ran}"
    np.testing.assert_array_equal(got, want, err_msg=name)
    assert intact, f"{name}: wrote outside the output view"


def test_fortran_output_order_is_chosen_for_f_inputs(L):
    """elemwise_out_order picks F for F- but not C-contiguous inputs, and the F output keeps the
    call on the 128-bit flat kernel."""
    from aesara_b200.runtime.device import DeviceArray
    from aesara_b200.runtime.kernels import elemwise_out_order

    a = np.asfortranarray(np.arange(37 * 41, dtype=np.int32).reshape(37, 41))
    A = DeviceArray.from_numpy(np.ascontiguousarray(a.T)).view(a.shape, (1, 37))
    assert elemwise_out_order([A, A], a.shape) == "F"
    out = DeviceArray.empty(a.shape, "int32", order="F")
    assert _launch(L, _sum_expr(["int32", "int32"], "int32"), a.shape, [A, A], [out]) == "flat_vec"
    np.testing.assert_array_equal(out.to_numpy(), 2 * a)


@pytest.mark.parametrize("flavour", ["flat_vec", "rows_vec", "nd"])
def test_in_place_output(L, flavour):
    """An output that is input 0 (destroy_map): every element read before it is written."""
    rng = np.random.default_rng(11)
    if flavour == "flat_vec":
        shape, st0, st1 = (4099,), None, None
    elif flavour == "rows_vec":
        shape, st0, st1 = (37, 64), (72, 1), None
    else:
        shape, st0, st1 = (15, 15), None, _t_strides((15, 15))
    a, b = _ints(shape, "int32", rng), _ints(shape, "int32", rng)
    A, B = Placed(a, st0), Placed(b, st1)
    ran = _launch(L, _sum_expr(["int32", "int32"], "int32"), shape, [A.view, B.view], [A.view])
    assert ran == flavour
    got, intact = A.result()
    np.testing.assert_array_equal(got, a + b)
    assert intact


def test_nine_unmergeable_dims_raise(L):
    from aesara_b200.runtime import lib
    from aesara_b200.runtime.device import f_strides

    s = (2,) * 9
    rng = np.random.default_rng(1)
    x = Placed(_ints(s, "int32", rng), f_strides(s))
    out = Placed(np.zeros(s, np.int32))
    before = _counts(L)
    with pytest.raises(lib.AbError, match="non-mergeable"):
        _kernel(_sum_expr(["int32"], "int32")).launch(s, [x.view], [out.view])
    assert _counts(L) == before
    assert out.result()[1] and not out.result()[0].any()


def test_zero_size_launches_nothing(L):
    x = Placed(np.zeros((5, 0, 3), np.int32))
    out = Placed(np.zeros((5, 0, 3), np.int32))
    assert _launch(L, _sum_expr(["int32"], "int32"), (5, 0, 3), [x.view], [out.view]) is None
    assert out.result()[1]


# ------------------------------------------------------------------------------------------
# B. the scalar op table
# ------------------------------------------------------------------------------------------
def _run_expr(L, expr, arrays):
    """Evaluate ``expr`` on 1-D operands of equal length through the flat kernel."""
    from aesara_b200.runtime.device import DeviceArray

    n = len(arrays[0])
    ins = [DeviceArray.from_numpy(np.ascontiguousarray(a)) for a in arrays]
    outs = [DeviceArray.empty((n,), dt) for dt in expr["out_dtypes"]]
    assert _launch(L, expr, (n,), ins, outs) in ("flat_vec", "flat")
    return [o.to_numpy() for o in outs]


def _multi(ops, in_dts, out_dts, extra=None):
    """One body with one statement (and one output) per op, all on the same inputs."""
    stmts, outs = [], []
    for k, (op, dt) in enumerate(zip(ops, out_dts)):
        args = ["i0", "i1", "i2"][: len(in_dts)]
        stmts.append(_st(op, args, dt, in_dts, **((extra or {}).get(op, {}))))
        outs.append(f"t{k}")
    return {"inputs": list(in_dts), "out_dtypes": list(out_dts), "outputs": outs, "stmts": stmts,
            "name": "table_" + "_".join(in_dts)}


# -- C semantics on Python integers (the ab_types.cuh typedefs) -----------------------------
def _bits(dt):
    dt = np.dtype(dt)
    return 8 * dt.itemsize, dt.kind == "i"


def _wrap(v, dt):
    """Conversion of an integer value to ``dt`` (modular, as nvcc does)."""
    dt = np.dtype(dt)
    if dt.kind == "b":
        return v & 0xFF  # ab_bool is unsigned char: a plain conversion, not != 0
    if dt.kind == "f":
        return float(v) if dt == np.float64 else float(np.float32(float(v)))
    n, signed = _bits(dt)
    v &= (1 << n) - 1
    return v - (1 << n) if signed and v >> (n - 1) else v


def _promote(dt):
    """Integer promotion: bool, 8- and 16-bit types become int."""
    return "int32" if dt in ("bool", "int8", "int16", "uint8", "uint16") else dt


def _c_common(a, b):
    a, b = _promote(a), _promote(b)
    if a == b:
        return a
    (na, sa), (nb, sb) = _bits(a), _bits(b)
    if sa == sb:
        return a if na > nb else b
    s, u = (a, b) if sa else (b, a)
    return u if _bits(u)[0] >= _bits(s)[0] else s


def _np_upcast(a, b):
    return np.result_type(np.dtype(a), np.dtype(b)).name


def _floordiv(x, y):
    return 0 if y == 0 else x // y  # Python // is floor division


def _pymod(x, y):
    return 0 if y == 0 else x % y  # Python % has the sign of y


def _int_truth(op, x, y, dx, dy):
    """Value of the device body for discrete operands (Python ints), before the conversion to
    the statement's dtype."""
    if op in ("add", "sub", "mul", "and", "or", "xor"):
        t = _c_common(dx, dy)
        a, b = _wrap(x, t), _wrap(y, t)
        r = {"add": a + b, "sub": a - b, "mul": a * b, "and": a & b, "or": a | b, "xor": a ^ b}[op]
        return _wrap(r, t)
    if op in ("lt", "gt", "le", "ge", "eq", "neq"):
        t = _c_common(dx, dy)
        a, b = _wrap(x, t), _wrap(y, t)
        return int({"lt": a < b, "gt": a > b, "le": a <= b, "ge": a >= b, "eq": a == b, "neq": a != b}[op])
    t = _np_upcast(dx, dy)  # int_div / mod / maximum / minimum cast both to the NumPy upcast
    a, b = _wrap(x, t), _wrap(y, t)
    if op == "int_div":
        return _wrap(_floordiv(a, b), t)
    if op == "mod":
        return _wrap(_pymod(a, b), t)
    if op == "maximum":
        return max(a, b)
    if op == "minimum":
        return min(a, b)
    raise KeyError(op)


def _extremes(dt):
    if dt == "bool":
        return [0, 1]
    i = np.iinfo(dt)
    vals = {int(i.min), int(i.min) + 1, -1, 0, 1, 2, 3, -3, 7, -7, int(i.max) - 1, int(i.max)}
    return sorted(v for v in vals if i.min <= v <= i.max)


_BINARY_INT_OPS = ["add", "sub", "mul", "int_div", "mod", "and", "or", "xor", "lt", "gt", "le",
                   "ge", "eq", "neq", "maximum", "minimum"]


def _out_dtype(op, dx, dy):
    if op in ("lt", "gt", "le", "ge", "eq", "neq"):
        return "bool"
    t = _np_upcast(dx, dy)
    if op in ("add", "mul") and t == "bool":
        return "bool"
    return t


@pytest.mark.parametrize("dx", DISCRETE)
def test_integer_binary_ops_at_every_dtype_pair(L, dx):
    """Every binary op on every pair of discrete dtypes, at MIN, MIN+1, -1, 0, 1, MAX-1, MAX (and
    a few small values) of each: all four sign combinations of floor division and modulo, the
    divisor 0 (the device's documented 0), MIN // -1 and MIN % -1, mixed signedness (int32 with
    uint32 compares as uint32), and the wrap of every C conversion."""
    for dy in DISCRETE:
        ops = [op for op in _BINARY_INT_OPS
               if not (op == "sub" and "bool" in (dx, dy))
               and not (op in ("int_div", "mod") and (dx == dy == "bool"
                                                       or _np_upcast(dx, dy) == "float64"))]
        outs = [_out_dtype(op, dx, dy) for op in ops]
        pairs = list(itertools.product(_extremes(dx), _extremes(dy)))
        x = np.array([p[0] for p in pairs], dtype=dx)
        y = np.array([p[1] for p in pairs], dtype=dy)
        got = _run_expr(L, _multi(ops, [dx, dy], outs), [x, y])
        for op, odt, g in zip(ops, outs, got):
            if op in ("add", "mul") and odt == "bool":
                want = [int((a or b) if op == "add" else (a and b)) for a, b in pairs]
            else:
                want = [_wrap(_int_truth(op, a, b, dx, dy), odt) if odt != "bool"
                        else _int_truth(op, a, b, dx, dy) for a, b in pairs]
            want = np.array(want, dtype=object)
            gv = np.array([int(v) if odt != "float64" and odt != "float32" else float(v) for v in g], dtype=object)
            bad = [(pairs[i], gv[i], want[i]) for i in range(len(pairs)) if gv[i] != want[i]]
            assert not bad, f"{op}({dx}, {dy}) -> {odt}: (x, y), got, want: {bad[:6]}"


@pytest.mark.parametrize("dt", DISCRETE)
def test_integer_unary_ops_and_casts(L, dt):
    """abs / neg of MIN (wraps), invert on bool (logical not), unsigned and signed, sgn, sqr and
    every int-to-int cast (modular)."""
    vals = _extremes(dt)
    x = np.array(vals, dtype=dt)
    ops, outs = [], []
    if dt != "bool":
        ops += ["abs", "neg", "sgn", "sqr"]
        outs += [dt] * 4
    ops.append("invert")
    outs.append(dt)
    ops += ["cast"] * len(DISCRETE)
    outs += DISCRETE
    got = _run_expr(L, _multi(ops, [dt], outs), [x])
    for op, odt, g in zip(ops, outs, got):
        want = []
        for v in vals:
            if op == "abs":
                w = _wrap(abs(v), dt)
            elif op == "neg":
                w = _wrap(-v, dt)
            elif op == "sgn":
                w = (v > 0) - (v < 0)
            elif op == "sqr":
                w = _wrap(v * v, dt)
            elif op == "invert":
                w = int(not v) if dt == "bool" else _wrap(~v, dt)
            else:
                w = int(v != 0) if odt == "bool" else _wrap(v, odt)
            want.append(w)
        assert [int(a) for a in g] == want, f"{op}({dt}) -> {odt}"


@pytest.mark.parametrize("fdt", FLOATS)
def test_float_to_int_and_bool_casts(L, fdt):
    """In-range float-to-int casts truncate toward zero, including +-(n + 0.5) and the values
    just inside each bound; float-to-bool of NaN is 1 and of -0 is 0."""
    for idt in INTS:
        info = np.iinfo(idt)
        f = np.dtype(fdt).type
        lo = f(info.min)  # 0 or -2**(n-1): exact
        hi = f(info.max)
        while float(hi) > info.max:
            hi = np.nextafter(hi, f(0))
        base = [0.0, -0.0, 0.5, -0.5, 1.5, -1.5, 2.5, -2.5, 7.999, -7.999, 100.5, -100.5]
        vals = np.array([v for v in base if info.min <= v <= info.max] + [lo, hi,
                        np.nextafter(hi, f(0)), np.nextafter(lo, f(0))], dtype=fdt)
        if info.min == 0:
            vals = vals[vals >= 0]
        got = _run_expr(L, _multi(["cast"], [fdt], [idt]), [vals])[0]
        want = np.array([int(math.trunc(float(v))) for v in vals], dtype=object)
        assert [int(v) for v in got] == list(want), f"cast {fdt} -> {idt}: {vals}"
    vals = np.array([np.nan, -0.0, 0.0, 1e-45 if fdt == "float32" else 5e-324, -np.inf], dtype=fdt)
    got = _run_expr(L, _multi(["cast"], [fdt], ["bool"]), [vals])[0]
    np.testing.assert_array_equal(got, [True, False, False, True, True])


def _float_grid(dt, rng, n=4096):
    """Random bit patterns over the whole range, plus zeros, infinities, NaN, subnormals, the
    largest finite values and small integers and halves."""
    dt = np.dtype(dt)
    ut = np.uint32 if dt == np.float32 else np.uint64
    bits = rng.integers(0, np.iinfo(ut).max, n, dtype=ut, endpoint=True)
    x = bits.view(dt)
    fi = np.finfo(dt)
    special = [0.0, -0.0, np.inf, -np.inf, np.nan, fi.tiny, -fi.tiny, fi.smallest_subnormal,
               -fi.smallest_subnormal, fi.tiny / 3, fi.max, -fi.max, 1.0, -1.0, 0.5, -0.5, 1.5,
               -1.5, 2.5, -2.5, 3.0, -3.0, 1e-3, 1e10, -1e10, 4503599627370497.0]
    sub = (rng.integers(1, 1 << 20, 64).astype(ut)).view(dt)  # subnormals
    return np.concatenate([np.array(special, dt), sub, -sub, x])


def _same_bits(a, b):
    """Equal bit patterns, or both NaN."""
    a, b = np.asarray(a), np.asarray(b)
    ut = np.uint32 if a.dtype == np.float32 else np.uint64
    return (a.view(ut) == b.view(ut)) | (np.isnan(a) & np.isnan(b))


@pytest.mark.parametrize("dt", FLOATS)
def test_correctly_rounded_float_ops_bit_exact(L, dt):
    """+ - * / sqrt floor ceil trunc rint round fabs maximum minimum sgn are correctly rounded
    (or exact): bit-for-bit NumPy in the same dtype, subnormal inputs and results included."""
    from oracle.scalar_np import apply_op

    rng = np.random.default_rng(zlib.crc32(dt.encode()))
    x = _float_grid(dt, rng)
    y = np.concatenate([_float_grid(dt, rng, 0)[::-1], rng.permutation(x[26:])])[: len(x)]
    y[:8] = [np.nan, 1.0, np.nan, -0.0, 3.0, np.inf, -np.inf, 2.0]  # NaN in the second slot
    binary = ["add", "sub", "mul", "true_divide", "maximum", "minimum"]
    got = _run_expr(L, _multi(binary, [dt, dt], [dt] * len(binary)), [x, y])
    with np.errstate(all="ignore"):
        want = [x + y, x - y, x * y, x / y, np.maximum(x, y), np.minimum(x, y)]
    for op, g, w in zip(binary, got, want):
        if op in ("maximum", "minimum"):  # +-0 order is not part of the contract
            ok = _same_bits(g, w) | ((g == 0) & (w == 0))
        else:
            ok = _same_bits(g, w)
        assert ok.all(), f"{op} {dt}: x={x[~ok][:4]} y={y[~ok][:4]} got={g[~ok][:4]} want={w[~ok][:4]}"
    unary = ["sqrt", "floor", "ceil", "trunc", "round_half_to_even", "round_half_away_from_zero",
             "abs", "sgn", "neg"]
    got = _run_expr(L, _multi(unary, [dt], [dt] * len(unary)), [x])
    for op, g in zip(unary, got):
        w = apply_op(_st(op, ["i0"], dt, [dt]), [x])
        if op == "round_half_away_from_zero":  # C round(): halfway cases away from zero
            with np.errstate(all="ignore"):
                t = np.floor(np.abs(x))
                w = np.copysign(t + (np.abs(x) - t >= 0.5), x).astype(dt)
        ok = _same_bits(g, w)
        assert ok.all(), f"{op} {dt}: x={x[~ok][:4]} got={g[~ok][:4]} want={w[~ok][:4]}"


@pytest.mark.parametrize("dt", FLOATS)
def test_float_int_div_and_mod(L, dt):
    """Float IntDiv and Mod follow the reference's C (basic.py:2083-2121, :2207-2236) as restated
    in float64 by the oracle: infinite divisors, +-0, and quotients that round up to an integer."""
    from oracle.scalar_np import apply_op

    rng = np.random.default_rng(5)
    x = _float_grid(dt, rng, 2048)
    y = rng.permutation(x)
    f = np.dtype(dt).type
    extra_x = np.array([0.5, -0.5, 0.5, -0.5, 1.0, -1.0, 0.0, -0.0, 7.0, -7.0, 1.0, 1.0 - np.finfo(dt).eps / 2,
                        np.inf, 5.0, 5.0, -5.0], dt)
    extra_y = np.array([np.inf, np.inf, -np.inf, -np.inf, 0.0, 0.0, 3.0, -3.0, -0.0, 0.0,
                        f(1.0) / f(3.0), f(1.0) / f(3.0), 2.0, np.nextafter(f(5.0), f(0)),
                        np.nextafter(f(5.0), f(10)), np.nextafter(f(5.0), f(0))], dt)
    x, y = np.concatenate([extra_x, x]), np.concatenate([extra_y, y])
    got = _run_expr(L, _multi(["int_div", "mod"], [dt, dt], [dt, dt]), [x, y])
    for op, g in zip(["int_div", "mod"], got):
        w = apply_op(_st(op, ["i0", "i1"], dt, [dt, dt]), [x, y])
        ok = _same_bits(g, w)
        assert ok.all(), f"{op} {dt}: x={x[~ok][:4]} y={y[~ok][:4]} got={g[~ok][:4]} want={w[~ok][:4]}"


# -- transcendental ops in ulps -------------------------------------------------------------
# Maximum ulp errors documented in the CUDA 12.9 Math API ("CUDA C++ Programming Guide",
# Mathematical Functions appendix, tables "Single-Precision Mathematical Standard Library
# Functions with Maximum ULP Error" and the double-precision table), for full-range arguments
# with the default -prec-div / -prec-sqrt and no -ftz.
CUDA_ULP = {
    "exp": (2, 1), "exp2": (2, 1), "expm1": (1, 1), "log": (1, 1), "log2": (1, 1),
    "log10": (2, 1), "log1p": (1, 1), "sin": (2, 2), "cos": (2, 2), "tan": (4, 2),
    "arcsin": (2, 2), "arccos": (2, 2), "arctan": (2, 2), "sinh": (3, 2), "cosh": (2, 1),
    "tanh": (2, 1), "arcsinh": (3, 3), "arccosh": (4, 3), "arctanh": (3, 2), "erf": (2, 2),
    "erfc": (4, 5), "erfinv": (2, 5), "erfcinv": (4, 6), "erfcx": (4, 4), "gamma": (5, 10),
    "gammaln": (6, 4), "arctan2": (3, 2), "pow": (4, 2),
}
# The project's own helpers (ab_types.cuh), bounded by the error analysis of their formulas in
# units of the result's ulp: sigmoid = 1 / (1 + e), e = exp(-x): the relative error of e is
# damped by e / (1 + e) <= 1, then one rounding each for the sum and the quotient.  softplus =
# max(x, 0) + log1p(e): log1p(e) has the errors of exp (damped) and log1p, then one addition.
# log1mexp: log1p(-exp(x)) or log(-expm1(x)) amplify the argument's relative error by at most
# 1 / ln 2 at the switch point -ln 2, plus the outer function's error and one rounding.
HELPER_ULP = {"sigmoid": (3.5, 2.5), "softplus": (3.5, 2.5), "log1mexp": (5.0, 3.5)}

_DOMAIN = {  # sample range of each op (before the random bit patterns are clipped into it)
    "arcsin": (-1, 1), "arccos": (-1, 1), "arctanh": (-1, 1), "erfinv": (-1, 1),
    "erfcinv": (0, 2), "arccosh": (1, None), "log1mexp": (None, 0),
    "log": (0, None), "log2": (0, None), "log10": (0, None), "log1p": (-1, None),
}


def _ref32(op, x):
    import scipy.special as sp

    d = x.astype(np.float64)
    with np.errstate(all="ignore"):
        f = {"gamma": sp.gamma, "gammaln": sp.gammaln, "erf": sp.erf, "erfc": sp.erfc,
             "erfinv": sp.erfinv, "erfcinv": sp.erfcinv, "erfcx": sp.erfcx,
             "sigmoid": lambda v: 1.0 / (1.0 + np.exp(-v)),
             "softplus": lambda v: np.where(v > 30, v + np.exp(-v), np.log1p(np.exp(v))),
             "log1mexp": lambda v: np.where(v < -0.7, np.log1p(-np.exp(v)), np.log(-np.expm1(v)))}
        return (f[op] if op in f else getattr(np, op))(d)


def _ref64(op, v):
    import mpmath as mp

    x = mp.mpf(float(v))
    try:
        r = {
            "exp": mp.exp, "exp2": lambda t: mp.power(2, t), "expm1": mp.expm1, "log": mp.log,
            "log2": lambda t: mp.log(t, 2), "log10": mp.log10, "log1p": mp.log1p, "sin": mp.sin,
            "cos": mp.cos, "tan": mp.tan, "arcsin": mp.asin, "arccos": mp.acos, "arctan": mp.atan,
            "sinh": mp.sinh, "cosh": mp.cosh, "tanh": mp.tanh, "arcsinh": mp.asinh,
            "arccosh": mp.acosh, "arctanh": mp.atanh, "erf": mp.erf, "erfc": mp.erfc,
            "erfinv": lambda t: mp.erfinv(t),
            # 1 - t exactly (t may be 1e-300): at 100 bits it keeps too few bits of a small t
            "erfcinv": _erfcinv_exact,
            # exp(t^2) erfc(t) loses everything for huge t: the asymptotic series there
            "erfcx": lambda t: mp.exp(t * t) * mp.erfc(t) if t < 1e6 else
            (1 - 1 / (2 * t * t)) / (t * mp.sqrt(mp.pi)), "gamma": mp.gamma,
            "gammaln": lambda t: mp.log(abs(mp.gamma(t))),
            "sigmoid": lambda t: 1 / (1 + mp.exp(-t)), "softplus": lambda t: mp.log1p(mp.exp(t)),
            "log1mexp": lambda t: mp.log1p(-mp.exp(t)) if t < -1 else mp.log(-mp.expm1(t)),
        }[op](x)
        return r
    except (ValueError, ZeroDivisionError, OverflowError):
        return None


def _erfcinv_exact(t):
    import mpmath as mp

    with mp.workprec(1400):
        return +mp.erfinv(mp.mpf(1) - t)


def _ulp_err(got, ref, dt):
    """|got - ref| in ulps of the result type at ref's magnitude (float64 / mpf ref)."""
    fi = np.finfo(dt)
    mag = abs(float(ref))
    if mag == 0:
        return 0.0 if got == 0 else math.inf
    e = max(math.frexp(mag)[1] - 1, fi.minexp)
    ulp = 2.0 ** (e - fi.nmant)
    return abs(float(got) - float(ref)) / ulp if isinstance(ref, float) else float(abs(got - ref) / ulp)


def _points(op, dt, rng, n):
    x = _float_grid(dt, rng, n)
    x = x[np.isfinite(x)]
    lo, hi = _DOMAIN.get(op, (None, None))
    # most random bit patterns are huge or tiny: also sample the interesting decades densely
    dense = (rng.standard_normal(n) * rng.choice([0.1, 1.0, 10.0, 100.0], n)).astype(dt)
    x = np.concatenate([x, dense])
    if lo is not None:
        x = np.where(x < lo, lo + (lo - x) % (1 if hi is None else (hi - lo)), x)
        x = x[x >= lo]
    if hi is not None:
        x = x[x <= hi]
    f = np.dtype(dt).type
    edges = {
        "softplus": [-37.0, 18.0, 33.3, 0.0], "log1mexp": [-0.6931471805599453, -1e-30],
        "sigmoid": [-88.7, -89.0, -709.0, -710.0, -745.0],
        "exp": [88.72, 88.73, -87.3, -103.9, 709.78, -708.4, -745.1],
        "expm1": [88.72, -20.0, 1e-30], "sinh": [89.4, 710.4], "cosh": [89.4, 710.4],
        "gamma": [35.0, 171.6, 0.5, -0.5, 1e-30], "gammaln": [1.0, 2.0, 1e30],
        "erfcx": [-9.0, 26.5, 1e5],
    }.get(op, [])
    near = []
    for e in edges:
        v = f(e)
        near += [v, np.nextafter(v, f(np.inf)), np.nextafter(v, f(-np.inf))]
    x = np.concatenate([np.array(near, dt), x]).astype(dt)
    if op == "gammaln":  # the documented bound holds outside the interval around the poles
        lo_, hi_ = (-10.001, -2.264) if dt == "float32" else (-11.0001, -2.2637)
        x = x[(x < lo_) | (x > hi_)]
    if op in ("gamma", "gammaln"):
        x = x[(x > 0) | (x != np.round(x))]
    if op == "gammaln" and dt == "float64":
        # finding: next to the zeros of lgamma at 1 and 2 the float64 result carries an absolute
        # error of ~1e-32, not 4 ulp of the small result (measured 26 ulp at 1 - 2**-53); the
        # ulp bound is checked outside those neighbourhoods, the absolute error inside them
        # (test_helper_underflow)
        x = x[(np.abs(x - 1) > 0.1) & (np.abs(x - 2) > 0.1)]
    return x


TRANSCENDENTAL = sorted(set(CUDA_ULP) - {"arctan2", "pow"}) + sorted(HELPER_ULP)
ULP_TABLE = []


@pytest.mark.parametrize("dt", FLOATS)
def test_transcendental_ulps(L, dt):
    rng = np.random.default_rng(zlib.crc32(("ulp" + dt).encode()))
    n = 4096 if dt == "float32" else 300
    worst = {}
    pts = {op: _points(op, dt, rng, n) for op in TRANSCENDENTAL}
    # one module per op: every statement a separate body keeps fma contraction out of the way
    for op in TRANSCENDENTAL:
        x = pts[op]
        g = _run_expr(L, _multi([op], [dt], [dt]), [x])[0]
        errs = []
        for xi, gi in zip(x, g):
            if dt == "float32":
                r = float(_ref32(op, np.array([xi]))[0])
                if not math.isfinite(r) or abs(r) > np.finfo(dt).max:
                    continue
                if op in HELPER_ULP and abs(r) < np.finfo(dt).tiny:
                    continue  # underflowing helpers: pinned in test_helper_underflow
                if not math.isfinite(float(gi)):
                    errs.append((math.inf, xi, gi, r))
                    continue
                errs.append((_ulp_err(float(gi), r, dt), xi, gi, r))
            else:
                import mpmath as mp

                mp.mp.prec = 100
                r = _ref64(op, xi)
                if r is None or not mp.isfinite(r) or abs(r) > np.finfo(dt).max:
                    continue
                if op in HELPER_ULP and abs(r) < np.finfo(dt).tiny:
                    continue  # underflowing helpers: pinned in test_helper_underflow
                if not math.isfinite(float(gi)):
                    errs.append((math.inf, xi, gi, float(r)))
                    continue
                errs.append((_ulp_err(mp.mpf(float(gi)), r, dt), xi, gi, float(r)))
        w = max(errs, key=lambda t: t[0])
        k = 0 if dt == "float32" else 1
        bound = (CUDA_ULP.get(op) or HELPER_ULP[op])[k]
        worst[op] = (bound, w)
        ULP_TABLE.append((op, dt, bound, w[0], len(errs)))
    lines = [f"{op:10s} {dt} bound {b:4} measured {w[0]:.3f} at x={w[1]!r} (got {w[2]!r}, ref {w[3]!r})"
             for op, (b, w) in worst.items()]
    print("\n" + "\n".join(lines))
    bad = [ln for (op, (b, w)), ln in zip(worst.items(), lines) if not w[0] <= b + 0.5]
    assert not bad, "\n".join(bad)


@pytest.mark.parametrize("dt", FLOATS)
def test_special_values(L, dt):
    """C99 Annex F values, exactly."""
    inf, nan = np.inf, np.nan
    cases = {
        "exp": [(-inf, 0.0), (inf, inf), (0.0, 1.0), (-0.0, 1.0), (nan, nan)],
        "expm1": [(-inf, -1.0), (-0.0, -0.0), (inf, inf)],
        "log": [(0.0, -inf), (-0.0, -inf), (1.0, 0.0), (-1.0, nan), (inf, inf)],
        "log1p": [(-1.0, -inf), (-0.0, -0.0), (-2.0, nan)],
        "sqrt": [(-0.0, -0.0), (-1.0, nan), (inf, inf)],
        "sin": [(-0.0, -0.0), (inf, nan)], "cos": [(inf, nan), (0.0, 1.0)],
        "tanh": [(inf, 1.0), (-inf, -1.0), (-0.0, -0.0)],
        "arctanh": [(1.0, inf), (-1.0, -inf), (2.0, nan)],
        "arcsin": [(-0.0, -0.0), (1.5, nan)], "arccosh": [(1.0, 0.0), (0.5, nan)],
        "erf": [(inf, 1.0), (-inf, -1.0), (-0.0, -0.0)], "erfc": [(inf, 0.0), (-inf, 2.0)],
        "erfinv": [(1.0, inf), (-1.0, -inf), (0.0, 0.0), (1.5, nan)],
        "erfcinv": [(0.0, inf), (2.0, -inf), (1.0, 0.0)],
        "gammaln": [(0.0, inf), (1.0, 0.0), (2.0, 0.0), (-inf, inf), (-3.0, inf)],
        "gamma": [(0.0, inf), (-0.0, -inf), (inf, inf), (-inf, nan), (-2.0, nan)],
        "sigmoid": [(inf, 1.0), (-inf, 0.0), (nan, nan)],
        "softplus": [(inf, inf), (-inf, 0.0)],
        "log1mexp": [(0.0, -inf), (-inf, -0.0)],
    }
    for op, pairs in cases.items():
        x = np.array([p[0] for p in pairs], dt)
        w = np.array([p[1] for p in pairs], dt)
        g = _run_expr(L, _multi([op], [dt], [dt]), [x])[0]
        ok = _same_bits(g, w)
        assert ok.all(), f"{op} {dt}: x={x[~ok]} got={g[~ok]} want={w[~ok]}"


@pytest.mark.parametrize("dt", FLOATS)
def test_helper_underflow(L, dt):
    """Finding, pinned: ab_sigmoid = 1 / (1 + exp(-x)) returns 0 once exp(-x) overflows
    (x < -88.72 in float32, -709.78 in float64), where the true result is still a subnormal
    (2.2e-39 at x = -89 in float32).  It is the reference's own formula (math.py:1110), so the
    device keeps it; the ulp bound above is checked where the result is a normal number.  And
    lgamma next to its zero at 1 has a small absolute error."""
    x = np.array([-89.0, -100.0, -745.0] if dt == "float32" else [-710.0, -745.0, -800.0], dt)
    g = _run_expr(L, _multi(["sigmoid"], [dt], [dt]), [x])[0]
    np.testing.assert_array_equal(g, np.zeros(3, dt))
    x = np.array([1 - 2.0 ** -52, 1 + 2.0 ** -52, 2 - 2.0 ** -51, 1.0005, 1.9995], "float64")
    if dt == "float64":
        import mpmath as mp

        g = _run_expr(L, _multi(["gammaln"], [dt], [dt]), [x])[0]
        with mp.workprec(200):
            ref = [float(mp.log(mp.gamma(mp.mpf(float(v))))) for v in x]
        assert np.all(np.abs(g - np.array(ref)) <= 1e-31 + 4 * np.spacing(np.abs(ref))), (g, ref)


def test_trunc_of_integers(L):
    """trunc(int32) is float64 (the reference's upgrade_to_float_no_complex) and of INT32_MIN
    is -2**31, as NumPy gives."""
    for dt, odt in (("int32", "float64"), ("int64", "float64"), ("uint32", "float64"),
                    ("int8", "float32"), ("uint64", "float64")):
        x = np.array(_extremes(dt), dt)
        g = _run_expr(L, _multi(["trunc"], [dt], [odt]), [x])[0]
        np.testing.assert_array_equal(g, np.trunc(x.astype(odt)), err_msg=dt)


# ------------------------------------------------------------------------------------------
# C. the same bodies as a CAReduce pre-map and behind copy / cast / increment
# ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("geom", ["rows_1stage_vec128", "rows_1stage_offset1", "rows_2stage_vec128",
                                  "rows_2stage_offset1", "rows_2stage_negstride",
                                  "rows_2stage_strided_keep63", "rows_2stage_all_keep1",
                                  "rows_1stage_multidim_red", "rows_1stage_size1_dims",
                                  "cols_1stage_keep1057", "cols_2stage_keep64", "rows_1stage_nred0"])
@pytest.mark.parametrize("pre", ["int32_plus1", "int8_cast_int64"])
def test_careduce_premap_once_per_element(L, geom, pre):
    """sum(f(x)) with f = x + 1 (or a widening cast of int8 to int64): on all-zero input the sum
    of x + 1 counts the elements, so a map applied to the identity or to the stage-2 partials,
    or an element mapped twice or not at all, changes the count."""
    from tests.test_gpu_kernel_edges import _geometry, _place

    from aesara_b200.runtime import kernels as K

    if pre == "int32_plus1":
        dt, mid = "int32", "int64"
        expr = {"inputs": [dt], "out_dtypes": [mid], "outputs": ["t0"],
                "stmts": [_st("add", ["i0", {"const": 1, "dtype": "int8"}], mid, [dt, "int8"])]}
    else:
        dt, mid = "int8", "int64"
        expr = {"inputs": [dt], "out_dtypes": [mid], "outputs": ["t0"],
                "stmts": [_st("cast", ["i0"], mid, [dt])]}
    shape, axis, layout, launches = _geometry(geom, dt)
    rng = np.random.default_rng(zlib.crc32(geom.encode()))
    x = np.zeros(shape, dt) if pre == "int32_plus1" else rng.integers(-128, 128, shape).astype(dt)
    k = K.CAReduceKernel.get("add", dt, "int64", "int64", pre_expr=expr)
    before = L.ab_launch_count()
    got = k.launch(_place(x, layout, dt), axis).to_numpy()
    assert L.ab_launch_count() - before == (launches if got.size else 0)
    want = np.sum(x.astype(np.int64) + (1 if pre == "int32_plus1" else 0), axis=axis)
    np.testing.assert_array_equal(got, want, err_msg=geom)


@pytest.mark.parametrize("src", ["transposed", "neg_stride", "bcast_row", "bcast_col"])
def test_copy_cast_and_add_into(L, src):
    """copy_into (identity body), _cast_kernel (int16 -> float64 and float64 -> int32) and
    add_into (IncSubtensor) from transposed, negative-stride and broadcast sources."""
    from aesara_b200.runtime import kernels as K
    from aesara_b200.runtime.device import DeviceArray

    rng = np.random.default_rng(zlib.crc32(src.encode()))
    R, C = 70, 45
    base = rng.integers(-1000, 1000, (R, C)).astype(np.int16)
    if src == "transposed":
        s = Placed(base, _t_strides((R, C)))
        logical = base
    elif src == "neg_stride":
        s = Placed(base, (-C, -1))
        logical = base
    elif src == "bcast_row":
        s = Placed(base[:1])
        logical = np.broadcast_to(base[:1], (R, C))
    else:
        s = Placed(base[:, :1])
        logical = np.broadcast_to(base[:, :1], (R, C))
    dst = DeviceArray.from_numpy(np.zeros((R, C), np.int16))
    K.copy_into(dst, s.view)
    np.testing.assert_array_equal(dst.to_numpy(), logical)
    f = DeviceArray.from_numpy(np.zeros((R, C), np.float64))
    K.copy_into(f, s.view)
    np.testing.assert_array_equal(f.to_numpy(), logical.astype(np.float64))
    fsrc = Placed(base.astype(np.float64) + 0.75, s.view.strides if src in ("transposed", "neg_stride") else None)
    i = DeviceArray.from_numpy(np.zeros(fsrc.shape, np.int32))
    K.copy_into(i, fsrc.view)
    np.testing.assert_array_equal(i.to_numpy(), np.trunc(base.astype(np.float64) + 0.75)[:fsrc.shape[0]]
                                  .astype(np.int32)[:, :fsrc.shape[1]])
    acc = Placed(np.ones((R, C), np.int16) * 3, (C + 5, 1))
    K.add_into(acc.view, s.view)
    got, intact = acc.result()
    np.testing.assert_array_equal(got, 3 + logical)
    assert intact


# ------------------------------------------------------------------------------------------
# D. host and device agree
# ------------------------------------------------------------------------------------------
def _host_ops():
    from aesara_b200.runtime import host_eval

    return sorted(host_eval._OPS)


def _agree_values(dt, rng, n):
    if dt == "bool":
        return rng.random(n) < 0.5
    if np.dtype(dt).kind == "f":
        v = np.array([0.0, -0.0, 1.5, -2.5, 3.0, np.nan, np.inf, -np.inf, 16777217.0, -1.0,
                      4294967295.0, 2.0 ** 63, 0.1, -7.0, 2.5, 1e300], dt)
        return rng.choice(v, n)
    return rng.choice(np.array(_extremes(dt), dt), n)


_AGREE_OPS = ["lt", "gt", "le", "ge", "eq", "neq", "add", "sub", "mul", "and", "or", "xor",
              "maximum", "minimum", "int_div", "mod", "true_divide", "switch", "clip"]


def _agree_out(op, dts):
    kinds = {np.dtype(d).kind for d in dts}
    if op in ("lt", "gt", "le", "ge", "eq", "neq"):
        return "bool"
    if op == "true_divide" and kinds <= set("biu"):
        return "float64"
    return np.result_type(*[np.dtype(d) for d in dts]).name


@pytest.mark.parametrize("dx", DISCRETE + FLOATS)
def test_host_and_device_agree(L, dx):
    """Every op host_eval evaluates, at every dtype pair (switch(c, x, y) with a bool c, and
    clip(x, lo, hi) with lo and hi of the second dtype), on the same 64-element operands:
    host_eval.eval_expr and the device body return identical values.  Mixed signedness (int32
    with uint32, int64 with uint64) and int64 with float32 beyond 2**24 follow C's
    conversions in both."""
    from aesara_b200.runtime import host_eval

    rng = np.random.default_rng(zlib.crc32(dx.encode()))
    bad, n = [], 0
    for dy in DISCRETE + FLOATS:
        ins = [dx, dy, "bool", dy]
        stmts, host = [], []
        for op in _AGREE_OPS:
            if op == "switch":
                args, dts = ["i2", "i0", "i1"], ["bool", dx, dy]
                out = np.result_type(np.dtype(dx), np.dtype(dy)).name
            elif op == "clip":
                args, dts = ["i0", "i1", "i3"], [dx, dy, dy]
                out = _agree_out(op, dts)
            else:
                args, dts = ["i0", "i1"], [dx, dy]
                out = _agree_out(op, dts)
            if op == "sub" and "bool" in dts or op in ("int_div", "mod") and "bool" == dx == dy:
                continue
            if op in ("and", "or", "xor") and {np.dtype(d).kind for d in dts} & {"f"}:
                continue
            st = _st(op, args, out, dts)
            one = {"inputs": ins, "out_dtypes": [out], "outputs": ["t0"], "stmts": [st]}
            if out == "float16" or not host_eval.supports(one):
                continue  # float IntDiv / Mod are device-only
            stmts.append(st)
            host.append((op, one))
        expr = {"inputs": ins, "out_dtypes": [st["dtype"] for st in stmts],
                "outputs": [f"t{k}" for k in range(len(stmts))], "stmts": stmts,
                "name": f"agree_{dx}_{dy}"}
        vals = [_agree_values(d, rng, 64) for d in ins]
        if np.dtype(dy).kind != "f":  # clip bounds in order
            lo, hi = np.minimum(vals[1], vals[3]), np.maximum(vals[1], vals[3])
            vals[1], vals[3] = lo, hi
        dev = _run_expr(L, expr, vals)
        for (op, one), d in zip(host, dev):
            with np.errstate(all="ignore"):
                h = np.asarray(host_eval.eval_expr(one, vals)[0])
            n += 1
            assert h.dtype == d.dtype, (op, dx, dy, h.dtype, d.dtype)
            if h.dtype.kind == "f":
                same = _same_bits(h, d)
                if op in ("maximum", "minimum", "clip"):
                    same |= (h == 0) & (d == 0)  # the order of +-0 is not part of the contract
            else:
                same = h == d
            if not same.all():
                i = int(np.argmin(same))
                bad.append((op, dx, dy, [v[i] for v in vals], h[i], d[i]))
    assert n > 100
    assert not bad, f"host vs device differ in {len(bad)} cases: {bad[:6]}"


def test_zz_every_flavour_reached(L):
    print("\nElemwise flavours reached:", sorted(REACHED))
    if ULP_TABLE:
        print("op         dtype    bound  measured  points")
        for op, dt, b, w, n in ULP_TABLE:
            print(f"{op:10s} {dt:8s} {b:5} {w:9.3f} {n:7d}")
    assert REACHED == set(FLAVOURS), f"not reached: {set(FLAVOURS) - REACHED}"
