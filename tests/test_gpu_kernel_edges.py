"""GPU: the hand-written kernels outside the GEMM, at the edges of their launch paths.

CAReduce, Softmax / LogSoftmax / SoftmaxGrad, MaxAndArgmax, CumOp, the row gather and
scatter, and Gemv / Ger each pick a path from host-side constants (how many outputs fill the
132 SMs, whether a run is 16-byte aligned, whether a row fits one warp or x fits in shared
memory).  Every case here is chosen to land on one named side of such a switch, and its id says
which.  Where the launch count shows the path (a two-stage reduction and the Gemv column
pattern launch two kernels) it is asserted.

Truth is NumPy: exact where the operands make the answer exact (integers, integer-valued or
dyadic floats whose partial results stay representable, NaN / tie positions placed by hand), so
that a wrong tile, chunk, carry or winner fails by equality; elsewhere float64 with the bound of
the operation's error analysis given where it is used.  ``u32 = 2**-24`` and ``u64 = 2**-53`` are
the unit roundoffs.  The duplicate-index semantics of the scatters are checked at the op level,
through ``aesara.function(mode="B200")``.
"""
import math
import zlib

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

U32, U64 = 2.0 ** -24, 2.0 ** -53


def _u(dt):
    return U32 if np.dtype(dt) == np.float32 else U64


@pytest.fixture(scope="module")
def L():
    import torch

    from aesara_b200.runtime import lib

    lib.check(lib.load().ab_init(0))
    torch.cuda.set_device(0)
    return lib.load()


def _dev(a):
    from aesara_b200.runtime.device import DeviceArray

    return DeviceArray.from_numpy(a)


def _code(dt):
    from aesara_b200.ir import DTYPE_CODE

    return DTYPE_CODE[np.dtype(dt).name]


def _stream():
    from aesara_b200.runtime.device import stream_handle

    return stream_handle()


def _check(rc):
    from aesara_b200.runtime import lib

    lib.check(rc)


def _vec(dt):
    return max(1, 16 // np.dtype(dt).itemsize)


def _per_cta(dt):
    """Reduced elements one CTA of the row pattern takes before the range is split."""
    return 256 * _vec(dt) * 8


# ---------------------------------------------------------------------------------------------
# CAReduce
# ---------------------------------------------------------------------------------------------
_INTS = ["int8", "int16", "int32", "int64", "uint8", "uint64"]
_WIDE = {"int8": "int64", "int16": "int64", "int32": "int64", "int64": "int64",
         "uint8": "uint64", "uint64": "uint64", "bool": "int64",
         "float32": "float64", "float64": "float64"}


def _signature(op, dt):
    """(op, in, acc, out) as the reference types the reduction (elemwise.py:1371-1385):
    sums and products accumulate wide, float32 sums in float64 with a float32 result."""
    if op in ("add", "mul", "mul_without_zeros"):
        acc = _WIDE[dt]
        return op, dt, acc, ("float32" if dt == "float32" else acc)
    return op, dt, dt, dt


REDUCE_SIGNATURES = sorted(
    {_signature(op, dt) for op in ("add", "mul") for dt in ["float32", "float64", "bool"] + _INTS}
    | {_signature("mul_without_zeros", dt) for dt in ["float32", "float64", "int8", "int32", "int64", "uint8"]}
    | {_signature(op, dt) for op in ("and", "or", "xor") for dt in ["bool", "int16"] + _INTS}
    | {_signature(op, dt) for op in ("maximum", "minimum") for dt in ["float32", "float64", "bool", "int16"] + _INTS}
)


def _geometry(geom, dt):
    """-> (logical shape, reduced axes, memory layout, kernels launched)."""
    P = _per_cta(dt)
    return {
        # one CTA per output, reduced run contiguous and 16-byte aligned (128-bit loads): the
        # 4 x 256 x vec unrolled body, its vector remainder and a scalar tail (n_red % vec != 0)
        "rows_1stage_vec128": ((5, P - 3), (1,), "pad", 1),
        # the same run one element off 16-byte alignment: vec_ok = 0, scalar loads
        "rows_1stage_offset1": ((5, P - 3), (1,), "off1", 1),
        # n_keep < 8 * SMs and n_red > 256 * vec * 8: the range is split, stage 2 folds slices
        "rows_2stage_vec128": ((3, 2 * P + 5), (1,), "pad", 2),
        "rows_2stage_offset1": ((3, 2 * P + 5), (1,), "off1", 2),
        "rows_2stage_negstride": ((3, 2 * P + 5), (1,), "neg", 2),
        # n_keep = 63 < 64 along axis 0: row pattern with a strided reduced index, split
        "rows_2stage_strided_keep63": ((P + 1, 63), (0,), "c", 2),
        # everything reduced (n_keep = 1), split
        "rows_2stage_all_keep1": ((3 * P + 7,), (0,), "c", 2),
        # two reduced dims that cannot merge (nr = 2)
        "rows_1stage_multidim_red": ((7, 33, 70), (1, 2), "swap12", 1),
        # size-1 dims on both sides are dropped
        "rows_1stage_size1_dims": ((1, 5, 1, 300), (0, 3), "c", 1),
        # column pattern: reduced axis leading, n_keep >= 64 outputs contiguous
        "cols_1stage_keep1057": ((40, 1057), (0,), "c", 1),
        "cols_2stage_keep64": ((300, 64), (0,), "c", 2),
        # an empty reduced range gives the identity
        "rows_1stage_nred0": ((6, 0), (1,), "c", 1),
    }[geom]


GEOMS = ["rows_1stage_vec128", "rows_1stage_offset1", "rows_2stage_vec128", "rows_2stage_offset1",
         "rows_2stage_negstride", "rows_2stage_strided_keep63", "rows_2stage_all_keep1",
         "rows_1stage_multidim_red", "rows_1stage_size1_dims", "cols_1stage_keep1057",
         "cols_2stage_keep64", "rows_1stage_nred0"]


def _place(a, layout, dt):
    """A device view holding the logical array ``a`` in the given memory layout."""
    from aesara_b200.runtime.device import DeviceArray

    if layout == "c":
        return _dev(a)
    if layout == "swap12":  # [k, r1, r2] stored as [k, r2, r1]
        d = _dev(np.ascontiguousarray(a.transpose(0, 2, 1)))
        k, r1, r2 = a.shape
        return d.view(a.shape, (r1 * r2, 1, r1))
    rows, cols = a.shape
    v = _vec(dt)
    pitch = -(-cols // v) * v
    if layout == "neg":  # row r, column c at buf[r, cols - 1 - c]
        d = _dev(np.ascontiguousarray(a[:, ::-1]))
        return d.view(a.shape, (cols, -1), cols - 1)
    off = 1 if layout == "off1" else 0
    buf = np.zeros(rows * pitch + off + v, dtype=a.dtype)
    buf[off:off + rows * pitch].reshape(rows, pitch)[:, :cols] = a
    d = _dev(buf)
    out = d.view(a.shape, (pitch, 1), off)
    assert isinstance(out, DeviceArray)
    return out


def _red_data(op, dt, shape, rng):
    dt = np.dtype(dt)
    if dt.kind == "b":
        p = {"and": 0.999, "mul": 0.999, "or": 0.001}.get(op, 0.5)
        return rng.random(shape) < p
    info = np.iinfo(dt) if dt.kind in "iu" else None
    if op in ("mul", "mul_without_zeros"):
        # +-1 and at most 30 twos per array: every product is an exact power of two (or its
        # integer), whatever the order; mul_without_zeros also gets zeros to skip
        x = np.ones(shape, dt)
        if dt.kind != "u":
            x[rng.random(shape) < 0.5] = -1
        flat = x.reshape(-1)
        if flat.size:
            flat[rng.integers(0, flat.size, 30)] = 2
        if op == "mul_without_zeros":
            x[rng.random(shape) < 0.05] = 0
        return x
    if op == "add":
        if dt.kind == "f":  # integer-valued: every partial sum is exact in the accumulator
            return rng.integers(-64, 65, shape).astype(dt)
        return rng.integers(info.min, info.max, shape, dtype=dt, endpoint=True)
    if op in ("and", "or"):
        fill = (info.max if dt.kind == "u" else -1) if op == "and" else 0
        x = np.full(shape, fill, dt)
        m = rng.random(shape) < 0.002
        x[m] = rng.integers(info.min, info.max, int(m.sum()), dtype=dt, endpoint=True)
        return x
    if dt.kind == "f":
        return rng.integers(-10 ** 6, 10 ** 6, shape).astype(dt)
    return rng.integers(info.min, info.max, shape, dtype=dt, endpoint=True)


def _red_truth(op, x, axis, acc, out):
    if op == "add":
        return np.sum(x.astype(acc), axis=axis, dtype=acc).astype(out)
    if op == "mul":
        return np.prod(x.astype(acc), axis=axis, dtype=acc).astype(out)
    if op == "mul_without_zeros":
        xa = x.astype(acc)
        p = np.prod(np.where(xa == 0, np.ones((), acc), xa), axis=axis, dtype=acc)
        return np.where(np.all(xa == 0, axis=axis), np.zeros((), acc), p).astype(out)
    f = {"and": np.bitwise_and, "or": np.bitwise_or, "xor": np.bitwise_xor,
         "maximum": np.maximum, "minimum": np.minimum}[op]
    return f.reduce(x, axis=axis).astype(out)


def _reduce(L, sig, X, axis):
    from aesara_b200.runtime import kernels as K

    k = K.CAReduceKernel.get(*sig)
    before = L.ab_launch_count()
    out = k.launch(X, axis)
    return out.to_numpy(), L.ab_launch_count() - before


def _sig_id(sig):
    return "-".join(sig)


@pytest.mark.parametrize("geom", GEOMS)
@pytest.mark.parametrize("sig", REDUCE_SIGNATURES, ids=_sig_id)
def test_careduce_exact(L, sig, geom):
    """Every combine op and dtype on every geometry, with operands that make the answer exact:
    integer results match NumPy in the same accumulator dtype (wraparound included: an int8
    sum leaves int8, an int64 sum wraps like NumPy's), float results are exact because every
    partial result is an integer (sums) or a power of two (products)."""
    op, dt, acc, out = sig
    shape, axis, layout, launches = _geometry(geom, dt)
    if 0 in shape and op in ("maximum", "minimum"):
        pytest.skip("maximum/minimum have no identity: the op raises before launching")
    rng = np.random.default_rng(zlib.crc32(f"{sig}{geom}".encode()))
    x = _red_data(op, dt, shape, rng)
    if op == "mul_without_zeros" and len(shape) > len(axis):  # the first output: all zeros
        np.moveaxis(x, axis, tuple(range(-len(axis), 0)))[(0,) * (len(shape) - len(axis))] = 0
    got, n = _reduce(L, sig, _place(x, layout, dt), axis)
    want = _red_truth(op, x, axis, acc, out)
    assert n == launches, f"{geom}: {n} kernels launched, expected {launches}"
    np.testing.assert_array_equal(got, want, err_msg=f"{_sig_id(sig)} {geom}")


@pytest.mark.parametrize("op,dt", [("add", "float32"), ("maximum", "int16")])
@pytest.mark.parametrize("n_keep,axis,launches", [
    (1, 1, 2), (63, 1, 2), (64, 1, 2), (1055, 1, 2), (1056, 1, 1), (1057, 1, 1),
    (63, 0, 1), (64, 0, 2),
], ids=["rows_keep1_2stage", "rows_keep63_2stage", "rows_keep64_2stage", "rows_keep1055_2stage",
        "rows_keep1056_1stage", "rows_keep1057_1stage", "axis0_keep63_rows", "axis0_keep64_cols_2stage"])
def test_careduce_n_keep_boundaries(L, op, dt, n_keep, axis, launches):
    """The split decision at n_keep = 8 * SMs (1056 on an H100), with n_red one past what a CTA
    takes alone; and the row / column choice at n_keep = 64 for a leading reduced axis."""
    if axis == 1:
        shape = (n_keep, _per_cta(dt) + 1)
    else:
        shape = (100, n_keep)
    sig = _signature(op, dt)
    rng = np.random.default_rng(n_keep)
    x = _red_data(op, dt, shape, rng)
    got, n = _reduce(L, sig, _dev(x), (axis,))
    assert n == launches
    np.testing.assert_array_equal(got, _red_truth(op, x, (axis,), sig[2], sig[3]))


@pytest.mark.parametrize("dt", ["float32", "float64"])
@pytest.mark.parametrize("op", ["maximum", "minimum"])
def test_careduce_nan_propagates(L, op, dt):
    """max / min return NaN for any slice with a NaN: in the scalar tail after the 128-bit
    body, in one slice of a split row (stage 1 of the other slices sees none, so only stage 2's
    input carries it), in the first and in the last slice, and in one column of a split column
    reduction."""
    sig = _signature(op, dt)
    rng = np.random.default_rng(3)
    P = _per_cta(dt)
    cases = []
    x = _red_data(op, dt, (5, P - 3), rng)
    x[2, -1] = np.nan  # scalar tail
    x[4, 1] = np.nan   # first vector of the unrolled body
    cases.append(("rows_1stage_vec128", x, "pad", (1,), 1))
    x = _red_data(op, dt, (4, 2 * P + 5), rng)
    x[0, P + 3] = np.nan   # middle slice only
    x[1, 0] = np.nan       # first slice
    x[2, -1] = np.nan      # last slice (its tail)
    cases.append(("rows_2stage_vec128", x, "pad", (1,), 2))
    cases.append(("rows_2stage_offset1", x, "off1", (1,), 2))
    x = _red_data(op, dt, (300, 64), rng)
    x[299, 5] = np.nan     # last row slice of column 5
    x[0, 63] = np.nan
    cases.append(("cols_2stage_keep64", x, "c", (0,), 2))
    x = _red_data(op, dt, (3 * P + 7,), rng)
    x[-1] = np.nan
    cases.append(("rows_2stage_all_keep1", x, "c", (0,), 2))
    for name, x, layout, axis, launches in cases:
        got, n = _reduce(L, sig, _place(x, layout, dt), axis)
        assert n == launches, name
        want = np.max(x, axis=axis) if op == "maximum" else np.min(x, axis=axis)
        assert np.isnan(want).any()
        np.testing.assert_array_equal(got, want, err_msg=name)


def test_careduce_uint64_max_above_2_63(L):
    """Unsigned 64-bit comparisons: the maximum sits above 2**63 (a signed compare would
    pick a small value), the minimum below, on a split 128-bit row reduction, a strided one and
    the whole array."""
    rng = np.random.default_rng(7)
    P = _per_cta("uint64")
    x = rng.integers(0, 2 ** 62, (3, 2 * P + 5), dtype=np.uint64)
    x[:, 17] = np.uint64(2 ** 63 + 5)
    x[1, -2] = np.uint64(2 ** 64 - 1)
    for op, f in (("maximum", np.max), ("minimum", np.min)):
        sig = _signature(op, "uint64")
        for X, axis in ((_place(x, "pad", "uint64"), (1,)), (_dev(np.ascontiguousarray(x.T)), (0,))):
            got, _ = _reduce(L, sig, X, axis)
            np.testing.assert_array_equal(got, f(x, axis=1))
    assert _reduce(L, _signature("maximum", "uint64"), _dev(x), (0, 1))[0] == np.uint64(2 ** 64 - 1)


@pytest.mark.parametrize("geom", ["rows_1stage_vec128", "rows_2stage_vec128", "rows_2stage_offset1",
                                  "rows_2stage_negstride", "rows_2stage_all_keep1",
                                  "rows_1stage_multidim_red", "cols_2stage_keep64", "cols_1stage_keep1057"])
@pytest.mark.parametrize("dt", ["float32", "float64"])
def test_careduce_float_sum_bound(L, dt, geom):
    """Random normal sums.  The device accumulates in float64 in an order fixed by the launch
    geometry: |S64 - S| <= (n - 1) * u64 * sum|x| for any order.  A float32 result then rounds
    once, so it is within one float32 ulp of float32(fsum) plus that bound; a float64 result
    is within the bound of fsum."""
    sig = _signature("add", dt)
    shape, axis, layout, launches = _geometry(geom, dt)
    rng = np.random.default_rng(11)
    x = rng.standard_normal(shape).astype(dt)
    got, n = _reduce(L, sig, _place(x, layout, dt), axis)
    assert n == launches
    xm = np.moveaxis(x, axis, tuple(range(-len(axis), 0)))
    xm = xm.reshape(xm.shape[: xm.ndim - len(axis)] + (-1,)).astype(np.float64)
    lines = xm.reshape(-1, xm.shape[-1])
    exact = np.array([math.fsum(r) for r in lines]).reshape(got.shape)
    nred = lines.shape[1]
    bound = (nred - 1) * U64 * np.abs(lines).sum(axis=1).reshape(got.shape)
    if dt == "float32":
        ref = exact.astype(np.float32)
        bound = bound + np.spacing(np.abs(ref)).astype(np.float64)
        err = np.abs(got.astype(np.float64) - ref.astype(np.float64))
    else:
        err = np.abs(got - exact)
    assert (err <= bound).all(), f"{geom}: max excess {np.max(err - bound)}"


def test_careduce_two_stage_sum_is_deterministic(L):
    """Two launches of a split float32 sum give the same bits (no floating-point atomics)."""
    sig = _signature("add", "float32")
    rng = np.random.default_rng(12)
    x = rng.standard_normal((3, 4 * _per_cta("float32") + 1)).astype("float32")
    X = _dev(x)
    a, n = _reduce(L, sig, X, (1,))
    b, _ = _reduce(L, sig, X, (1,))
    assert n == 2
    np.testing.assert_array_equal(a.view(np.uint32), b.view(np.uint32))


# ---------------------------------------------------------------------------------------------
# Softmax / LogSoftmax / SoftmaxGrad
# ---------------------------------------------------------------------------------------------
_SM_SHAPES = ([(outer, R, 1) for R in (1, 2, 31, 32, 33, 1023, 1024, 1025, 4099) for outer in (1, 7, 8, 9, 1001)]
              + [(outer, R, inner) for R in (1, 33, 1025) for outer in (1, 9) for inner in (3, 257)])


def _sm_id(s):
    outer, R, inner = s
    path = "cols" if inner > 1 else ("warp" if R <= 1024 else "cta")
    return f"{path}-outer{outer}-R{R}-inner{inner}"


def _sm_lines(outer, R, inner, dt, rng):
    """[outer, R, inner] with the line (o, j) of kind (o * inner + j) % 6: normal, about +-80,
    about +-1e4 (exp overflows without the max shift), some -inf, all -inf, one NaN.  Values are
    multiples of 1/64 below 2**14: x - max is exact in float32."""
    lines = rng.standard_normal((outer * inner, R))
    kind = np.arange(outer * inner) % 6
    lines[kind == 1] *= 80
    lines[kind == 2] *= 1e4
    lines = np.round(lines * 64) / 64
    lines = np.clip(lines, -16000, 16000)
    for li in np.nonzero(kind == 3)[0]:
        lines[li, rng.integers(0, R, max(1, R // 3))] = -np.inf
        if R > 1:
            lines[li, rng.integers(0, R)] = 1.5  # keeps one finite entry
    lines[kind == 4] = -np.inf
    for li in np.nonzero(kind == 5)[0]:
        lines[li, rng.integers(0, R)] = np.nan
    return np.ascontiguousarray(lines.reshape(outer, inner, R).transpose(0, 2, 1)).astype(dt)


def _softmax_launch(L, mode, x, s=None):
    outer, R, inner = x.shape
    out = _dev(np.zeros_like(x))
    a = _dev(x)
    b = _dev(s) if s is not None else None
    _check(L.ab_softmax(_code(x.dtype), mode, outer, R, inner, a.ptr, b.ptr if b is not None else None,
                        out.ptr, _stream()))
    return out.to_numpy()


def _same_specials(got, want):
    np.testing.assert_array_equal(np.isnan(got), np.isnan(want))
    fin = np.isfinite(want)
    np.testing.assert_array_equal(got[~fin & ~np.isnan(want)], want[~fin & ~np.isnan(want)])
    return fin


@pytest.mark.parametrize("shape", _SM_SHAPES, ids=_sm_id)
@pytest.mark.parametrize("dt", ["float32", "float64"])
def test_softmax_and_log_softmax(L, dt, shape):
    """Truth: float64 NumPy with the max shift.  x - max is exact (dyadic operands), the sum of
    exponentials is a float64 sum of float64 exponentials on the device (relative error
    <= (R + 4) u64, and as much again for the NumPy truth) and the rest are three single
    roundings in the row dtype (exp, 1/sum, product; log and subtraction), so

    softmax:      |y - t| <= (4 u + 2 (R + 4) u64) |t| + 2**-125 (float32 subnormals)
    log-softmax:  |y - t| <= 2 u (|t| + |L|) + 2 (R + 4) u64,  L = log(sum exp(x - max)).

    An all -inf line is NaN (like the reference: -inf - -inf), NaN stays in its own line, -inf
    entries give 0 / -inf exactly."""
    outer, R, inner = shape
    rng = np.random.default_rng(R * 31 + outer * 7 + inner)
    x = _sm_lines(outer, R, inner, dt, rng)
    x64 = x.astype(np.float64)
    with np.errstate(invalid="ignore", over="ignore", divide="ignore"):
        m = np.max(x64, axis=1, keepdims=True)
        d = x64 - m
        e = np.exp(d)
        S = e.sum(axis=1, keepdims=True)
        sm = e / S
        lsm = d - np.log(S)
    u = _u(dt)
    got = _softmax_launch(L, 0, x)
    fin = _same_specials(got, sm)
    bound = (4 * u + 2 * (R + 4) * U64) * np.abs(sm) + (2.0 ** -125 if dt == "float32" else 2.0 ** -1020)
    err = np.abs(got.astype(np.float64) - sm)
    assert (err[fin] <= bound[fin]).all(), f"softmax: max excess {np.max((err - bound)[fin])}"
    got = _softmax_launch(L, 1, x)
    fin = _same_specials(got, lsm)
    with np.errstate(invalid="ignore", divide="ignore"):
        bound = 2 * u * (np.abs(lsm) + np.abs(np.log(S))) + 2 * (R + 4) * U64
    with np.errstate(invalid="ignore"):
        err = np.abs(got.astype(np.float64) - lsm)
    assert (err[fin] <= bound[fin]).all(), f"log-softmax: max excess {np.max((err - bound)[fin])}"


@pytest.mark.parametrize("shape", _SM_SHAPES, ids=_sm_id)
@pytest.mark.parametrize("dt", ["float32", "float64"])
def test_softmax_grad(L, dt, shape):
    """dy*sm - sum(dy*sm)*sm with dy in [-4, 4] integers and sm multiples of 1/256: dy*sm and
    the float64 row sum are exact (and the sum fits float32), so the only roundings are
    tot*sm and the subtraction: |y - t| <= 2 u (|tot * sm| + |t|)."""
    outer, R, inner = shape
    rng = np.random.default_rng(R + outer + inner)
    dy = rng.integers(-4, 5, shape).astype(dt)
    sm = (rng.integers(0, 256, shape) / 256).astype(dt)
    tot = (dy.astype(np.float64) * sm).sum(axis=1, keepdims=True)
    want = dy.astype(np.float64) * sm - tot * sm
    got = _softmax_launch(L, 2, dy, sm).astype(np.float64)
    bound = 2 * _u(dt) * (np.abs(tot * sm) + np.abs(want))
    assert (np.abs(got - want) <= bound).all()


# ---------------------------------------------------------------------------------------------
# MaxAndArgmax
# ---------------------------------------------------------------------------------------------
def _argmax_rows(R, dt, rng):
    """Rows, each with a hand-placed winner: ties at i and i+256 (one thread, two strided
    passes), i and i+128 (two threads meeting in the tree), i and i+1, the maximum at the last
    element, two NaNs (the first wins), all equal (index 0), all -inf / all at the type's minimum."""
    dt = np.dtype(dt)
    if dt.kind == "b":
        rows = [rng.random(R) < 0.01, np.zeros(R, bool), np.ones(R, bool)]
        last = np.zeros(R, bool)
        last[-1] = True
        return np.array(rows + [last])
    if dt.kind == "f":
        base = lambda: rng.integers(-1000, 1000, R).astype(dt)  # noqa: E731
        top, low = dt.type(5000), dt.type(-np.inf)
    elif dt == np.uint64:
        base = lambda: rng.integers(0, 2 ** 63 + 12345, R, dtype=np.uint64)  # noqa: E731
        top, low = np.uint64(2 ** 63 + 99999), np.uint64(0)
    else:
        info = np.iinfo(dt)
        base = lambda: rng.integers(info.min, info.max - 1, R, dtype=dt, endpoint=True)  # noqa: E731
        top, low = dt.type(info.max), dt.type(info.min)
    rows = [base()]
    for gap in (256, 128, 1):
        if R > gap:
            r = base()
            i = int(rng.integers(0, R - gap))
            r[i] = r[i + gap] = top
            rows.append(r)
    r = base()
    r[-1] = top
    rows.append(r)
    if dt.kind == "f" and R > 1:
        r = base()
        i = int(rng.integers(0, R - 1))
        r[i + 1:] = top  # larger values after the first NaN do not win
        r[i] = r[R - 1] = np.nan
        rows.append(r)
    rows.append(np.full(R, base()[0], dt))
    rows.append(np.full(R, low, dt))
    return np.array(rows)


@pytest.mark.parametrize("R", [1, 255, 256, 257, 513, 100003])
@pytest.mark.parametrize("dt", ["float32", "float64", "int8", "uint64", "bool"])
def test_max_and_argmax(L, dt, R):
    """Exact: the maximum and the index of its first occurrence (np.argmax; NaN wins, the first
    NaN)."""
    rng = np.random.default_rng(R)
    x = _argmax_rows(R, dt, rng)
    outer = x.shape[0]
    X = _dev(x)
    omax = _dev(np.zeros(outer, x.dtype))
    oidx = _dev(np.full(outer, -1, np.int64))
    _check(L.ab_max_and_argmax(_code(dt), outer, R, X.ptr, omax.ptr, oidx.ptr, _stream()))
    np.testing.assert_array_equal(oidx.to_numpy(), np.argmax(x, axis=1))
    np.testing.assert_array_equal(omax.to_numpy(), np.max(x, axis=1))


# ---------------------------------------------------------------------------------------------
# CumOp
# ---------------------------------------------------------------------------------------------
_CUM_SHAPES = ([(3, Ln, 1) for Ln in (1, 255, 256, 2047, 2048, 2049, 6145)] + [(2, 10 ** 6 + 7, 1)]
               + [(3, 2049, inner) for inner in (2, 255, 257)] + [(2, 1, 257)])


def _cum_id(s):
    return f"{'lines' if s[2] > 1 else 'block'}-outer{s[0]}-L{s[1]}-inner{s[2]}"


def _cum(L, mul, x):
    outer, Ln, inner = x.shape
    out = _dev(np.zeros_like(x))
    _check(L.ab_cumulative(_code(x.dtype), int(mul), _dev(x).ptr, out.ptr, outer, Ln, inner, _stream()))
    return out.to_numpy()


@pytest.mark.parametrize("shape", _CUM_SHAPES, ids=_cum_id)
@pytest.mark.parametrize("dt", ["float32", "float64"])
def test_cumsum_cumprod_exact_floats(L, dt, shape):
    """Integer-valued summands in [-8, 8] (every prefix sum below 2**24) and factors +-1 with
    sparse 2s and 1/2s (every prefix product a power of two): each carry between 2048-element
    chunks and each warp-scan step is checked by equality."""
    rng = np.random.default_rng(shape[1] + shape[2])
    x = rng.integers(-8, 9, shape).astype(dt)
    np.testing.assert_array_equal(_cum(L, False, x), np.cumsum(x.astype(np.float64), axis=1).astype(dt))
    f = np.where(rng.random(shape) < 0.5, -1.0, 1.0)
    p = min(0.05, 40.0 / shape[1])
    f[rng.random(shape) < p] = 2.0
    f[rng.random(shape) < p] = 0.5
    f = f.astype(dt)
    np.testing.assert_array_equal(_cum(L, True, f), np.cumprod(f.astype(np.float64), axis=1).astype(dt))


@pytest.mark.parametrize("shape", [(3, 6145, 1), (2, 10 ** 6 + 7, 1), (3, 2049, 257)], ids=_cum_id)
def test_cumsum_random_float32_bound(L, shape):
    """Random normal float32: element k (1-based) of any summation order is within
    k * eps32 * sum_{i<=k} |x_i| of the exact prefix sum."""
    rng = np.random.default_rng(5)
    x = rng.standard_normal(shape).astype("float32")
    got = _cum(L, False, x).astype(np.float64)
    x64 = x.astype(np.float64)
    want = np.cumsum(x64, axis=1)  # float64: its own error is far below the bound
    k = np.arange(1, shape[1] + 1, dtype=np.float64)[None, :, None]
    bound = k * np.finfo(np.float32).eps * np.cumsum(np.abs(x64), axis=1)
    assert (np.abs(got - want) <= bound).all()


@pytest.mark.parametrize("shape", [(3, 2049, 1), (2, 6145, 1), (3, 257, 255)], ids=_cum_id)
@pytest.mark.parametrize("dt", ["int8", "int16", "int32", "int64", "uint8", "uint64"])
def test_cumsum_cumprod_integers_wrap(L, dt, shape):
    """Integer CumOp wraps in the input dtype, exactly like np.cumsum(x, dtype=x.dtype) (int8
    products overflow on the first few elements)."""
    info = np.iinfo(dt)
    rng = np.random.default_rng(shape[1])
    x = rng.integers(info.min, info.max, shape, dtype=dt, endpoint=True)
    np.testing.assert_array_equal(_cum(L, False, x), np.cumsum(x, axis=1, dtype=x.dtype))
    y = rng.integers(max(info.min, -7), 8, shape).astype(dt)
    np.testing.assert_array_equal(_cum(L, True, y), np.cumprod(y, axis=1, dtype=y.dtype))


# ---------------------------------------------------------------------------------------------
# Row gather (AdvancedSubtensor1)
# ---------------------------------------------------------------------------------------------
# (element dtype, inner, extra elements of row padding, element offset, vector width chosen)
_GATHER = [
    ("uint8", 16, 0, 0, "uint4"), ("uint8", 8, 0, 0, "uint2"), ("uint8", 4, 0, 0, "u32"),
    ("uint8", 2, 0, 0, "u16"), ("uint8", 3, 0, 0, "u8"), ("uint8", 16, 0, 1, "u8_oddptr"),
    ("int16", 8, 0, 0, "uint4"), ("int16", 4, 0, 0, "uint2"), ("int16", 8, 2, 0, "u32_padded"),
    ("int16", 3, 0, 0, "u16"), ("float32", 4, 0, 0, "uint4"), ("float32", 6, 0, 0, "uint2"),
    ("float32", 3, 0, 0, "u32"), ("float32", 4, 0, 1, "u32_offset"), ("float64", 2, 0, 0, "uint4"),
    ("float64", 3, 0, 0, "uint2"), ("float64", 4, 1, 0, "uint2_padded"),
]
_IDX_DTYPES = ["int8", "int16", "int32", "int64", "uint8", "uint16", "uint32"]


@pytest.mark.parametrize("idx_dt", _IDX_DTYPES)
@pytest.mark.parametrize("dt,inner,pad,off,width", _GATHER, ids=[f"{g[0]}-inner{g[1]}-{g[4]}" for g in _GATHER])
def test_take_rows_byte_exact(L, dt, inner, pad, off, width, idx_dt):
    """out[r] = x[idx[r]] byte for byte at each vector width (row bytes, row stride and pointer
    alignment select it), with every index dtype; negative indices wrap."""
    n_rows, n_idx = 100, 1000
    rng = np.random.default_rng(inner * 7 + off)
    raw = rng.integers(0, 256, (n_rows * (inner + pad) + off) * np.dtype(dt).itemsize, dtype=np.uint8)
    buf = raw.view(dt)
    x = buf[off:].reshape(n_rows, inner + pad)[:, :inner]
    lo = -n_rows if np.dtype(idx_dt).kind == "i" else 0
    idx = rng.integers(lo, n_rows, n_idx).astype(idx_dt)
    X = _dev(buf)
    out = _dev(np.zeros((n_idx, inner), dt))
    I = _dev(idx)
    _check(L.ab_take_rows(np.dtype(dt).itemsize, _code(idx_dt), X.ptr + off * X.itemsize, inner + pad,
                          n_rows, inner, I.ptr, 1, n_idx, out.ptr, 1, _stream()))
    want = x[idx.astype(np.int64)]
    np.testing.assert_array_equal(out.to_numpy().view(np.uint8), want.view(np.uint8))


def test_take_rows_out_of_range_then_in_range(L):
    """An out-of-range index returns AB_ERR_SHAPE (IndexError at the op): the kernel skips the
    index (no out-of-bounds read) and the flag is cleared, so the next call in the process
    succeeds."""
    from aesara_b200.runtime import lib

    x = np.arange(50 * 4, dtype=np.float32).reshape(50, 4)
    X = _dev(x)
    for bad in (50, -51):
        idx = np.array([1, bad, 3] * 40, np.int64)
        out = _dev(np.zeros((idx.size, 4), np.float32))
        I = _dev(idx)
        with pytest.raises(lib.AbError) as ei:
            _check(L.ab_take_rows(4, _code("int64"), X.ptr, 4, 50, 4, I.ptr, 1, idx.size, out.ptr, 1, _stream()))
        assert ei.value.code == 4
        good = np.array([49, -50, 7] * 40, np.int64)
        I = _dev(good)
        _check(L.ab_take_rows(4, _code("int64"), X.ptr, 4, 50, 4, I.ptr, 1, good.size, out.ptr, 1, _stream()))
        np.testing.assert_array_equal(out.to_numpy(), x[good])


# ---------------------------------------------------------------------------------------------
# Row scatter (AdvancedIncSubtensor1 / AdvancedIncSubtensor) through aesara.function
# ---------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def fe(L):
    from aesara_b200.compat import bootstrap

    if not bootstrap.available():
        pytest.skip("reference front-end (oracle/_ref) not present")
    aesara = bootstrap.load_aesara()
    import aesara.tensor as at

    import aesara_b200.linker as lk

    return aesara, at, lk


def _fn(fe, build, *types):
    aesara, at, lk = fe
    ins = [at.TensorType(dt, shape=(None,) * nd)() for dt, nd in types]
    f = aesara.function(ins, build(at, *ins), mode=lk.mode())
    return f


def _last_wins(n_rows, idx):
    """For each destination row, the position of its last occurrence in idx (-1 if none)."""
    last = np.full(n_rows, -1, np.int64)
    last[idx] = np.arange(idx.size)  # NumPy assigns in order: the last occurrence stays
    return last


@pytest.mark.parametrize("dt", ["int8", "uint8", "int16", "uint16", "int32", "int64", "float32", "float64"])
@pytest.mark.parametrize("pattern", ["all_equal", "random_dups", "y_broadcast_rows"])
def test_scatter_add_exact(fe, dt, pattern):
    """inc_subtensor(x[idx], y): np.add.at in the same dtype.  1- and 2-byte types go through
    a CAS on the containing word, 4- and 8-byte through native atomics; every index equal is
    the most contention.  Small types wrap; float y values are integers, so any order is exact."""
    n_rows, inner = 37, 3
    rng = np.random.default_rng(len(dt) + len(pattern))
    n_idx = 20_000
    idx = np.full(n_idx, 11, np.int64) if pattern == "all_equal" else rng.integers(-n_rows, n_rows, n_idx)
    dtn = np.dtype(dt)
    if dtn.kind == "f":
        x = rng.integers(-50, 50, (n_rows, inner)).astype(dt)
        y = rng.integers(-50, 50, (n_idx, inner)).astype(dt)
    else:
        info = np.iinfo(dt)
        x = rng.integers(info.min, info.max, (n_rows, inner), dtype=dt, endpoint=True)
        lo = info.min if dtn.itemsize < 4 else max(info.min, -1000)
        y = rng.integers(lo, min(info.max, 1000) if dtn.itemsize >= 4 else info.max, (n_idx, inner),
                         dtype=dt, endpoint=True)
    if pattern == "y_broadcast_rows":
        y = y[:1].reshape(inner)
    f = _fn(fe, lambda at, x_, i_, y_: at.inc_subtensor(x_[i_], y_), (dt, 2), ("int64", 1), (dt, y.ndim))
    want = x.copy()
    np.add.at(want, idx, y)
    np.testing.assert_array_equal(f(x, idx, y), want)


def _dup_indices(n_rows, rng, n_dup=100_000):
    """10**5 occurrences of row 7 among random others, in random order."""
    idx = np.concatenate([np.full(n_dup, 7), rng.integers(0, n_rows, 5000)])
    rng.shuffle(idx)
    return idx


@pytest.mark.parametrize("dt", ["float32", "int8", "int64"])
def test_set_with_duplicates_last_occurrence_wins_1d(fe, dt):
    """set_subtensor(x[idx], y) (AdvancedIncSubtensor1): a row named several times gets y of its
    LAST occurrence, as in the reference's perform (x[idx] = y) and its C loop."""
    n_rows, inner = 40, 3
    rng = np.random.default_rng(1)
    idx = _dup_indices(n_rows, rng)
    y = np.arange(idx.size * inner).reshape(idx.size, inner)
    y = (y % 120 if dt == "int8" else y).astype(dt)  # distinct values, except int8 (120 of them)
    x = np.full((n_rows, inner), -1, dt)
    f = _fn(fe, lambda at, x_, i_, y_: at.set_subtensor(x_[i_], y_), (dt, 2), ("int64", 1), (dt, 2))
    got = f(x, idx, y)
    last = _last_wins(n_rows, idx)
    want = x.copy()
    want[last >= 0] = y[last[last >= 0]]
    np.testing.assert_array_equal(got, want)


def test_set_with_duplicates_last_occurrence_wins_2d(fe):
    """set_subtensor(x[i, j], y) (AdvancedIncSubtensor, two index vectors): the last occurrence
    of each (i, j) pair wins."""
    rng = np.random.default_rng(2)
    A, B, inner = 6, 7, 5
    flat = _dup_indices(A * B, rng)
    i, j = flat // B, flat % B
    y = np.arange(flat.size * inner).reshape(flat.size, inner).astype("float32")  # distinct
    x = np.zeros((A, B, inner), "float32")
    f = _fn(fe, lambda at, x_, i_, j_, y_: at.set_subtensor(x_[i_, j_], y_),
            ("float32", 3), ("int64", 1), ("int64", 1), ("float32", 2))
    last = _last_wins(A * B, flat)
    want = x.reshape(A * B, inner).copy()
    want[last >= 0] = y[last[last >= 0]]
    np.testing.assert_array_equal(f(x, i, j, y), want.reshape(A, B, inner))


@pytest.mark.parametrize("set_", [False, True], ids=["inc", "set"])
@pytest.mark.parametrize("nidx", [1, 2])
def test_ignore_duplicates(fe, set_, nidx):
    """inc_subtensor(x[idx], y, ignore_duplicates=True) is the reference's out[idx] += y: each
    named row gets x[d] + y[last occurrence] (not the sum of all occurrences); with
    set_instead_of_inc it is y[last occurrence]."""
    rng = np.random.default_rng(3 + nidx)
    if nidx == 1:
        n_rows, inner = 40, 3
        flat = _dup_indices(n_rows, rng, 20_000)
        x = rng.integers(-100, 100, (n_rows, inner)).astype("float32")
        ins = [flat]
        build = lambda at, x_, i_, y_: at.inc_subtensor(x_[i_], y_, set_instead_of_inc=set_,  # noqa: E731
                                                        ignore_duplicates=True)
        types = [("float32", 2), ("int64", 1), ("float32", 2)]
    else:
        A, B, inner = 5, 8, 3
        n_rows = A * B
        flat = _dup_indices(n_rows, rng, 20_000)
        x = rng.integers(-100, 100, (A, B, inner)).astype("float32")
        ins = [flat // B, flat % B]
        build = lambda at, x_, i_, j_, y_: at.inc_subtensor(x_[i_, j_], y_, set_instead_of_inc=set_,  # noqa: E731
                                                            ignore_duplicates=True)
        types = [("float32", 3), ("int64", 1), ("int64", 1), ("float32", 2)]
    y = np.arange(flat.size * inner).reshape(flat.size, inner).astype("float32")  # distinct
    f = _fn(fe, build, *types)
    got = f(x, *ins, y)
    last = _last_wins(n_rows, flat)
    want = x.reshape(n_rows, inner).copy()
    hit = last >= 0
    want[hit] = y[last[hit]] if set_ else want[hit] + y[last[hit]]
    np.testing.assert_array_equal(got, want.reshape(x.shape))


@pytest.mark.parametrize("mode,launches", [(0, 1), (1, 2), (2, 2)], ids=["add_atomic", "set_last", "add_last"])
@pytest.mark.parametrize("dt", ["int8", "int64"])
def test_scatter_rows_modes_abi(L, dt, mode, launches):
    """ab_scatter_rows at the C ABI: the last-occurrence modes run a winner pass first (two
    kernels, an int64 of workspace per row and no less); np.add.at is one atomic pass.  An
    out-of-range index still returns AB_ERR_SHAPE, and the next call succeeds."""
    import ctypes as C

    from aesara_b200.runtime import lib

    n_rows, inner = 30, 5
    rng = np.random.default_rng(mode)
    idx = np.concatenate([np.full(5000, -3), rng.integers(0, n_rows, 3000)])
    rng.shuffle(idx)
    y = (np.arange(idx.size * inner) % 100).reshape(idx.size, inner).astype(dt)
    x = rng.integers(-20, 20, (n_rows, inner)).astype(dt)
    last = _last_wins(n_rows, idx % n_rows)
    want = x.copy()
    hit = last >= 0
    if mode == 0:
        np.add.at(want, idx, y)
    else:
        want[hit] = y[last[hit]] if mode == 1 else want[hit] + y[last[hit]]
    ws_bytes = C.c_size_t()
    _check(L.ab_scatter_rows_workspace_bytes(mode, n_rows, C.byref(ws_bytes)))
    assert ws_bytes.value == (0 if mode == 0 else 8 * n_rows)
    ws = _dev(np.zeros(max(ws_bytes.value, 1), np.uint8))
    X, I, Y = _dev(x), _dev(idx), _dev(y)

    def run(I, n_idx, nbytes):
        return L.ab_scatter_rows(_code(dt), _code("int64"), mode, X.ptr, inner, n_rows, inner, I.ptr, 1,
                                 n_idx, Y.ptr, inner, 1, ws.ptr, nbytes, 1, _stream())

    if mode:
        with pytest.raises(lib.AbError) as ei:
            _check(run(I, idx.size, ws_bytes.value - 1))
        assert ei.value.code == 3
    bad = _dev(np.array([0, n_rows, 1], np.int64))
    with pytest.raises(lib.AbError) as ei:
        _check(run(bad, 3, ws_bytes.value))
    assert ei.value.code == 4
    X = _dev(x)
    before = L.ab_launch_count()
    _check(run(I, idx.size, ws_bytes.value))
    assert L.ab_launch_count() - before == launches
    np.testing.assert_array_equal(X.to_numpy(), want)


# ---------------------------------------------------------------------------------------------
# Gemv / Ger
# ---------------------------------------------------------------------------------------------
def _int_operands(m, n, dt, rng, a_layout="c", a_off=0):
    """Integer-valued A in [-3, 3] and x in [-3, 3]: every dot product is an integer far below
    2**24, so the result is exact in any summation order."""
    from aesara_b200.runtime.device import DeviceArray

    a = rng.integers(-3, 4, (m, n)).astype(dt)
    x = rng.integers(-3, 4, n).astype(dt)
    if a_layout == "c":
        buf = np.zeros(m * n + a_off, dt)
        buf[a_off:] = a.reshape(-1)
        A = _dev(buf).view((m, n), (n, 1), a_off)
    elif a_layout == "f":  # column pattern: a_rs == 1
        buf = np.zeros(m * n + a_off, dt)
        buf[a_off:] = a.T.reshape(-1)
        A = _dev(buf).view((m, n), (1, m), a_off)
    else:  # "strided_row": one row with a column stride of 3
        buf = np.zeros((m, 3 * n), dt)
        buf[:, ::3] = a
        A = _dev(buf).view((m, n), (3 * n, 3))
    assert isinstance(A, DeviceArray)
    return a, x, A


def _smem_n(dt):
    return 40 * 1024 // np.dtype(dt).itemsize


_GEMV = [
    # (id, m, n, layout, A offset, kernels launched)
    ("rows_vec_x_in_smem_at_limit", 37, "smem", "c", 0, 1),
    ("rows_vec_x_in_global_one_past", 37, "smem+4", "c", 0, 1),
    ("rows_scalar_x_smem_limit_plus1", 37, "smem+1", "c", 0, 1),
    ("rows_scalar_n_mod4", 300, 1023, "c", 0, 1),
    ("rows_scalar_A_offset1", 300, 1024, "c", 1, 1),
    ("m1_strided_row_generic", 1, 777, "strided_row", 0, 1),
    ("m1_contiguous_row", 1, 5001, "c", 0, 1),
    ("cols_vec_split", 64, 20000, "f", 0, 2),
    ("cols_m3_split", 3, 30000, "f", 0, 2),
    ("cols_m_mod_nv_split", 1001, 4099, "f", 0, 2),
    ("cols_A_offset1_split", 256, 5000, "f", 1, 2),
]


@pytest.mark.parametrize("dt", ["float32", "float64"])
@pytest.mark.parametrize("case", _GEMV, ids=[c[0] for c in _GEMV])
def test_gemv_paths_exact(L, dt, case):
    """y <- alpha A x + beta y with integer-valued operands: exact on every path.  beta = 0 must
    not read y (it starts as NaN)."""
    from aesara_b200.runtime import kernels as K

    name, m, n, layout, off, launches = case
    if isinstance(n, str):
        n = _smem_n(dt) + (int(n.split("+")[1]) if "+" in n else 0)
    rng = np.random.default_rng(m + n)
    a, x, A = _int_operands(m, n, dt, rng, layout, off)
    want = a.astype(np.float64) @ x.astype(np.float64)
    for alpha, beta in ((1.0, 0.0), (2.0, -3.0)):
        y0 = rng.integers(-5, 6, m).astype(dt)
        y = _dev(np.full(m, np.nan, dt) if beta == 0.0 else y0)
        before = L.ab_launch_count()
        K.gemv(y, alpha, A, _dev(x), beta)
        assert L.ab_launch_count() - before == launches, name
        np.testing.assert_array_equal(y.to_numpy(), (alpha * want + beta * y0.astype(np.float64) * (beta != 0)).astype(dt))


@pytest.mark.parametrize("dt", ["float32", "float64"])
@pytest.mark.parametrize("m,n,order", [(4097, 3, "c"), (4097, 3, "f"), (3, 4097, "c"), (3, 4097, "f"), (130, 77, "f")],
                         ids=["m4097_rowmajor_gridy_clamp", "m4097_colmajor_swapped", "n4097_rowmajor",
                              "n4097_colmajor_swapped_gridy_clamp", "small_colmajor_swapped"])
def test_ger_exact(L, dt, m, n, order):
    """A <- A + alpha x y^T with integer-valued operands (exact): both axis orders of A (the
    thread index runs along the smaller stride, so a column-major A swaps x and y) and more
    than 4096 rows along grid.y (clamped, each CTA row loops)."""
    from aesara_b200.runtime import kernels as K

    rng = np.random.default_rng(m * n)
    a = rng.integers(-9, 10, (m, n)).astype(dt)
    x = rng.integers(-9, 10, m).astype(dt)
    y = rng.integers(-9, 10, n).astype(dt)
    A = _dev(a) if order == "c" else _dev(np.ascontiguousarray(a.T)).dimshuffle([1, 0])
    K.ger(A, 2.0, _dev(x), _dev(y))
    np.testing.assert_array_equal(A.to_numpy(), a + 2 * np.outer(x, y).astype(dt))
