"""ORACLE (test infrastructure only — never imported by the product path).

NumPy restatement of the reference's scalar Ops, i.e. of the C expressions the
reference C-linker compiles for each ``ScalarOp`` (``aesara/scalar/basic.py``
``c_code`` methods, lines cited per entry; ``aesara/scalar/math.py:1110-1258``
for sigmoid / softplus / log1mexp).  Evaluates the IR scalar expressions of
``aesara_b200.ir`` over whole arrays.

Pinned against the reference itself: ``tests/golden/make_golden.py`` runs the real
reference (C-linker ``Mode("cvm")``; its Python ``perform`` for the few Ops whose C code no
longer builds on NumPy 2) on seeded inputs and commits programs,
inputs and reference outputs under ``tests/golden/``; ``tests/test_oracle.py`` checks this
oracle against every one of them.
"""

import numpy as np

_ERR = dict(all="ignore")


def _f(dt):
    return np.dtype(dt)


def _cast_like_c(x, dtype):
    """C conversion ``(T)x`` (basic.py:2466 Cast): float->int truncates,
    anything->bool is ``x ? 1 : 0``."""
    dt = np.dtype(dtype)
    x = np.asarray(x)
    if dt == np.bool_:
        return x != 0
    with np.errstate(**_ERR):
        return x.astype(dt)


def _c_common(a, b):
    """C's usual arithmetic conversions (the reference's C writes ``x < y``, ``x + y``,
    ``c ? x : y`` on the typed operands): integer promotion to int first, then the wider type
    of one signedness, an unsigned type over a signed one no wider than it, an int64 over a
    uint32; a float over any integer (int64 with float32 is float32)."""
    a, b = (np.dtype(np.int32) if (d.kind in "iub" and d.itemsize < 4) else d
            for d in (np.dtype(a), np.dtype(b)))
    if a.kind == "f" or b.kind == "f":
        return np.dtype(np.float64) if np.dtype(np.float64) in (a, b) else np.dtype(np.float32)
    if a.kind == b.kind or a == b:
        return a if a.itemsize >= b.itemsize else b
    signed, unsigned = (a, b) if a.kind == "i" else (b, a)
    return unsigned if unsigned.itemsize >= signed.itemsize else signed


def _c_pair(x, y):
    x, y = np.asarray(x), np.asarray(y)
    t = _c_common(x.dtype, y.dtype)
    with np.errstate(**_ERR):
        return x.astype(t), y.astype(t)


def _c_where(c, x, y):  # c ? x : y
    return np.where(np.asarray(c) != 0, *_c_pair(x, y))


def _upgrade(x, out_dtype):
    """``exp((T)x)`` style ops cast the argument to the *output* type first
    (basic.py:3102-3109)."""
    return np.asarray(x).astype(out_dtype, copy=False)


def _softplus(x):  # scalar/math.py:1172-1198 (same thresholds for all precisions)
    x = np.asarray(x)
    with np.errstate(**_ERR):
        return np.where(
            x < -37.0,
            np.exp(x),
            np.where(
                x < 18.0,
                np.log1p(np.exp(x)),
                np.where(x < 33.3, x + np.exp(-x), x),
            ),
        ).astype(x.dtype)


def _sigmoid(x):  # scalar/math.py:1110-1119
    x = np.asarray(x)
    one = x.dtype.type(1)
    with np.errstate(**_ERR):
        return (one / (one + np.exp(-x))).astype(x.dtype)


def _log1mexp(x):  # scalar/math.py:1248-1258
    x = np.asarray(x)
    with np.errstate(**_ERR):
        return np.where(
            x < x.dtype.type(-0.6931471805599453),
            np.log1p(-np.exp(x)),
            np.log(-np.expm1(x)),
        ).astype(x.dtype)


def _py_mod(x, y):  # basic.py:2165-2240: result has the sign of y (Python %)
    with np.errstate(**_ERR):
        rt = np.result_type(x, y)
        if np.issubdtype(rt, np.integer) or rt == np.bool_:
            x, y = np.asarray(x).astype(rt), np.asarray(y).astype(rt)
            y_safe = np.where(y == 0, rt.type(1), y)
            return np.where(y == 0, rt.type(0), np.mod(x, y_safe))
        # floats: the reference's branches (basic.py:2222-2236), which give a zero remainder the
        # sign np.mod does not (-6 % 3 = +0, 6 % -3 = +0)
        rt = np.result_type(x, y)
        x, y = np.broadcast_arrays(np.asarray(x, dtype=rt), np.asarray(y, dtype=rt))
        zero = rt.type(0)
        mm = -np.fmod(-x, -y)
        pm = np.fmod(x, -y)
        pm = pm + np.where(pm != 0, y, zero)
        mp = np.fmod(-x, y)
        mp = -mp + np.where(mp != 0, y, zero)
        pp = np.fmod(x, y)
        return np.where(y == 0, pp, np.where(y < 0, np.where(x < 0, mm, pm),
                                             np.where(x < 0, mp, pp))).astype(rt)


def _int_div(x, y):  # basic.py:2055-2127: floor division
    with np.errstate(**_ERR):
        rt = np.result_type(x, y)
        if np.issubdtype(rt, np.integer) or rt == np.bool_:
            x, y = np.asarray(x).astype(rt), np.asarray(y).astype(rt)
            y_safe = np.where(y == 0, rt.type(1), y)
            return np.where(y == 0, rt.type(0), np.floor_divide(x, y_safe))
        # floats: the reference divides magnitudes and corrects with fmod (basic.py:2083-2121);
        # this is not floor(x / y) for infinite divisors or when |x|/|y| rounds up to an integer
        x = np.asarray(x, dtype=rt)
        y = np.asarray(y, dtype=rt)
        x, y = np.broadcast_arrays(x, y)
        one = rt.type(1)
        pp = np.floor(x / y)
        mm = np.floor((-x) / (-y))
        pm = -np.floor(x / (-y)) - np.where(np.fmod(x, -y) == 0, 0, one)
        mp = -np.floor((-x) / y) - np.where(np.fmod(-x, y) == 0, 0, one)
        neg_y = np.where(x < 0, mm, pm)
        pos_y = np.where(x < 0, mp, pp)
        return np.where(y == 0, pp, np.where(y < 0, neg_y, pos_y)).astype(rt)


def _sgn(x):  # basic.py:2614-2630
    x = np.asarray(x)
    return np.sign(x)


def _maximum(x, y):  # basic.py:1745-1752: NaN if either is NaN
    return np.maximum(x, y)


def _minimum(x, y):  # basic.py:1788-1793
    return np.minimum(x, y)


def _erf_family(name):
    import scipy.special as sp

    return getattr(sp, name)


def apply_op(st, args):
    """Evaluate one IR statement on numpy operands."""
    op = st["op"]
    out = np.dtype(st["dtype"])
    a = args
    with np.errstate(**_ERR):
        if op == "add":  # basic.py:1829-1837 (bool: ||)
            r = a[0]
            for x in a[1:]:
                r = np.logical_or(r, x) if out == np.bool_ else np.add(*_c_pair(r, x))
        elif op == "mul":  # basic.py:1897-1907 (bool: &&)
            r = a[0]
            for x in a[1:]:
                r = np.logical_and(r, x) if out == np.bool_ else np.multiply(*_c_pair(r, x))
        elif op == "sub":  # :1955
            r = np.subtract(*_c_pair(a[0], a[1]))
        elif op == "true_divide":  # :1997-2011 ((double)x / y for two discrete args)
            x, y = np.asarray(a[0]), np.asarray(a[1])
            if x.dtype.kind in "biu" and y.dtype.kind in "biu":
                r = x.astype(np.float64) / y
            else:
                r = np.true_divide(*_c_pair(x, y))
        elif op == "int_div":
            r = _int_div(a[0], a[1])
        elif op == "mod":
            r = _py_mod(a[0], a[1])
        elif op == "pow":  # :2263
            r = np.power(np.asarray(a[0]).astype(np.result_type(a[0], a[1], out)), a[1])
        elif op == "neg":
            r = -np.asarray(a[0])
        elif op == "abs":
            r = np.abs(a[0])
        elif op == "sgn":
            r = _sgn(a[0])
        elif op == "sqr":
            r = np.asarray(a[0]) * np.asarray(a[0])
        elif op == "reciprocal":  # :2892  1.0 / x
            r = 1.0 / np.asarray(a[0]).astype(out)
        elif op == "identity":
            r = a[0]
        elif op == "second":
            r = np.broadcast_to(a[1], np.broadcast_shapes(np.shape(a[0]), np.shape(a[1])))
        elif op == "cast":
            r = _cast_like_c(a[0], out)
        elif op in ("lt", "gt", "le", "ge", "eq", "neq"):
            fn = dict(lt=np.less, gt=np.greater, le=np.less_equal,
                      ge=np.greater_equal, eq=np.equal, neq=np.not_equal)[op]
            r = fn(*_c_pair(a[0], a[1]))
        elif op == "isnan":
            r = np.isnan(a[0]) if np.asarray(a[0]).dtype.kind == "f" else np.zeros(np.shape(a[0]), bool)
        elif op == "isinf":
            r = np.isinf(a[0]) if np.asarray(a[0]).dtype.kind == "f" else np.zeros(np.shape(a[0]), bool)
        elif op == "inrange":
            lo = np.greater if st.get("openlow") else np.greater_equal
            hi = np.less if st.get("openhi") else np.less_equal
            r = np.logical_and(lo(*_c_pair(a[0], a[1])), hi(*_c_pair(a[0], a[2])))
        elif op == "switch":  # :1586  cond ? a : b
            r = _c_where(a[0], a[1], a[2])
        elif op == "clip":  # :2355
            x, lo, hi = a
            inner = _c_where(np.greater(*_c_pair(x, hi)), hi, x)
            r = _c_where(np.less(*_c_pair(x, lo)), lo, inner)
        elif op == "maximum":
            r = _maximum(a[0], a[1])
        elif op == "minimum":
            r = _minimum(a[0], a[1])
        elif op == "or":
            r = np.bitwise_or(*_c_pair(a[0], a[1]))
        elif op == "and":
            r = np.bitwise_and(*_c_pair(a[0], a[1]))
        elif op == "xor":
            r = np.bitwise_xor(*_c_pair(a[0], a[1]))
        elif op == "invert":
            r = np.logical_not(a[0]) if out == np.bool_ else np.invert(a[0])
        elif op == "mean":
            r = sum(np.asarray(x).astype(np.float64) for x in a) / float(len(a))
        elif op in ("exp", "exp2", "expm1", "log", "log2", "log10", "log1p", "sqrt",
                    "cos", "sin", "tan", "arccos", "arcsin", "arctan", "cosh", "sinh",
                    "tanh", "arccosh", "arcsinh", "arctanh", "ceil", "floor"):
            r = getattr(np, op)(_upgrade(a[0], out))
        elif op == "arctan2":
            r = np.arctan2(_upgrade(a[0], out), _upgrade(a[1], out))
        elif op == "trunc":  # of the argument cast to the float output: trunc(INT32_MIN) = -2**31
            r = np.trunc(_upgrade(a[0], out))
        elif op == "round_half_to_even":
            r = np.rint(a[0])
        elif op == "round_half_away_from_zero":
            x = np.asarray(a[0])
            r = np.where(x >= 0, np.floor(x + 0.5), np.ceil(x - 0.5))
        elif op == "deg2rad":
            r = np.asarray(a[0]) * (np.pi / 180.0)
        elif op == "rad2deg":
            r = np.asarray(a[0]) * (180.0 / np.pi)
        elif op == "sigmoid":
            r = _sigmoid(_upgrade(a[0], out))
        elif op == "softplus":
            r = _softplus(_upgrade(a[0], out))
        elif op == "log1mexp":
            r = _log1mexp(_upgrade(a[0], out))
        elif op in ("erf", "erfc", "erfinv", "erfcinv", "erfcx", "gamma", "gammaln"):
            r = _erf_family(op)(_upgrade(a[0], out))
        else:
            raise NotImplementedError(f"oracle: scalar op {op}")
        return np.asarray(r).astype(out, copy=False)


def eval_expr(expr, inputs):
    """Evaluate an IR scalar expression; ``inputs`` are broadcast-compatible
    numpy arrays.  Returns the list of output arrays."""
    temps = []

    def ref(r):
        if isinstance(r, dict):
            return np.asarray(r["const"], dtype=r["dtype"])
        if r[0] == "i":
            return inputs[int(r[1:])]
        return temps[int(r[1:])]

    for st in expr["stmts"]:
        temps.append(apply_op(st, [ref(r) for r in st["args"]]))
    return [ref(r) for r in expr["outputs"]]
