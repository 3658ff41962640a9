"""GPU: random variables drawn on the device (csrc/ab_random.cu) against the NumPy restatement
of the Philox stream (oracle/random_np.py): uniform and Bernoulli draws bit for bit at every
broadcast form of the parameters, normal draws within the float32 / float64 bounds of the
long-double truth from the same words, and the Generator semantics of RandomStream graphs
compiled with aesara.function."""
import copy
import zlib

import numpy as np
import pytest

from aesara_b200.compat import bootstrap
from oracle.program_np import run_program
from oracle.random_np import random_sample  # also installs the RandomVariable handler of run_program

pytestmark = [pytest.mark.gpu,
              pytest.mark.skipif(not bootstrap.available(), reason="reference front-end not available")]

NORMAL_TOL = {"float32": 4e-6, "float64": 1e-14}


@pytest.fixture(scope="module")
def aes():
    aesara = bootstrap.load_aesara()
    import aesara.tensor as at

    import aesara_b200.linker as L

    return aesara, at, L


def _key(g):
    return int(copy.deepcopy(g).integers(0, 2 ** 64, dtype=np.uint64))


def _rv(at, dist, dtype, params, size, rng):
    from aesara.tensor.random.basic import NormalRV, UniformRV

    # the module-level uniform / normal draw floatX; an Op of its own dtype keeps it through
    # the rewrites
    if dist == "uniform":
        return UniformRV(dtype=dtype)(*params, size=size, rng=rng)
    if dist == "normal":
        return NormalRV(dtype=dtype)(*params, size=size, rng=rng)
    if dist == "bernoulli":
        return at.random.bernoulli(*params, size=size, rng=rng)
    return at.random.binomial(1, *params, size=size, rng=rng)


def _draw(aes, dist, dtype, params, size, seed=0, sym=(), views=None):
    """Compile one draw; params[k] is a constant unless k is in `sym` (then a function input,
    uploaded, optionally passed through views[k] inside the graph).  Returns (device sample,
    oracle sample, key)."""
    aesara, at, L = aes
    g = aesara.shared(np.random.default_rng(seed))
    ins, gp, vals = [], [], []
    for k, p in enumerate(params):
        p = np.asarray(p)
        if k in sym:
            v = at.tensor(dtype=p.dtype.name, shape=(None,) * p.ndim)
            ins.append(v)
            vals.append(p)
            gp.append(views[k](v) if views and k in views else v)
        else:
            gp.append(at.constant(p))
    x = _rv(at, dist, dtype, gp, size, g)
    f = aesara.function(ins, x, mode=L.mode(), updates={g: x.owner.outputs[0]})
    key = _key(g.get_value(borrow=True))
    got = f(*vals)
    eff = [views[k](p) if views and k in views else p for k, p in enumerate(params)]
    eff = [np.asarray(p) for p in eff]
    shape = got.shape
    want = random_sample("bernoulli" if dist == "binomial" else dist, x.dtype, key, shape,
                         eff[-1:] if dist in ("bernoulli", "binomial") else eff)
    return got, want, key


def _assert_draws(dist, got, want):
    assert got.shape == want.shape
    if dist == "normal":
        err = np.abs(got.astype(np.float64) - want) / (1 + np.abs(want))
        assert (err.max() if err.size else 0.0) <= NORMAL_TOL[got.dtype.name], err.max()
    else:
        assert got.dtype == want.dtype
        np.testing.assert_array_equal(got, want)


R, C = 6, 9
_FORMS = {
    # name: (params per distribution -> list, size, symbolic positions)
    "scalars": (lambda d: _params(d, (), ()), (R, C), ()),
    "per_row": (lambda d: _params(d, (R, 1), (R, 1)), (R, C), (0, 1)),
    "per_col": (lambda d: _params(d, (C,), (C,)), (R, C), (0, 1)),
    "full": (lambda d: _params(d, (R, C), (R, C)), (R, C), (0, 1)),
    "mixed": (lambda d: _params(d, (R, 1), (C,)), (R, C), (0, 1)),
    "zero_d": (lambda d: _params(d, (), ()), None, ()),
    "inferred": (lambda d: _params(d, (R, C), (1, C)), None, (0, 1)),
    "zero_size": (lambda d: _params(d, (), ()), (0, C), ()),
    "const_full": (lambda d: _params(d, (R, C), (R, C)), (R, C), ()),
    "size_3d": (lambda d: _params(d, (4, 1, 5), (1, 3, 1)), (4, 3, 5), (0, 1)),
}


def _params(dist, s0, s1, seed=1):
    r = np.random.default_rng(seed)
    if dist == "uniform":
        lo = r.uniform(-3, 0, s0)
        return [lo, lo + r.uniform(0.5, 4, s1)]
    if dist == "normal":
        return [r.uniform(-3, 3, s0), r.uniform(0.1, 3, s1)]
    p = r.uniform(0, 1, s1 if s1 else s0)
    return [p]


@pytest.mark.parametrize("form", list(_FORMS))
@pytest.mark.parametrize("dist, dtype", [("uniform", "float32"), ("uniform", "float64"), ("normal", "float32"),
                                         ("normal", "float64"), ("bernoulli", "int64"), ("binomial", "int64")])
def test_broadcast_forms_match_the_stream(aes, form, dist, dtype):
    mk, size, sym = _FORMS[form]
    params = mk(dist)
    sym = tuple(k for k in sym if k < len(params))
    got, want, _ = _draw(aes, dist, dtype, params, size, seed=zlib.crc32(f"{form}{dist}{dtype}".encode()) % 1000, sym=sym)
    _assert_draws(dist, got, want)


@pytest.mark.parametrize("n", [1, 3, 4, 5, 1000, 2 ** 24 + 3])
@pytest.mark.parametrize("dist, dtype", [("uniform", "float32"), ("uniform", "float64"), ("normal", "float32"),
                                         ("normal", "float64"), ("bernoulli", "int64")])
def test_sizes_match_the_stream(aes, n, dist, dtype):
    params = {"uniform": [-1.5, 2.5], "normal": [0.5, 2.0], "bernoulli": [0.37]}[dist]
    got, want, _ = _draw(aes, dist, dtype, params, (n,), seed=n)
    _assert_draws(dist, got, want)


@pytest.mark.parametrize("dist, dtype", [("uniform", "float32"), ("normal", "float64"), ("bernoulli", "int64")])
def test_strided_parameter_views(aes, dist, dtype):
    """Parameters read through a column-strided slice and a transposed view on the device."""
    r = np.random.default_rng(4)
    if dist == "bernoulli":
        params, views = [r.uniform(0, 1, (2 * C, R))], {0: lambda v: v.T[:, ::2]}
    else:
        base = r.uniform(0.1, 2, (R, 2 * C))
        params = [base, r.uniform(2.5, 4, (C, R))]
        views = {0: lambda v: v[:, ::2], 1: lambda v: v.T}
    got, want, _ = _draw(aes, dist, dtype, params, (R, C), sym=tuple(range(len(params))), views=views)
    _assert_draws(dist, got, want)


def test_probability_edges(aes):
    got, _, _ = _draw(aes, "bernoulli", "int64", [np.array([0.0, 1.0, 0.0, 1.0])], (1000, 4), sym=(0,))
    np.testing.assert_array_equal(got, np.broadcast_to([0, 1, 0, 1], (1000, 4)))


@pytest.mark.parametrize("dist, params, sym", [
    ("normal", [0.0, np.array([1.0, -0.5])], ()), ("normal", [0.0, np.array([1.0, -0.5])], (1,)),
    ("bernoulli", [np.array([0.2, 1.5])], ()), ("bernoulli", [np.array([0.2, np.nan])], (0,)),
    ("bernoulli", [np.array([-0.1, 0.5])], (0,)),
])
def test_invalid_parameters_raise_value_error(aes, dist, params, sym):
    with pytest.raises(ValueError, match="scale < 0" if dist == "normal" else "p < 0"):
        _draw(aes, dist, "float64", params, (2,), sym=sym)
    # the flag is cleared: a valid draw afterwards succeeds
    got, want, _ = _draw(aes, "bernoulli", "int64", [np.array([0.5, 0.5])], (2,), sym=(0,))
    _assert_draws("bernoulli", got, want)


# -- Function-level semantics ----------------------------------------------------------------------
def _stream_fn(aes, seed, **mode_kw):
    aesara, at, L = aes
    from aesara.tensor.random.utils import RandomStream

    srng = RandomStream(seed=seed)
    u = srng.uniform(0.0, 1.0, size=(5, 7))
    z = srng.normal(0.0, 1.0, size=(33,))
    return srng, aesara.function([], [u, z], mode=L.mode(**mode_kw))


def test_successive_calls_differ_and_the_generator_advances_once_per_draw(aes):
    aesara, at, L = aes
    s = 1234
    g = aesara.shared(np.random.default_rng(s))
    u = at.random.uniform(0.0, 1.0, size=(4, 4), rng=g)
    nxt = u.owner.outputs[0]
    v = at.random.normal(0.0, 1.0, size=(3,), rng=nxt)
    f = aesara.function([], [u, v], mode=L.mode(), updates={g: v.owner.outputs[0]})
    outs = [f() for _ in range(3)]
    assert not np.array_equal(outs[0][0], outs[1][0]) and not np.array_equal(outs[1][1], outs[2][1])
    want = np.random.default_rng(s)
    for _ in range(3 * 2):  # two RV nodes per call
        want.integers(0, 2 ** 64, dtype=np.uint64)
    assert g.get_value(borrow=True).bit_generator.state == want.bit_generator.state


def test_reseeding_and_recompiling_reproduce_the_draws(aes):
    srng, f = _stream_fn(aes, 77)
    first = f()
    f()
    srng.seed(77)
    again = f()
    for a, b in zip(first, again):
        np.testing.assert_array_equal(a, b)
    _, f2 = _stream_fn(aes, 77)
    for a, b in zip(first, f2()):
        np.testing.assert_array_equal(a, b)


def test_cuda_graph_mode_gives_the_eager_sequence(aes):
    _, eager = _stream_fn(aes, 5)
    _, graphed = _stream_fn(aes, 5, cuda_graph=True)
    for _ in range(4):
        for a, b in zip(eager(), graphed()):
            np.testing.assert_array_equal(a, b)
    assert graphed.vm._replay is not None and graphed.vm._replay.replays == 0


def test_output_subset_still_advances_the_rng(aes):
    aesara, at, L = aes
    from aesara.tensor.random.utils import RandomStream

    x = at.fvector("x")
    srng = RandomStream(seed=9)
    u = srng.uniform(0.0, 1.0, size=(6,))
    f = aesara.function([x], [u, x + 1], mode=L.mode())
    g = srng.state_updates[0][0]
    before = copy.deepcopy(g.get_value(borrow=True))
    f(np.zeros(2, "float32"), output_subset=[1])
    before.integers(0, 2 ** 64, dtype=np.uint64)
    assert g.get_value(borrow=True).bit_generator.state == before.bit_generator.state


# -- dropout MLP -------------------------------------------------------------------------------------
def _dropout_mlp(aes, p=0.25):
    aesara, at, L = aes
    from aesara.tensor.random.utils import RandomStream

    X, Y = at.fmatrix("X"), at.fmatrix("Y")
    W1, b1, W2, b2 = at.fmatrix("W1"), at.fvector("b1"), at.fmatrix("W2"), at.fvector("b2")
    srng = RandomStream(seed=2024)
    h = at.tanh(X @ W1 + b1)
    mask = srng.bernoulli(1 - p, size=h.shape)
    hd = h * mask / np.float32(1 - p)
    out = hd @ W2 + b2
    loss = at.mean((out - Y) ** 2)
    g = aesara.grad(loss, [W1, b1, W2, b2])
    ins = [X, Y, W1, b1, W2, b2]
    B, H = 64, 48
    r = np.random.default_rng(3)
    vals = [r.standard_normal((B, H)).astype("float32"), r.standard_normal((B, H)).astype("float32"),
            (r.standard_normal((H, H)) / 8).astype("float32"), np.zeros(H, "float32"),
            (r.standard_normal((H, H)) / 8).astype("float32"), np.zeros(H, "float32")]
    return ins, [loss] + list(g), vals


def test_dropout_mlp_step_matches_the_oracle(aes):
    aesara, at, L = aes
    ins, outs, vals = _dropout_mlp(aes)
    f = aesara.function(ins, outs, mode=L.mode())
    prog = f.maker.linker.program
    assert any(n.op == "RandomVariable" for n in prog.nodes)
    for _ in range(2):
        state = [copy.deepcopy(c[0]) for c in f.vm.input_storage[len(ins):]]
        got = f(*vals)
        want = run_program(prog, [np.array(a) for a in vals] + state)
        for k, (g, w) in enumerate(zip(got, want)):
            w = np.asarray(w, np.float64)
            err = float(np.max(np.abs(np.asarray(g, np.float64) - w)) / max(np.max(np.abs(w)), 1e-30))
            assert err < 1e-5, f"output {k}: normwise error {err}"


def test_check_function_passes_on_the_dropout_graph(aes):
    from aesara_b200.debug import check_function

    ins, outs, vals = _dropout_mlp(aes)
    report = check_function(ins, outs, vals)
    assert report


# -- sanity of the distributions -------------------------------------------------------------------
def test_moments_at_2_24_elements(aes):
    aesara, at, L = aes
    from aesara.tensor.random.utils import RandomStream

    n = 2 ** 24
    srng = RandomStream(seed=31337)
    p = 0.3
    from aesara.tensor.random.basic import NormalRV, UniformRV

    outs = []
    for dt in ("float32", "float64"):
        outs += [srng.gen(UniformRV(dtype=dt), 0.0, 1.0, size=(n,)), srng.gen(NormalRV(dtype=dt), 0.0, 1.0, size=(n,))]
    outs.append(srng.bernoulli(p, size=(n,)))
    assert [o.dtype for o in outs] == ["float32", "float32", "float64", "float64", "int64"]
    uf, nf, ud, nd, b = aesara.function([], outs, mode=L.mode())()
    for u in (uf, ud):
        u = u.astype(np.float64)
        assert abs(u.mean() - 0.5) < 5 * np.sqrt(1 / 12 / n)
        assert abs(u.var() - 1 / 12) < 5 * np.sqrt((1 / 80 - 1 / 144) / n)
        assert u.min() >= 0 and u.max() < 1
    for z in (nf, nd):
        z = z.astype(np.float64)
        assert abs(z.mean()) < 5 / np.sqrt(n)
        assert abs(z.var() - 1) < 5 * np.sqrt(2 / n)
    assert abs(b.mean() - p) < 5 * np.sqrt(p * (1 - p) / n)
