"""GPU: Cholesky factorisations and triangular solves on the device (csrc/ab_linalg.cu) against
float64 truth: backward errors within c*n*eps, the opposite triangle exactly 0, agreement with
scipy within a condition-aware bound, residuals of every (lower, trans, unit_diagonal) solve, the
reference's exceptions, a Gaussian-process likelihood with its gradients, the tensor-core and
CUDA-core update paths, and CUDA-graph mode."""
import numpy as np
import pytest
import scipy.linalg
import torch

from aesara_b200.compat import bootstrap

pytestmark = [pytest.mark.gpu,
              pytest.mark.skipif(not bootstrap.available(), reason="reference front-end not available")]

EPS = {"float32": np.finfo(np.float32).eps, "float64": np.finfo(np.float64).eps}


@pytest.fixture(scope="module")
def aes():
    aesara = bootstrap.load_aesara()
    import aesara.tensor as at

    import aesara_b200.linker as L

    return aesara, at, L


def _spd(n, cond, seed):
    """Symmetric positive definite n x n (float64) with eigenvalues geometric over [1, cond],
    built on the GPU in float64."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    q, _ = torch.linalg.qr(torch.randn(n, n, dtype=torch.float64, device="cuda", generator=g))
    ev = torch.logspace(0, np.log10(cond), n, dtype=torch.float64, device="cuda")
    a = (q * ev) @ q.T
    return ((a + a.T) / 2).cpu().numpy()


def _embed(a):
    """m with m[::-2, ::2] == a (the other elements are NaN: they must not be read)."""
    m = np.full((2 * a.shape[0], 2 * a.shape[1]), np.nan, a.dtype)
    m[::-2, ::2] = a
    return m


# graph-side view of the input -> host array that the view maps back to the matrix
_VIEWS = {
    "contiguous": (lambda A: A, lambda a: a),
    "transposed": (lambda A: A.T, lambda a: np.ascontiguousarray(a.T)),
    "strided": (lambda A: A[::-2, ::2], _embed),
}
_FUNCS = {}


def _chol_fn(aes, dtype, lower, view, on_error="raise"):
    key = ("chol", dtype, lower, view, on_error)
    if key not in _FUNCS:
        aesara, at, L = aes
        from aesara.tensor.slinalg import Cholesky

        A = at.matrix("A", dtype=dtype)
        _FUNCS[key] = aesara.function([A], Cholesky(lower=lower, on_error=on_error)(_VIEWS[view][0](A)), mode=L.mode())
    return _FUNCS[key]


def _backward_error(L, a, lower):
    """||L L^T - A||_F / ||A||_F in float64 on the GPU (L^T L for the upper factor)."""
    t = torch.from_numpy(np.asarray(L, np.float64)).cuda()
    r = t @ t.T if lower else t.T @ t
    a = torch.from_numpy(np.asarray(a, np.float64)).cuda()
    return float(torch.linalg.norm(r - a) / torch.linalg.norm(a))


def _check_factor(L, a, lower, dtype):
    n = a.shape[0]
    assert L.dtype == np.dtype(dtype) and L.shape == (n, n)
    other = np.triu(L, 1) if lower else np.tril(L, -1)
    assert not np.any(other), "the opposite triangle is not exactly 0"
    err = _backward_error(L, a, lower)
    assert err <= 4 * max(n, 16) * EPS[dtype], f"backward error {err:.3g} at n={n}"


@pytest.mark.parametrize("dtype", ["float32", "float64"])
@pytest.mark.parametrize("view", list(_VIEWS))
@pytest.mark.parametrize("lower", [True, False])
@pytest.mark.parametrize("n", [1, 2, 31, 63, 64, 65, 127, 128, 129, 1000, 4099])
def test_cholesky_backward_error(aes, n, lower, view, dtype):
    a = _spd(n, 100.0, seed=n).astype(dtype)
    f = _chol_fn(aes, dtype, lower, view)
    L = f(_VIEWS[view][1](a))
    _check_factor(L, a.astype(np.float64), lower, dtype)


@pytest.mark.parametrize("lower", [True, False])
def test_cholesky_float32_8192(aes, lower):
    n = 8192
    a = _spd(n, 1e3, seed=8192).astype("float32")
    L = _chol_fn(aes, "float32", lower, "contiguous")(a)
    _check_factor(L, a.astype(np.float64), lower, "float32")


@pytest.mark.parametrize("dtype", ["float32", "float64"])
@pytest.mark.parametrize("cond", [10.0, 1e3, 1e6])
def test_cholesky_matches_scipy_within_the_condition_bound(aes, cond, dtype):
    n = 300
    a = _spd(n, cond, seed=int(cond)).astype(dtype)
    for lower in (True, False):
        L = _chol_fn(aes, dtype, lower, "contiguous")(a)
        want = scipy.linalg.cholesky(a.astype(np.float64), lower=lower)
        err = np.linalg.norm(L.astype(np.float64) - want) / np.linalg.norm(want)
        assert err <= 2 * n * EPS[dtype] * cond, f"cond {cond:g}: forward error {err:.3g}"
        _check_factor(L, a.astype(np.float64), lower, dtype)


# -- triangular solves -----------------------------------------------------------------------------
def _tri(n, lower, unit, seed, dtype):
    """A triangular matrix with diagonal in [1, 2] (7 on it when unit: it must not be read) and
    off-diagonal entries of size 1/sqrt(n); the other triangle holds values that must not be read."""
    r = np.random.default_rng(seed)
    a = r.standard_normal((n, n)) / np.sqrt(n)
    np.fill_diagonal(a, 7.0 if unit else r.uniform(1.0, 2.0, n))
    return a.astype(dtype)


def _effective(a, lower, unit):
    t = np.tril(a) if lower else np.triu(a)
    if unit:
        np.fill_diagonal(t, 1.0)
    return t


@pytest.mark.parametrize("dtype", ["float32", "float64"])
@pytest.mark.parametrize("rhs", ["vector", "thin", "wide"])
@pytest.mark.parametrize("unit", [False, True])
@pytest.mark.parametrize("trans", [0, 1])
@pytest.mark.parametrize("lower", [True, False])
def test_solve_triangular_residual(aes, lower, trans, unit, rhs, dtype):
    aesara, at, L = aes
    from aesara.tensor.slinalg import solve_triangular

    n = 1000 if rhs != "wide" else 700
    a = _tri(n, lower, unit, seed=11, dtype=dtype)
    r = np.random.default_rng(12)
    b = {"vector": r.standard_normal(n), "thin": r.standard_normal((n, 7)), "wide": r.standard_normal((n, 4096))}[rhs]
    b = b.astype(dtype)
    A = at.matrix("A", dtype=dtype)
    B = at.tensor(dtype=dtype, shape=(None,) * b.ndim, name="B")
    f = aesara.function([A, B], solve_triangular(A, B, lower=lower, trans=trans, unit_diagonal=unit), mode=L.mode())
    x = f(a, b)
    assert x.dtype == np.dtype(dtype) and x.shape == b.shape
    t = torch.from_numpy(_effective(a.astype(np.float64), lower, unit)).cuda()
    t = t.T if trans else t
    xt = torch.from_numpy(x.astype(np.float64)).cuda()
    bt = torch.from_numpy(b.astype(np.float64)).cuda()
    res = float(torch.linalg.norm(t @ xt - bt) / (torch.linalg.norm(t) * torch.linalg.norm(xt) + torch.linalg.norm(bt)))
    assert res <= 4 * n * EPS[dtype], f"residual {res:.3g}"


@pytest.mark.parametrize("dtype", ["float32", "float64"])
def test_strided_and_broadcast_operands(aes, dtype):
    """A.T, negative steps and a broadcast right-hand side are read in place."""
    aesara, at, L = aes
    from aesara.tensor.extra_ops import broadcast_to
    from aesara.tensor.slinalg import cho_solve, cholesky, solve, solve_triangular

    n = 129
    a = _spd(2 * n, 50.0, seed=5).astype(dtype)
    A, c = at.matrix("A", dtype=dtype), at.vector("c", dtype=dtype)
    Av = A[::-2, ::-2]
    Bb = broadcast_to(c[:, None], (n, 5))
    Lv = cholesky(Av)
    outs = [solve_triangular(Lv.T, Bb, lower=False, trans=1), solve(Av, Bb, assume_a="pos"),
            cho_solve((Lv, True), c[::-1])]
    f = aesara.function([A, c], outs, mode=L.mode())
    cv = np.random.default_rng(6).standard_normal(n).astype(dtype)
    got = f(a, cv)
    av = a[::-2, ::-2].astype(np.float64)
    bb = np.broadcast_to(cv[:, None], (n, 5)).astype(np.float64)
    lt = np.linalg.cholesky(av)
    want = [scipy.linalg.solve_triangular(lt.T, bb, lower=False, trans=1), scipy.linalg.solve(av, bb, assume_a="pos"),
            scipy.linalg.cho_solve((lt, True), cv[::-1].astype(np.float64))]
    tol = 1e-3 if dtype == "float32" else 1e-10
    for g, w in zip(got, want):
        assert g.dtype == np.dtype(dtype)
        np.testing.assert_allclose(g, w, rtol=tol, atol=tol * np.max(np.abs(w)))


def test_empty_operands(aes):
    aesara, at, L = aes
    from aesara.tensor.slinalg import Cholesky, cho_solve, solve, solve_triangular

    A, B = at.dmatrix("A"), at.dmatrix("B")
    f = aesara.function([A, B], [Cholesky()(A), solve_triangular(A, B, lower=True), cho_solve((A, True), B),
                                 solve(A, B, assume_a="pos")], mode=L.mode())
    for n, k in ((0, 0), (0, 3), (4, 0)):
        a = np.eye(n) * 2.0
        outs = f(a, np.ones((n, k)))
        assert outs[0].shape == (n, n) and outs[0].dtype == np.float64
        for o in outs[1:]:
            assert o.shape == (n, k) and o.dtype == np.float64


# -- error semantics -------------------------------------------------------------------------------
def test_error_semantics(aes):
    aesara, at, L = aes
    from aesara.tensor.slinalg import Cholesky, cho_solve, solve, solve_triangular

    A, b = at.dmatrix("A"), at.dvector("b")
    n = 200
    spd = _spd(n, 10.0, seed=3)
    bad = spd.copy()
    bad[150, 150] = -5.0  # not positive definite at the 151st leading minor or before
    raise_f = aesara.function([A], Cholesky()(A), mode=L.mode())
    nan_f = aesara.function([A], Cholesky(on_error="nan")(A), mode=L.mode())
    with pytest.raises(np.linalg.LinAlgError, match="leading minor"):
        raise_f(bad)
    out = nan_f(bad)
    assert out.shape == (n, n) and np.all(np.isnan(out))
    # a NaN anywhere, even in the triangle that is not read, is a ValueError under both modes
    nanin = spd.copy()
    nanin[0, 5] = np.nan
    for f in (raise_f, nan_f):
        with pytest.raises(ValueError):
            f(nanin)
    np.testing.assert_allclose(raise_f(spd), np.linalg.cholesky(spd), rtol=1e-10, atol=1e-12)

    tri = _tri(n, True, False, seed=4, dtype="float64")
    rhs = np.random.default_rng(4).standard_normal(n)
    checked = aesara.function([A, b], solve_triangular(A, b, lower=True), mode=L.mode())
    unchecked = aesara.function([A, b], solve_triangular(A, b, lower=True, check_finite=False), mode=L.mode())
    tnan = tri.copy()
    tnan[3, 100] = np.nan  # upper triangle: not read
    with pytest.raises(ValueError):
        checked(tnan, rhs)
    np.testing.assert_allclose(unchecked(tnan, rhs), scipy.linalg.solve_triangular(tri, rhs, lower=True), rtol=1e-10)
    bnan = rhs.copy()
    bnan[10] = np.nan
    with pytest.raises(ValueError):
        checked(tri, bnan)
    x = unchecked(tri, bnan)
    assert not np.any(np.isnan(x[:10])) and np.all(np.isnan(x[10:]))
    zero = tri.copy()
    zero[77, 77] = 0.0
    with pytest.raises(np.linalg.LinAlgError, match="77"):
        checked(zero, rhs)
    with pytest.raises(np.linalg.LinAlgError):
        unchecked(zero, rhs)
    # cho_solve does not test the diagonal; solve(pos) raises for a matrix that is not positive definite
    cs = aesara.function([A, b], cho_solve((A, True), b, check_finite=False), mode=L.mode())
    assert not np.all(np.isfinite(cs(zero, rhs)))
    sp = aesara.function([A, b], solve(A, b, assume_a="pos"), mode=L.mode())
    with pytest.raises(np.linalg.LinAlgError):
        sp(bad, rhs)
    with pytest.raises(ValueError):
        sp(nanin, rhs)


# -- Gaussian process ------------------------------------------------------------------------------
def _gp(aes, dtype):
    aesara, at, L = aes
    from aesara.tensor.slinalg import cholesky, solve_triangular

    X, y = at.matrix("X", dtype=dtype), at.vector("y", dtype=dtype)
    ell, noise = at.scalar("ell", dtype=dtype), at.scalar("noise", dtype=dtype)
    Z = X / ell
    sq = at.sum(Z ** 2, axis=1)
    K = at.exp(-0.5 * (sq[:, None] + sq[None, :] - 2.0 * at.dot(Z, Z.T))) + noise * at.eye(X.shape[0])
    Lk = cholesky(K)
    alpha = solve_triangular(Lk.T, solve_triangular(Lk, y, lower=True), lower=False)
    nll = 0.5 * at.dot(y, alpha) + at.sum(at.log(at.diag(Lk)))
    return [X, y, ell, noise], [nll] + list(aesara.grad(nll, [ell, noise, y]))


def _gp_truth(Xv, yv, ell, noise):
    Z = Xv / ell
    d2 = ((Z[:, None, :] - Z[None, :, :]) ** 2).sum(-1)
    E = np.exp(-0.5 * d2)
    K = E + noise * np.eye(len(yv))
    Lk = np.linalg.cholesky(K)
    alpha = scipy.linalg.cho_solve((Lk, True), yv)
    Kinv = scipy.linalg.cho_solve((Lk, True), np.eye(len(yv)))
    W = 0.5 * (Kinv - np.outer(alpha, alpha))  # d nll / dK
    dK_dell = E * d2 / ell
    return [0.5 * yv @ alpha + np.sum(np.log(np.diag(Lk))), np.sum(W * dK_dell), np.trace(W), alpha]


@pytest.mark.parametrize("dtype", ["float32", "float64"])
def test_gp_likelihood_and_gradients(aes, dtype):
    aesara, at, L = aes
    ins, outs = _gp(aes, dtype)
    f = aesara.function(ins, outs, mode=L.mode())
    r = np.random.default_rng(41)
    n = 260
    Xv, yv = r.standard_normal((n, 2)), r.standard_normal(n)
    got = f(Xv.astype(dtype), yv.astype(dtype), np.asarray(1.5, dtype), np.asarray(0.05, dtype))
    want = _gp_truth(Xv.astype(dtype).astype(np.float64), yv.astype(dtype).astype(np.float64), 1.5,
                     float(np.asarray(0.05, dtype)))
    tol = 1e-2 if dtype == "float32" else 1e-9
    for k, (g, w) in enumerate(zip(got, want)):
        err = np.max(np.abs(np.asarray(g, np.float64) - w)) / max(np.max(np.abs(w)), 1e-30)
        assert err < tol, f"output {k}: normwise error {err:.3g}"


def test_gp_through_check_function(aes):
    from aesara_b200.debug import check_function

    ins, outs = _gp(aes, "float64")
    r = np.random.default_rng(42)
    vals = [r.standard_normal((90, 2)), r.standard_normal(90), np.float64(1.2), np.float64(0.1)]
    report = check_function(ins, outs, vals)
    assert report


# -- launch paths ----------------------------------------------------------------------------------
def _updates():
    from aesara_b200.runtime import lib

    return lib.load().ab_linalg_update_count(1), lib.load().ab_linalg_update_count(0)


@pytest.mark.parametrize("n, tc", [(1024, True), (1027, False), (1536, True), (1534, False)])
def test_update_path_follows_the_pitch(aes, n, tc):
    aesara, at, L = aes
    from aesara.tensor.slinalg import solve_triangular

    a = _spd(n, 1e3, seed=n).astype("float32")
    tc0, simt0 = _updates()
    Lf = _chol_fn(aes, "float32", True, "contiguous")(a)
    tc1, simt1 = _updates()
    # the last updates are too small for the tensor-core tiles and run on the CUDA cores anyway
    assert (tc1 > tc0) == tc and (simt1 > simt0 or tc)
    _check_factor(Lf, a.astype(np.float64), True, "float32")
    A, B = at.fmatrix("A"), at.fmatrix("B")
    f = aesara.function([A, B], solve_triangular(A, B, lower=True), mode=L.mode())
    b = np.random.default_rng(1).standard_normal((n, n)).astype("float32")
    x = f(Lf, b)
    tc2, simt2 = _updates()
    assert (tc2 > tc1) == tc and (simt2 > simt1 or tc)
    res = np.linalg.norm(Lf.astype(np.float64) @ x - b) / (np.linalg.norm(Lf) * np.linalg.norm(x) + np.linalg.norm(b))
    assert res <= 4 * n * EPS["float32"]


# -- CUDA graphs -----------------------------------------------------------------------------------
def test_cuda_graph_mode_returns_the_eager_results(aes):
    """Graph replays need device-resident arguments.  A node that checks its errors reads the
    status word back, so its program stays eager; one that checks nothing is captured."""
    aesara, at, L = aes
    from aesara.tensor.slinalg import cho_solve, cholesky, solve_triangular

    from aesara_b200.runtime.device import DeviceArray

    A, b = at.dmatrix("A"), at.dvector("b")
    a, v = _spd(300, 100.0, seed=9), np.random.default_rng(9).standard_normal(300)
    c = np.linalg.cholesky(a)
    Lk = cholesky(A)
    cases = [([A, b], [Lk, solve_triangular(Lk, b, lower=True)], (a, v), False),
             ([A, b], [cho_solve((A, True), b, check_finite=False)], (c, v), True)]
    for ins, outs, vals, captured in cases:
        eager = aesara.function(ins, outs, mode=L.mode())
        graphed = aesara.function(ins, outs, mode=L.mode(device_outputs=True, cuda_graph=True))
        graphed.trust_input = True
        dev = [DeviceArray.from_numpy(x) for x in vals]
        want = eager(*vals)
        for _ in range(4):
            got = graphed(*dev)
            for g, e in zip(got, want):
                np.testing.assert_array_equal(g.to_numpy(), e)
        assert graphed.vm._replay is not None
        assert (graphed.vm._replay.replays >= 2) == captured and graphed.vm._replay._uncapturable != captured


# -- reference fixtures ----------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["cho_solve", "cholesky_upper", "gp_nll", "solve_pos", "solve_triangular"])
def test_device_matches_the_reference_fixtures_and_the_oracle(name):
    """The programs of tests/golden/linalg/ on the device against the reference's outputs and the
    oracle's (tests/test_linalg_golden.py pins the oracle on the same fixtures)."""
    from oracle.program_np import run_program
    from tests._cases import assert_matches, uses_blas
    from tests._linalg_cases import load_case

    from aesara_b200.runtime import lib
    from aesara_b200.runtime.vm import ProgramExecutor

    lib.check(lib.load().ab_init(0))
    prog, ins, want = load_case(name)
    before = lib.load().ab_launch_count()
    got = ProgramExecutor(prog)(*[np.array(a) for a in ins])
    assert lib.load().ab_launch_count() > before
    oracle = run_program(prog, [np.array(a) for a in ins])
    blas = uses_blas(prog)
    for k, (g, w, o) in enumerate(zip(got, want, oracle)):
        assert_matches(g, w, blas=blas, what=f"{name} output {k} vs reference")
        assert_matches(g, o, blas=blas, what=f"{name} output {k} vs oracle")
