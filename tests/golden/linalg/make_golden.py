"""Generate the dense linear-algebra fixtures under tests/golden/linalg/ with the REFERENCE itself.

    PYTHONPATH=. python tests/golden/linalg/make_golden.py [name ...]

Same procedure as tests/golden/make_golden.py (whose set-up this script reuses): the reference
rewriter optimises each graph and its C VM evaluates it on seeded inputs; the lowered program goes
to ``<case>.json``, inputs and reference outputs to ``<case>.npz``.  These fixtures need the
slinalg handlers of the oracle (oracle/linalg_np.py) and are checked by tests/test_linalg_golden.py
(CPU) and tests/test_gpu_linalg.py (GPU).
"""

import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
import make_golden as _mg  # noqa: E402  (materialises and activates the reference front-end)

aesara, at = _mg.aesara, _mg.at
CASES = {}


def case(name):
    def deco(fn):
        CASES[name] = fn
        return fn

    return deco


# ---------------------------------------------------------------- dense linear algebra (tensor/slinalg.py)
def _spd(r, n, cond=100.0):
    """A symmetric positive definite matrix with eigenvalues spread over [1, cond]."""
    q, _ = np.linalg.qr(r.standard_normal((n, n)))
    return (q * np.geomspace(1.0, cond, n)) @ q.T


@case("gp_nll")
def _():
    """A Gaussian-process negative log marginal likelihood (squared-exponential kernel) and its
    gradient with respect to the lengthscale, the noise variance and y."""
    from aesara.tensor.slinalg import cholesky, solve_triangular

    X, y = at.dmatrix("X"), at.dvector("y")
    ell, noise = at.dscalar("ell"), at.dscalar("noise")
    Z = X / ell
    sq = at.sum(Z ** 2, axis=1)
    K = at.exp(-0.5 * (sq[:, None] + sq[None, :] - 2.0 * at.dot(Z, Z.T))) + noise * at.eye(X.shape[0])
    L = cholesky(K)
    alpha = solve_triangular(L.T, solve_triangular(L, y, lower=True), lower=False)
    nll = 0.5 * at.dot(y, alpha) + at.sum(at.log(at.diag(L))) + 0.5 * X.shape[0] * np.log(2 * np.pi)
    g_ell, g_noise, g_y = aesara.grad(nll, [ell, noise, y])
    r = np.random.default_rng(31)
    n = 48
    return [X, y, ell, noise], [nll, g_ell, g_noise, g_y], [r.standard_normal((n, 3)), r.standard_normal(n),
                                                            np.float64(1.3), np.float64(0.1)]


@case("solve_triangular")
def _():
    """solve_triangular in the four (lower, trans) combinations on a matrix right-hand side, and
    with unit_diagonal on a vector; the triangle that is not named holds values that must not be read."""
    from aesara.tensor.slinalg import solve_triangular

    A, B, b = at.dmatrix("A"), at.dmatrix("B"), at.dvector("b")
    outs = [solve_triangular(A, B, lower=lo, trans=tr) for lo in (True, False) for tr in (0, 1)]
    outs += [solve_triangular(A, b, lower=True, unit_diagonal=True), solve_triangular(A, b, lower=False, trans=2)]
    r = np.random.default_rng(32)
    n = 40
    a = r.standard_normal((n, n)) * 0.2 + np.diag(r.uniform(1.0, 2.0, n))
    return [A, B, b], outs, [a, r.standard_normal((n, 5)), r.standard_normal(n)]


@case("cho_solve")
def _():
    """cho_solve with the lower factor and with the upper one, matrix and vector right-hand sides."""
    from aesara.tensor.slinalg import cho_solve

    C, B, b = at.dmatrix("C"), at.dmatrix("B"), at.dvector("b")
    outs = [cho_solve((C, True), B), cho_solve((C.T, False), b)]
    r = np.random.default_rng(33)
    n = 37
    return [C, B, b], outs, [np.linalg.cholesky(_spd(r, n)), r.standard_normal((n, 6)), r.standard_normal(n)]


@case("solve_pos")
def _():
    """solve(assume_a="pos") from the upper triangle (the default) and from the lower one."""
    from aesara.tensor.slinalg import solve

    A, B, b = at.dmatrix("A"), at.dmatrix("B"), at.dvector("b")
    outs = [solve(A, B, assume_a="pos"), solve(A, b, assume_a="pos", lower=True)]
    r = np.random.default_rng(34)
    n = 45
    return [A, B, b], outs, [_spd(r, n), r.standard_normal((n, 3)), r.standard_normal(n)]


@case("cholesky_upper")
def _():
    """Cholesky(lower=False) in float32 and float64, and on_error="nan" on a matrix that is not
    positive definite."""
    from aesara.tensor.slinalg import Cholesky

    A32, A64, N = at.fmatrix("A32"), at.dmatrix("A64"), at.dmatrix("N")
    outs = [Cholesky(lower=False)(A32), Cholesky(lower=False)(A64), Cholesky(on_error="nan")(N)]
    r = np.random.default_rng(35)
    n = 33
    a = _spd(r, n, cond=10.0)
    return [A32, A64, N], outs, [a.astype("float32"), _spd(r, n), a - 2.0 * np.eye(n)]


def main(names):
    from aesara_b200.graphs import optimized_program

    for name in names:
        ins, outs, values = CASES[name]()
        prog, f = optimized_program(ins, outs, name=name, linker="cvm")
        ref = f(*values)
        prog.save(os.path.join(HERE, name + ".json"))
        blob = {f"in_{k}": np.asarray(v) for k, v in enumerate(values)}
        blob.update({f"out_{k}": np.asarray(v) for k, v in enumerate(ref)})
        np.savez_compressed(os.path.join(HERE, name + ".npz"), **blob)
        print(f"{name}: {len(prog.nodes)} nodes {prog.op_counts()}")


if __name__ == "__main__":
    main(sys.argv[1:] or list(CASES))
