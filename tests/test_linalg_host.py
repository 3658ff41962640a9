"""CPU: dense linear algebra (aesara/tensor/slinalg.py) -- the lowering of Cholesky,
SolveTriangular, CholeskySolve and Solve(assume_a="pos"), the refusals, the oracle against
scipy on the error cases, the shard-plan refusal and the spill-free sm_90a build of
csrc/ab_linalg.cu.  The device results are checked in tests/test_gpu_linalg.py."""
import os
import re
import subprocess

import numpy as np
import pytest
import scipy.linalg

from aesara_b200.compat import bootstrap

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
needs_ref = pytest.mark.skipif(not bootstrap.available(), reason="reference front-end not available")


def _compile(inputs, outputs):
    aesara = bootstrap.load_aesara()
    from aesara.compile.mode import Mode
    from aesara.graph.rewriting.db import RewriteDatabaseQuery

    from aesara_b200.lower import lower_fgraph

    f = aesara.function(inputs, outputs, mode=Mode(linker="py", optimizer=RewriteDatabaseQuery(include=["fast_run"])))
    return f, lower_fgraph(f.maker.fgraph)


@needs_ref
def test_the_four_ops_lower_with_their_parameters():
    bootstrap.load_aesara()
    import aesara.tensor as at
    from aesara.tensor.slinalg import Cholesky, CholeskySolve, Solve, SolveTriangular

    A, B, v, i = at.dmatrix("A"), at.fmatrix("B"), at.fvector("v"), at.imatrix("i")
    outs = [Cholesky(lower=False, on_error="nan")(A), SolveTriangular(trans="C", lower=True, unit_diagonal=True)(A, v),
            SolveTriangular(trans=1, check_finite=False)(B, B), CholeskySolve(lower=False)(B, v),
            Solve(assume_a="pos", lower=True, check_finite=False)(i, B)]
    _, prog = _compile([A, B, v, i], outs)
    got = {n.op: [] for n in prog.nodes}
    for n in prog.nodes:
        got[n.op].append((n.params, prog.vars[n.outputs[0]].dtype))
    assert got["Cholesky"] == [({"lower": False, "on_error": "nan"}, "float64")]
    assert sorted(got["SolveTriangular"], key=str) == sorted([
        ({"lower": True, "trans": 1, "unit_diagonal": True, "check_finite": True}, "float64"),
        ({"lower": False, "trans": 1, "unit_diagonal": False, "check_finite": False}, "float32")], key=str)
    assert got["CholeskySolve"] == [({"lower": False, "check_finite": True}, "float32")]
    # an integer operand makes the output float64 (make_node asks scipy.linalg.solve)
    assert got["Solve"] == [({"lower": True, "check_finite": False}, "float64")]


@needs_ref
def test_refusals_name_the_op_and_the_reason():
    bootstrap.load_aesara()
    import aesara.tensor as at
    from aesara.tensor.nlinalg import MatrixInverse
    from aesara.tensor.slinalg import Cholesky, Solve

    from aesara_b200.lower import UnsupportedOp

    A, b, i = at.dmatrix("A"), at.dvector("b"), at.lmatrix("i")
    with pytest.raises(UnsupportedOp, match="Cholesky of a int64 matrix.*truncates"):
        _compile([i], [Cholesky()(i)])
    for assume in ("gen", "sym", "her"):
        with pytest.raises(UnsupportedOp, match=f"Solve\\(assume_a='{assume}'\\).*LU / LDL"):
            _compile([A, b], [Solve(assume_a=assume)(A, b)])
    # every other slinalg / nlinalg Op fails as before, through lower_apply
    with pytest.raises(UnsupportedOp, match="no device implementation for Op MatrixInverse"):
        _compile([A], [MatrixInverse()(A)])


@needs_ref
def test_shardplan_refuses_factorisations():
    bootstrap.load_aesara()
    import aesara.tensor as at
    from aesara.tensor.slinalg import cholesky

    from aesara_b200 import shardplan

    X = at.dmatrix("X")
    _, prog = _compile([X], [cholesky(X.T @ X) * 2.0])
    with pytest.raises(shardplan.ReplicasOnly, match="not a row-wise batch map"):
        shardplan.analyse(prog, [0])
    with pytest.raises(shardplan.ReplicasOnly):
        shardplan.infer_sharded_inputs(prog)


@needs_ref
def test_oracle_restates_the_reference_on_the_error_cases():
    """run_program raises what the reference's perform raises, and agrees with it otherwise."""
    bootstrap.load_aesara()
    import aesara.tensor as at
    from aesara.tensor.slinalg import Cholesky, cho_solve, solve, solve_triangular

    import oracle.linalg_np  # noqa: F401  (the slinalg handlers of run_program)
    from oracle.program_np import run_program

    A, b = at.dmatrix("A"), at.dvector("b")
    r = np.random.default_rng(0)
    n = 12
    m = r.standard_normal((n, n))
    spd = m @ m.T + n * np.eye(n)
    notpd = spd - 100 * np.eye(n)
    nan = spd.copy()
    nan[0, n - 1] = np.nan  # the upper triangle: not read, still checked
    zero = np.tril(spd)
    zero[4, 4] = 0.0
    v = r.standard_normal(n)
    cases = [
        (Cholesky()(A), [notpd], np.linalg.LinAlgError),
        (Cholesky()(A), [nan], ValueError),
        (Cholesky(on_error="nan")(A), [nan], ValueError),
        (solve_triangular(A, b, lower=True), [zero, v], np.linalg.LinAlgError),
        (solve_triangular(A, b, lower=True, check_finite=False), [zero, v], np.linalg.LinAlgError),
        (solve_triangular(A, b, lower=True), [nan, v], ValueError),
        (solve(A, b, assume_a="pos"), [notpd, v], np.linalg.LinAlgError),
        (solve(A, b, assume_a="pos"), [nan, v], ValueError),
    ]
    for out, vals, exc in cases:
        ins = [A] if len(vals) == 1 else [A, b]
        f, prog = _compile(ins, [out])
        with pytest.raises(exc):
            f(*vals)
        with pytest.raises(exc):
            run_program(prog, vals)
    # on_error="nan" gives an all-NaN factor; check_finite=False lets NaN through; cho_solve does
    # not test the diagonal
    for out, vals in ((Cholesky(on_error="nan")(A), [notpd]),
                      (solve_triangular(A, b, lower=True, check_finite=False), [nan.T.copy(), v]),
                      (solve_triangular(A, b, lower=False, check_finite=False), [nan, v]),
                      (cho_solve((A, True), b, check_finite=False), [zero, v]),
                      (solve(A, b, assume_a="pos", lower=True, check_finite=False), [nan, v])):
        ins = [A] if len(vals) == 1 else [A, b]
        f, prog = _compile(ins, [out])
        with np.errstate(all="ignore"):
            (want,) = f(*vals)
            (got,) = run_program(prog, vals)
        np.testing.assert_array_equal(np.isnan(got), np.isnan(want))
        np.testing.assert_allclose(got, want, rtol=1e-12, equal_nan=True)
    assert np.all(np.isnan(run_program(_compile([A], [Cholesky(on_error="nan")(A)])[1], [notpd])[0]))
    assert np.allclose(run_program(_compile([A], [Cholesky(lower=False)(A)])[1], [spd])[0],
                       scipy.linalg.cholesky(spd, lower=False))


def test_linalg_kernels_compile_for_sm90a_without_spills(tmp_path):
    nvcc = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "nvcc")
    src = os.path.join(ROOT, "aesara_b200", "csrc", "ab_linalg.cu")
    r = subprocess.run([nvcc, "-c", src, "-o", str(tmp_path / "l.o"), "-gencode", "arch=compute_90a,code=sm_90a",
                        "-O3", "-std=c++17", "-Xcompiler", "-fPIC", "-Xptxas", "-v"],
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert r.returncode == 0, r.stdout
    kernels = re.findall(r"Compiling entry function '(\w+)' for 'sm_90a'", r.stdout)
    # check_finite, zero_diagonal, copy, nan_fill, potrf_diag, trsm_diag, trsv_diag, trsv_update x f32 / f64
    assert len(kernels) == 16, r.stdout
    spills = re.findall(r"(\d+) bytes spill stores, (\d+) bytes spill loads", r.stdout)
    assert len(spills) == 16 and all(s == ("0", "0") for s in spills), r.stdout
    frames = re.findall(r"(\d+) bytes stack frame", r.stdout)
    assert all(f == "0" for f in frames), r.stdout
