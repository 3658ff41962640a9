"""CPU: the oracle's slinalg handlers (oracle/linalg_np.py) reproduce the reference outputs stored
in tests/golden/linalg/: a Gaussian-process likelihood with its gradients, solve_triangular in
every (lower, trans) case and with unit_diagonal, cho_solve, solve(assume_a="pos") and
Cholesky(lower=False) with on_error="nan".  The device runs the same fixtures in
tests/test_gpu_linalg.py."""
import numpy as np
import pytest

from oracle.program_np import run_program
from tests._cases import assert_matches, uses_blas
from tests._linalg_cases import case_names, load_case


def test_the_fixtures_are_there():
    assert case_names() == ["cho_solve", "cholesky_upper", "gp_nll", "solve_pos", "solve_triangular"]


@pytest.mark.parametrize("name", case_names())
def test_oracle_matches_reference(name):
    prog, ins, want = load_case(name)
    got = run_program(prog, [np.array(a) for a in ins])
    assert len(got) == len(want)
    blas = uses_blas(prog)
    for k, (g, w) in enumerate(zip(got, want)):
        assert_matches(g, w, blas=blas, what=f"{name} output {k}")
