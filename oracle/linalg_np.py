"""ORACLE (test infrastructure only -- never imported by the product path).

The dense linear-algebra nodes of lowered programs (aesara/tensor/slinalg.py: Cholesky,
SolveTriangular, CholeskySolve, Solve with assume_a="pos") restated with scipy, exactly as the
reference's ``perform`` methods compute them.  Importing this module installs the handlers in
the program interpreter of ``oracle/program_np.py`` (``run_program``).
"""

import numpy as np
import scipy.linalg

from .program_np import _h


@_h("Cholesky")
def _cholesky(node, args, prog):  # aesara/tensor/slinalg.py:64-73
    (x,) = args
    try:
        return scipy.linalg.cholesky(x, lower=node.params["lower"]).astype(x.dtype)
    except scipy.linalg.LinAlgError:
        if node.params["on_error"] == "raise":
            raise
        return (np.zeros(x.shape) * np.nan).astype(x.dtype)


@_h("SolveTriangular")
def _solve_triangular(node, args, prog):  # aesara/tensor/slinalg.py:301-310
    p = node.params
    return scipy.linalg.solve_triangular(args[0], args[1], lower=p["lower"], trans=p["trans"],
                                         unit_diagonal=p["unit_diagonal"], check_finite=p["check_finite"])


@_h("CholeskySolve")
def _cholesky_solve(node, args, prog):  # aesara/tensor/slinalg.py:158-166
    return scipy.linalg.cho_solve((args[0], node.params["lower"]), args[1], check_finite=node.params["check_finite"])


@_h("Solve")
def _solve(node, args, prog):  # aesara/tensor/slinalg.py:388-396, assume_a="pos"
    p = node.params
    return scipy.linalg.solve(a=args[0], b=args[1], lower=p["lower"], check_finite=p["check_finite"], assume_a="pos")
