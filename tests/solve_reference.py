"""numpy restatement of cholinv::solve (capital_cholinv_solve_f64) on the global factors, for the solve tests.

It sits next to the tests rather than in oracle/capital_oracle.py so that the oracle module the existing suites check against stays
as it is; it uses that module's `cholinv` outputs (R, Rinv) and its split rule."""
import numpy as np


def top_split(n: int, complete_inv: bool, split: int, bc_dim: int, d: int = 1):
    """Global split point n1 of the top node when its Rinv12 block was skipped, else None (the same rule as cholinv::invoke,
    cholinv.hpp:92-93,147: a top node that is the base case has the full inverse)."""
    s1 = (n // d) >> split
    if complete_inv or n <= bc_dim or s1 < split:
        return None
    return d * s1


def cholesky_solve(r: np.ndarray, ri: np.ndarray, b: np.ndarray, complete_inv: bool, split: int, bc_dim: int, d: int = 1) -> np.ndarray:
    """X with R^T R X = B from the global R, Rinv of `capital_oracle.cholinv(a, complete_inv, split, bc_dim, d)`.
    Rinv complete: X = Rinv (Rinv^T B).  Rinv12 skipped (split n1):
      Y1 = Rinv11^T B1,  Y2 = Rinv22^T (B2 - R12^T Y1),  X2 = Rinv22 Y2,  X1 = Rinv11 (Y1 - R12 X2)."""
    n = r.shape[0]
    n1 = top_split(n, complete_inv, split, bc_dim, d)
    if n1 is None:
        return ri @ (ri.T @ b)
    b1, b2 = b[:n1], b[n1:]
    ri11, ri22, r12 = ri[:n1, :n1], ri[n1:, n1:], r[:n1, n1:]
    y1 = ri11.T @ b1
    y2 = ri22.T @ (b2 - r12.T @ y1)
    x2 = ri22 @ y2
    x1 = ri11 @ (y1 - r12 @ x2)
    return np.concatenate([x1, x2], axis=0)
