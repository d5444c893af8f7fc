"""numpy restatement of cholinv::inverse (capital_cholinv_inverse_f64) on the global factors, for the inverse tests.

Like solve_reference.py it sits next to the tests, so that the oracle module the existing suites check against stays as it is; it
takes that module's `cholinv` outputs (R, Rinv) and the top-level split rule of solve_reference."""
import numpy as np
from solve_reference import top_split


def rebuild_rinv(r: np.ndarray, ri: np.ndarray, complete_inv: bool, split: int, bc_dim: int, d: int = 1) -> np.ndarray:
    """Rinv with the top-level Rinv12 block filled in where the factor skipped it (complete_inv = 0 and the top node splits at n1),
    by the two products the factor issues for that block (cholinv.hpp:151-155):  T^T = R12^T Rinv11^T,  Rinv12 = -(T^T)^T Rinv22."""
    n1 = top_split(r.shape[0], complete_inv, split, bc_dim, d)
    if n1 is None:
        return ri
    out = ri.copy()
    tt = r[:n1, n1:].T @ ri[:n1, :n1].T
    out[:n1, n1:] = -(tt.T @ ri[n1:, n1:])
    return out


def cholesky_inverse(r: np.ndarray, ri: np.ndarray, complete_inv: bool, split: int, bc_dim: int, d: int = 1) -> np.ndarray:
    """A^-1 = Rinv Rinv^T from the global factors of `capital_oracle.cholinv(a, complete_inv, split, bc_dim, d)`."""
    full = rebuild_rinv(r, ri, complete_inv, split, bc_dim, d)
    return full @ full.T
