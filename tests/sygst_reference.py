"""numpy restatement of cholinv::sygst (capital_cholinv_sygst_f64) on the global factors, for the sygst tests.

Like inverse_reference.py it sits next to the tests; it takes the oracle module's `cholinv` outputs (R, Rinv) and rebuilds a skipped
top-level Rinv12 with inverse_reference.rebuild_rinv."""
import numpy as np
from inverse_reference import rebuild_rinv

U = 2.0 ** -53  # unit roundoff of FP64


def u_transpose(a: np.ndarray) -> np.ndarray:
    """U^T for the split A = U + U^T, U = triu(A) with its diagonal halved: A's lower triangle with the diagonal halved (exact)"""
    ut = np.tril(a)
    ut[np.diag_indices_from(ut)] *= 0.5
    return ut


def sygst(a: np.ndarray, r: np.ndarray, ri: np.ndarray, complete_inv: bool, split: int, bc_dim: int, d: int = 1) -> np.ndarray:
    """C = Rinv^T A Rinv in the library's n^3 form: V = (U^T)^T Rinv, C_upper = triu(Rinv^T V + V^T Rinv), mirrored to a full C.
    Only A's lower triangle is read."""
    full = rebuild_rinv(r, ri, complete_inv, split, bc_dim, d)
    v = np.triu(u_transpose(a).T @ full)  # upper triangular: U and Rinv are
    c = np.triu(full.T @ v + v.T @ full)
    return c + np.triu(c, 1).T


def bound(a: np.ndarray, ri: np.ndarray) -> np.ndarray:
    """Elementwise first-order rounding bound of the n^3 form: each entry of C is a sum of products of three factors over at most 2n
    terms per product, so |C - C_exact| <= 2 n u (|Rinv|^T |A| |Rinv|) to first order.  The numpy model stays 10x inside it (test_sygst_cpu),
    and the GPU results are held to it."""
    n = a.shape[0]
    m = np.abs(ri)
    return 2 * n * U * (m.T @ np.abs(a) @ m)


def dsygst_full(a: np.ndarray, r: np.ndarray) -> np.ndarray:
    """LAPACK's dsygst (itype 1, upper) on the upper R of B = R^T R, mirrored to a full matrix"""
    from scipy.linalg import lapack
    c, info = lapack.dsygst(a, r, itype=1, lower=0)
    assert info == 0
    c = np.triu(c)
    return c + np.triu(c, 1).T
