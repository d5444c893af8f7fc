"""numpy restatement of cholinv::sygst for itype 2 and 3 (capital_cholinv_sygst_ab_f64) on the global factor R, for the sygst_ab tests.

A B x = lambda x and B A x = lambda x with B = R^T R both reduce to C = R A R^T.  The library forms it in n^3 flops by LAPACK's split
A = U + U^T, U = triu(A) with its diagonal halved: W = R U (upper triangular), then C = W R^T + R W^T, upper half only."""
import numpy as np
from sygst_reference import U, u_transpose


def sygst_ab(a: np.ndarray, r: np.ndarray) -> np.ndarray:
    """C = R A R^T in the library's n^3 form, mirrored to a full C.  Only A's lower triangle is read."""
    w = np.triu(r @ u_transpose(a).T)  # upper triangular: R and U are
    c = np.triu(w @ r.T + r @ w.T)
    return c + np.triu(c, 1).T


def bound(a: np.ndarray, r: np.ndarray) -> np.ndarray:
    """Elementwise first-order rounding bound of the n^3 form: each entry of C is a sum of products of three factors over at most 2n
    terms per product, so |C - C_exact| <= 2 n u (|R| |A| |R|^T) to first order.  The numpy model stays 10x inside it
    (test_sygst_ab_cpu), and the GPU results are held to it."""
    n = a.shape[0]
    m = np.abs(r)
    return 2 * n * U * (m @ np.abs(a) @ m.T)


def dsygst_full(a: np.ndarray, r: np.ndarray, itype: int) -> np.ndarray:
    """LAPACK's dsygst (itype 2 or 3, upper) on the upper R of B = R^T R, mirrored to a full matrix"""
    from scipy.linalg import lapack
    c, info = lapack.dsygst(a, r, itype=itype, lower=0)
    assert info == 0
    c = np.triu(c)
    return c + np.triu(c, 1).T
