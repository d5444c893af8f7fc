"""numpy restatement of shifted CholeskyQR3 (cacqr num_iter = 3), built on the oracle's CholInv (oracle/capital_oracle.py).

Sweep 1 factors the shifted Gram matrix G + s I, s = 11 (m n + n (n + 1)) 2^-53 trace(G); sweeps 2 and 3 are CholeskyQR2 on
Q1 = A R1^-1; R = R3 (R2 R1), multiplied in that order as the library does.  Each sweep's R and R^-1 come from the oracle's
recursive cholinv with the given base case -- the explicit inverse the GPU path applies -- or, with bc = None, from LAPACK potrf +
trtri as in the oracle's CholeskyQR2."""
import numpy as np
import scipy.linalg as sla
from oracle import capital_oracle as co


def shift_coef(m, n):
    return 11.0 * (m * n + n * (n + 1)) * 2.0 ** -53


def _chol_inv(g, bc, c=1):
    if bc is None:
        r = sla.cholesky(g + np.triu(g, 1).T, lower=False, check_finite=False)
        rinv, info = sla.lapack.dtrtri(r, lower=0, unitdiag=0)
        assert info == 0
        return np.triu(r), np.triu(rinv)
    return co.cholinv(g, True, 1, bc, c)


def scqr3(a, bc=None, c=1):
    """(Q, R) of shifted CholeskyQR3 on the global m x n matrix a.  c > 1: the 3D / tunable grids' CholInv (process-face edge c,
    base case co.bc_dimension's global size bc)."""
    m, n = a.shape
    q = np.array(a, dtype=np.float64)
    rs = []
    for it in range(3):
        g = np.triu(q.T @ q)
        if it == 0:
            g[np.diag_indices(n)] += shift_coef(m, n) * np.trace(g)
        r, ri = _chol_inv(g, bc, c)
        q = q @ ri
        rs.append(r)
    return q, np.triu(rs[2] @ np.triu(rs[1] @ rs[0]))


def ill_conditioned(m, n, kappa, seed):
    """A = U diag(logspace(0, -log10 kappa, n)) V^T with random orthogonal U (m x n) and V (n x n)."""
    rng = np.random.default_rng(seed)
    u, _ = np.linalg.qr(rng.standard_normal((m, n)))
    v, _ = np.linalg.qr(rng.standard_normal((n, n)))
    return (u * np.logspace(0, -np.log10(kappa), n)) @ v.T
