"""What the batched inverse / sygst / apply tests share (numpy / scipy only): long-double products from given factors, a-priori normwise
bounds for them, the perturbation bounds that gate eigh_batched against scipy, and a restatement of the chunk rule of the five batched
entry points (api.cu), which the GPU tests use to put matrices at chunk edges.

tests/test_batched_sygst_cpu.py checks the chunk rule and that the bounds reject wrong results; tests/test_gpu_batched_sygst.py gates the
batched kernels on them."""
import math
import numpy as np

from batched_reference import LD, U, WORKSPACE_CAP, GRID_MAX, SOLVE_W, gamma, solve_bound, spd_spectrum, graded, ramp_exponents  # noqa: F401


def _ru(x, k):
    return (x + k - 1) // k * k


# ---- chunk rule (api.cu: batched_chunk) ----------------------------------------------------------------------------------------------
def chunk(call, n, batch):
    """matrices per chunk of capital_cholinv_<call>_batched_f64: the workspace holds ld x n doubles per buffer and matrix (ld =
    roundup(n, 16)), 3 buffers for the inverse and 4 for sygst; the products hold the panel T (n x 32) and tri_apply's partials
    (roundup(n, 64) x 32), as the batched solve does"""
    ld = _ru(n, 16)
    per = {"inverse": 3 * ld * n * 8, "sygst": 4 * ld * n * 8, "sygst_ab": 4 * ld * n * 8,
           "apply_rinv": (n + _ru(n, 64)) * SOLVE_W * 8, "apply_r": (n + _ru(n, 64)) * SOLVE_W * 8}[call]
    return min(batch, GRID_MAX, WORKSPACE_CAP // per)


# ---- long-double products from the given FP64 factors ---------------------------------------------------------------------------------
def inverse_ld(rinv):
    r = np.asarray(rinv, dtype=LD)
    return r @ r.T


def sygst_ld(a, f, itype):
    """Rinv^T A Rinv (itype 1, f = Rinv) or R A R^T (itypes 2, 3, f = R) in np.longdouble"""
    fl, al = np.asarray(f, dtype=LD), np.asarray(a, dtype=LD)
    return fl.T @ (al @ fl) if itype == 1 else fl @ (al @ fl.T)


def sygst_half(a, f, itype):
    """M of C = M + M^T (A = U + U^T, U = triu(A) with its diagonal halved), in FP64: the result of a product that drops one operand
    class, which the bounds must reject (it is off by about ||C|| / 2, far above any rounding)"""
    u = np.triu(np.asarray(a, dtype=np.float64))
    u[np.diag_indices_from(u)] *= 0.5
    return f.T @ (u @ f) if itype == 1 else f @ (u @ f.T)


def product_bound(a, f):
    """A-priori bound on ||C - C_ld||_F for the FP64 C of the batched sygst from the factor f (Rinv for itype 1, R for 2 and 3), any
    summation order and tiling.  V = fl(U F) (or fl(F U)) has |dV| <= gamma_n |U| |F|; C = fl(F^T V + V^T F) adds gamma_2n (|F^T| |V| +
    |V^T| |F|), and dV reaches C through F twice.  With || |M| ||_2 <= sqrt(n) ||M||_2 and ||U||_F <= ||A||_F:
    ||dC||_F <= (2 gamma_n + 2 gamma_2n) n ||A||_F ||F||_2^2 to first order, doubled for the higher orders."""
    n = a.shape[0]
    return 2 * (2 * gamma(n) + 2 * gamma(2 * n)) * n * float(np.linalg.norm(a)) * float(np.linalg.norm(f, 2)) ** 2


def inverse_product_bound(rinv):
    """A-priori bound on ||Ainv - Rinv Rinv^T||_F: one product, |dP| <= gamma_n |Rinv| |Rinv^T|, n gamma_n ||Rinv||_2^2 in norm, doubled"""
    n = rinv.shape[0]
    return 2 * n * gamma(n) * float(np.linalg.norm(rinv, 2)) ** 2


def inverse_residual_bound(a):
    """A-priori bound on ||A Ainv - I||_F / sqrt(n) for Ainv = Rinv Rinv^T from the CholInv factor of a.  Ainv is the batched solve's
    X = Rinv (Rinv^T B) at B = I with one product instead of two, so ||Ainv - A^-1||_F <= solve_bound(a) ||A^-1||_F, and
    ||A Ainv - I||_F <= ||A||_2 ||Ainv - A^-1||_F.  Grows as kappa^3: gated at kappa = 10 only."""
    n = a.shape[0]
    return float(np.linalg.norm(a, 2)) * float(np.linalg.norm(np.linalg.inv(a))) * solve_bound(a) / math.sqrt(n)


# ---- eigh_batched against scipy --------------------------------------------------------------------------------------------------------
class EighBounds:
    """Perturbation bounds for the generalized eigenpairs (w, X) of eigh_batched on the pencil (a, b), b = R^T R with 2-norm condition
    number kappa.  The computed C is the exact reduction of a nearby problem: the factor is backward stable (R^T R = b + dB,
    ||dB|| <= c n u ||b||), Rinv is R^-1 up to c n u kappa(R) (trtri), and sygst adds product_bound, which is c n u ||A|| ||F||^2 =
    c n u ||A|| ||b^-1|| for itype 1 and c n u ||A|| ||b|| for itypes 2 and 3 (S below); eigh adds c n u ||C||.  Eigenvalues (Weyl, on
    C's symmetric perturbation, and the relative shift kappa(b) n u from the factor): |w_i - w_ref_i| <= 20 n u (S + |w_i| kappa +
    max|w|).  Residuals and B-orthonormality are mapped back through F (at most kappa), so each bound carries a factor kappa:
      itype 1: ||A X - B X W||_F, itype 2: ||A B X - X W||_F, itype 3: ||B A X - X W||_F  <= 10 n u (S' + max|w|) kappa ||X||_F,
               S' = ||A|| + max|w| ||b|| for itype 1 and ||A|| ||b|| + max|w| for 2 and 3;
      ||X^T B X - I||_F (itypes 1, 2), ||X^T B^-1 X - I||_F (itype 3)  <= 10 n^1.5 u kappa."""

    def __init__(self, a, b, itype):
        self.n, self.itype = a.shape[0], itype
        ev = np.linalg.eigvalsh(b)
        self.bnorm, self.kappa = float(ev[-1]), float(ev[-1] / ev[0])
        self.anorm = float(np.linalg.norm(a, 2))
        self.S = self.anorm / float(ev[0]) if itype == 1 else self.anorm * self.bnorm

    def eigenvalues(self, w):
        wmax = float(np.abs(w).max())
        return 20 * self.n * U * (self.S + np.abs(w) * self.kappa + wmax)

    def residual(self, w, x):
        wmax = float(np.abs(w).max())
        s = self.anorm + wmax * self.bnorm if self.itype == 1 else self.anorm * self.bnorm + wmax
        return 10 * self.n * U * s * self.kappa * float(np.linalg.norm(x))

    def orthonormality(self):
        return 10 * self.n ** 1.5 * U * self.kappa


def eigh_residual(a, b, w, x, itype):
    """||A X - B X W||_F (itype 1), ||A B X - X W||_F (2), ||B A X - X W||_F (3), evaluated in FP64 (its rounding, n u times the bound's
    scale, is a factor 10 kappa below the bound)"""
    lhs = a @ x if itype == 1 else a @ (b @ x) if itype == 2 else b @ (a @ x)
    rhs = (b @ x) * w if itype == 1 else x * w
    return float(np.linalg.norm(lhs - rhs))


def eigh_orthonormality(b, x, itype):
    """||X^T B X - I||_F (itypes 1, 2) or ||X^T B^-1 X - I||_F (itype 3), evaluated in FP64 (n u kappa, under the bound)"""
    m = b if itype != 3 else np.linalg.inv(b)
    return float(np.linalg.norm(x.T @ (m @ x) - np.eye(x.shape[1])))
