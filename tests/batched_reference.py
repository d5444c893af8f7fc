"""What the batched reference tests share (numpy / scipy only): extended-precision QR, least-squares and SPD-solve references, a-priori
error bounds for batched CholeskyQR and the batched CholInv solve, the first failing pivot in LAPACK's numbering, and a restatement
of the chunk rules of the four batched entry points (api.cu, dist.cu), which the GPU tests use to put matrices at chunk edges.

tests/test_batched_reference_cpu.py checks the references and the bounds against LAPACK on the CPU; tests/test_gpu_batched_reference.py
gates the batched kernels on them.

np.longdouble is the x87 80-bit format here (u = 2^-64, 2^11 times below FP64's) and runs at about 0.1 Gflop/s in products, so every
reference is kept to a few times 10^8 flops and the GPU tests cache them per module."""
import math
import numpy as np

from grid_edges_reference import Bounds, chol_ld  # noqa: F401  (re-exported for the tests)
from conditioning_reference import chol_ratio, inv_ratio, spd_spectrum, graded, ramp_exponents, scaled  # noqa: F401

U = 2.0 ** -53  # unit roundoff of FP64
LD = np.longdouble


# ---- extended-precision references ----------------------------------------------------------------------------------------------
def _householder(w, ncols):
    """Householder QR of the first `ncols` columns of the long double array w (m x k, k >= ncols), in place; every column of w gets
    the reflectors, so the trailing columns end as Q^T w.  Returns the signs that make R's diagonal positive."""
    m = w.shape[0]
    sign = np.ones(ncols, dtype=LD)
    for j in range(min(ncols, m)):
        x = w[j:, j]
        alpha = np.sqrt(x @ x)
        if alpha == 0:
            continue
        v = x.copy()
        s = 1 if v[0] >= 0 else -1
        v[0] += s * alpha
        beta = 2 / (v @ v)
        w[j:, j:] -= np.outer(beta * v, v @ w[j:, j:])
        sign[j] = -s  # w[j, j] = -s alpha
    return sign


def qr_ld(a, want_q=True):
    """(Q, R) of the m x n matrix a (m >= n) in np.longdouble: R by Householder QR with a positive diagonal, Q = A R^-1 by forward
    substitution (Q is None without want_q).  About 2 m n^2 flops for R and m n^2 more for Q."""
    m, n = a.shape
    w = np.array(a, dtype=LD)
    sign = _householder(w, n)
    r = np.triu(w[:n]) * sign[:, None]
    if not want_q:
        return None, r
    al = np.asarray(a, dtype=LD)
    q = np.empty((m, n), dtype=LD)
    for j in range(n):
        q[:, j] = (al[:, j] - q[:, :j] @ r[:j, j]) / r[j, j]
    return q, r


def lstsq_ld(a, b):
    """(X, residual norms): argmin ||A X - B||_2 per column in np.longdouble, from Householder QR of [A B] (Q^T B through the
    reflectors, then back substitution with R); the residual norm of column j is ||(Q^T B)[n:, j]||."""
    m, n = a.shape
    b2 = b.reshape(m, -1)
    w = np.hstack([np.asarray(a, dtype=LD), np.asarray(b2, dtype=LD)])
    sign = _householder(w, n)
    r = np.triu(w[:n, :n]) * sign[:, None]
    c = w[:n, n:] * sign[:, None]
    x = _back(r, c)
    res = np.sqrt((w[n:, n:] ** 2).sum(axis=0))
    return x.reshape((n,) + b.shape[1:]), res


def _back(r, c):
    """R^-1 C by back substitution (R upper, long double)"""
    n = r.shape[0]
    x = np.zeros(c.shape, dtype=LD)
    for i in range(n - 1, -1, -1):
        x[i] = (c[i] - r[i, i + 1:] @ x[i + 1:]) / r[i, i]
    return x


def solve_ld(a, b):
    """A^-1 B in np.longdouble from chol_ld's R: forward substitution with R^T, then back substitution with R"""
    r = chol_ld(a)[0]
    n = a.shape[0]
    c = np.asarray(b, dtype=LD).reshape(n, -1)
    y = np.zeros(c.shape, dtype=LD)
    for i in range(n):
        y[i] = (c[i] - r[:i, i] @ y[:i]) / r[i, i]
    return _back(r, y).reshape(b.shape)


def first_bad_pivot(a):
    """LAPACK dpotrf's INFO for the upper triangle of a (the lower one is not read): the 1-based column of the first pivot that is
    NaN or not positive (reference dpotrf2 / dpotf2 test `AJJ.LE.ZERO .OR. DISNAN(AJJ)`), 0 when the factor completes.  Long double
    row-oriented Cholesky as in chol_ld, stopped at the first bad pivot."""
    n = a.shape[0]
    w = np.triu(np.asarray(a, dtype=LD))
    r = np.zeros((n, n), dtype=LD)
    for i in range(n):
        v = w[i, i:] - r[:i, i] @ r[:i, i:]
        if not v[0] > 0:
            return i + 1
        r[i, i] = np.sqrt(v[0])
        r[i, i + 1:] = v[1:] / r[i, i]
    return 0


# ---- a-priori bounds ----------------------------------------------------------------------------------------------------------------
def gamma(k):
    return k * U / (1 - k * U)


class QRBounds:
    """A-priori rounding bounds of batched CholeskyQR (num_iter = 1), CholeskyQR2 (2) and shifted CholeskyQR3 (3) on an m x n matrix
    of 2-norm `norm2` and 2-norm condition number `kappa`.  Each bound adds the FP64 rounding of its own evaluation.

      orth  ||Q^T Q - I||_F.  CholeskyQR2: 6 (m n u + n (n + 1) u) (Yamamoto, Nakatsukasa, Yanagisawa, Fukaya, ETNA 44, 2015,
            under 8 kappa sqrt(m n u + n (n + 1) u) <= 1).  Shifted CholeskyQR3 ends with CholeskyQR2 on Q1 = A R1^-1, whose condition
            number the shift keeps below that condition (Fukaya, Kannan, Nakatsukasa, Yamamoto, Yanagisawa, SISC 42, 2020), so the
            same bound holds.  CholeskyQR: the same paper's ||Q^T Q - I||_2 <= (5/64) delta^2 with delta = 8 kappa sqrt(m n u +
            n (n + 1) u), i.e. 5 kappa^2 (m n u + n (n + 1) u), times sqrt(n) for the Frobenius norm.  The theorems' hypothesis
            8 kappa sqrt(m n u + n (n + 1) u) <= 1 holds for the kappa = 10 rows of the GPU table but not for most kappa = 1e5 rows
            (at m = n = 129 its left side is about 1.5; at m = 4097 it fails from n = 4 on): there the hypothesis is conservative
            and the bounds are used as they stand, beyond the range the theorems cover.  Evaluating Q^T Q - I in FP64
            adds at most gamma_m |Q|^T |Q| + u per entry, n (m + 1) u in norm for columns of norm about 1.
      res   ||A - Q R||_F / ||A||_2 <= 5 n^2 sqrt(n) u for CholeskyQR and CholeskyQR2 (Yamamoto et al. 2015).
            Shifted CholeskyQR3 forms R = R3 (R2 R1) with one more sweep and one more product: twice that constant.  Evaluating
            A - Q R in FP64 adds gamma_n ||Q||_F ||R||_F <= n^2 u ||A||_2 (1 + orth).
      fwd_r ||R - R_exact||_F / ||A||_2, R_exact the QR factor of A with a positive diagonal.  A + dA = Q R with dA = Q R - A; write
            Q = Q0 T with Q0 orthonormal and T = chol(Q^T Q), ||T - I||_F <= ||Q^T Q - I||_F to first order.  T R is the exact R
            factor of A + dA, and R(A + dA) - R(A) is at most sqrt(2) kappa ||dA||_F / ||A||_2 ||R||_2 to first order (J.-G. Sun,
            perturbation bounds for the Cholesky and QR factorizations, BIT 31, 1991); with ||R||_2 = ||A||_2,
            ||R - R_exact||_F <= (orth + sqrt(2) kappa res) ||A||_2, doubled for the higher-order terms.
    The bounds are worst-case: at kappa ~ 10 measured errors are 10^3 - 10^6 times smaller.  The tight checks of the GPU tests are
    the bit identities and the componentwise ratios; these catch anything not rounding-sized at the matrix's own scale."""

    def __init__(self, m, n, num_iter, kappa, norm2=1.0):
        self.m, self.n, self.kappa, self.norm2 = m, n, kappa, norm2
        base = (m * n + n * (n + 1)) * U
        if num_iter == 1:
            orth = 5 * kappa ** 2 * base * math.sqrt(n)
        else:
            orth = 6 * base
        res = (10 if num_iter == 3 else 5) * n ** 2.5 * U
        self.orth = orth + n * (m + 1) * U
        self.res = res + n ** 2 * U * (1 + orth)
        self.fwd_r = 2 * (orth + math.sqrt(2) * kappa * res)

    def check(self, a, q, r, r_ref):
        """(orth, res, fwd_r) ratios of the FP64 Q and R of the FP64 matrix a against these bounds; r_ref from qr_ld"""
        n = self.n
        o = np.linalg.norm(q.T @ q - np.eye(n)) / self.orth
        s = np.linalg.norm(a - q @ r) / self.norm2 / self.res
        f = float(np.linalg.norm((np.asarray(r, dtype=LD) - r_ref).astype(np.float64))) / self.norm2 / self.fwd_r
        return float(o), float(s), f


def spd_norms(a):
    """(||A||_2, kappa_2(A)) of a symmetric positive definite float64 matrix"""
    ev = np.linalg.eigvalsh(a)
    return float(ev[-1]), float(ev[-1] / ev[0])


def solve_bound(a):
    """A-priori bound on ||X - A^-1 B||_F / ||A^-1 B||_F for X = Rinv (Rinv^T B), the batched solve, with R and Rinv from the CholInv
    factor of a (any number of columns: the bound holds column by column).  With Bounds(a): R = R_c, the exact factor of
    A_c = A + dA, ||dA||_2 <= n Bounds.backward; Rinv = (I + E) R_c^-1 with ||E||_2 <= n Bounds.inverse.  Then
      P = Rinv Rinv^T satisfies P A_c - I = E + A_c^-1 E^T A_c + O(E^2), norm <= ||E|| (1 + kappa);
      replacing A_c by A moves the solution by at most kappa ||dA|| / ||A|| relatively;
      the two products add gamma_n |Rinv^T||B| and gamma_n |Rinv||T|, at most 2 gamma_n sqrt(n) ||A^-1|| ||B|| <= 2 gamma_n sqrt(n)
      kappa ||X||.
    Doubled for the higher orders.  Worst-case (Bounds' inverse term is kappa(A), not kappa(R)): it grows as kappa^2 and exceeds 1
    at kappa = 1e8 for n >= 17, so the tests gate with it only where it is below 1; solve_product_bound gates the solve at every
    kappa."""
    n = a.shape[0]
    b = Bounds(a)
    e = n * b.inverse
    return 2 * (e * (1 + b.kappa) + b.kappa * n * b.backward / b.norm2 + 2 * gamma(n) * math.sqrt(n) * b.kappa)


def lstsq_bound(m, n, num_iter, kappa, norm2, xnorm, rnorm):
    """A-priori bound on ||X - X_exact||_F / ||X_exact||_F for X = R^-1 (Q^T B) from batched CholeskyQR factors, column-wise with the
    worst column's ||r|| / ||x||.  Least-squares perturbation theory (Higham, Accuracy and Stability, 2nd ed., Thm 20.1): for
    perturbations ||dA|| <= eps ||A||, ||db|| <= eps ||b|| with kappa eps < 1,
        ||dx|| / ||x|| <= kappa eps / (1 - kappa eps) (2 + (kappa + 1) ||r|| / (||A|| ||x||)).
    X is the exact least-squares solution of Q0 (T R) = A + dA (QRBounds.fwd_r's notation) up to the non-orthogonality T - I and the
    roundings of Q^T B (gamma_m sqrt(n) ||B|| in norm) and of the substitution (|dR| <= gamma_n |R|, sqrt(n) gamma_n in norm), so
    eps = res + 2 orth + gamma_m sqrt(n) + gamma_n sqrt(n), doubled; infinite when kappa eps >= 1/2."""
    qb = QRBounds(m, n, num_iter, kappa, norm2)
    eps = 2 * (qb.res + 2 * qb.orth + (gamma(m) + gamma(n)) * math.sqrt(n))
    if kappa * eps >= 0.5:
        return math.inf
    return kappa * eps / (1 - kappa * eps) * (2 + (kappa + 1) * rnorm / (norm2 * xnorm))


def solve_product_ld(rinv, b):
    """Rinv (Rinv^T B) in np.longdouble: the batched solve's operation on the factor it was given (rinv upper, float64)"""
    rl = np.asarray(rinv, dtype=LD)
    return rl @ (rl.T @ np.asarray(b, dtype=LD))


def solve_product_bound(rinv, b):
    """A-priori bound on ||X - Rinv (Rinv^T B)||_F for the FP64 X of the batched solve, Rinv its upper factor (any summation order and
    tiling).  T = fl(Rinv^T B) has |T - Rinv^T B| <= gamma_n |Rinv^T| |B|, at most gamma_n sqrt(n) ||Rinv||_2 ||B||_F in norm
    (|| |M| ||_2 <= sqrt(n) ||M||_2); X = fl(Rinv T) adds gamma_n sqrt(n) ||Rinv||_2 ||T||_F, and the first error reaches X through
    Rinv.  So ||X - Rinv Rinv^T B||_F <= 2 gamma_n sqrt(n) ||Rinv||_2^2 ||B||_F to first order, doubled for the higher orders.
    Relative to ||X||_F >= ||B||_F / ||A||_2 this is 4 gamma_n sqrt(n) kappa(A): 5e-4 at n = 512, kappa = 1e8, linear in kappa.  With
    the factor checked against chol_ld, this checks the solve at every kappa without the kappa^2 of solve_bound."""
    n = rinv.shape[0]
    return 4 * gamma(n) * math.sqrt(n) * float(np.linalg.norm(rinv, 2)) ** 2 * float(np.linalg.norm(b))


def lstsq_product_ld(q, r, b):
    """R^-1 (Q^T B) in np.longdouble: the batched lstsq's operation on the factors it was given (q m x n, r upper, float64)"""
    y = np.asarray(q, dtype=LD).T @ np.asarray(b, dtype=LD).reshape(q.shape[0], -1)
    return _back(np.asarray(r, dtype=LD), y).reshape((q.shape[1],) + b.shape[1:])


def lstsq_product_bound(q, r, b, x):
    """A-priori bound on ||X - R^-1 (Q^T B)||_F for the FP64 X of the batched lstsq on the FP64 factors q, r (x: that operation in
    long double).  Y = fl(Q^T B) has |Y - Q^T B| <= gamma_m |Q^T| |B|, at most gamma_m ||Q||_F ||B||_F in norm (Cauchy-Schwarz per
    entry), which reaches X through R^-1.  The substitution (blocked back substitution with divisions, updates by products: no
    inverses) is backward stable, (R + dR) X = Y with |dR| <= gamma_2n |R| (Higham, Accuracy and Stability, 2nd ed., Thm 8.5 and
    its block form), so it adds at most kappa(R) gamma_2n sqrt(n) ||X||_F.  Doubled for the higher orders; linear in kappa."""
    m, n = q.shape
    sv = np.linalg.svd(r, compute_uv=False)
    return 2 * (gamma(m) * float(np.linalg.norm(q)) / float(sv[-1]) * float(np.linalg.norm(b)) +
                gamma(2 * n) * math.sqrt(n) * float(sv[0] / sv[-1]) * float(np.linalg.norm(np.asarray(x, dtype=np.float64))))


# ---- the GPU tables (tests/test_gpu_batched_reference.py), shared with the CPU check of the bounds -----------------------------------
FACTOR_N = [1, 2, 3, 17, 33, 63, 64, 65, 127, 128, 129, 191, 192, 255, 256, 257, 383, 449, 511, 512]
FACTOR_KAPPAS = (10.0, 1e8)  # plus a graded D A D of a kappa = 10 matrix
GRADE = 60                   # its exponents run from -GRADE to GRADE
QR_N = [1, 2, 7, 17, 33, 63, 65, 127, 129, 255, 257, 511, 512]
QR_FLOPS = 1.4e8             # m n^2 of one long-double QR at most: m in {n, n + 1, 1023, 4097} where affordable
QR_RUNS = {1: (10.0,), 2: (10.0, 1e5), 3: (1e10,)}  # num_iter -> kappas
SOLVE_N = [1, 17, 63, 65, 129, 257, 512]
SOLVE_KAPPAS = (10.0, 1e8)
SOLVE_K = [1, 32, 33, 65]
LS_CASES = [(1000, 100, 10.0, 2), (1000, 100, 1e5, 2), (300, 32, 1e10, 3)]  # (m, n, kappa, num_iter)
LS_RHO = (0.0, 1e-3)         # ||r|| / (||A|| ||x||); times 1e-9 at kappa = 1e10
LS_K = 33


def qr_shapes():
    out = []
    for n in QR_N:
        for m in sorted({n, n + 1, 1023, 4097}):
            if m >= n and m * n * n <= QR_FLOPS:
                out.append((m, n))
    return out


def qr_matrix(m, n, kappa):
    """the seeded ill_conditioned input of the QR table (scqr3_reference)"""
    from scqr3_reference import ill_conditioned
    return ill_conditioned(m, n, kappa, 31 * m + n + int(math.log10(kappa)))


def factor_inputs(n):
    """(name, A, grading) of each matrix of the factor table's batch at n; grading = (ungraded A, exponents) for D A D"""
    core = spd_spectrum(n, 10.0, 3 * n + 2)
    e = ramp_exponents(n, GRADE)
    return [(f"kappa={k:.0e}", spd_spectrum(n, k, 3 * n + i), None) for i, k in enumerate(FACTOR_KAPPAS)] + \
        [("graded", graded(core, e), (core, e))]


def solve_inputs(n):
    return [spd_spectrum(n, k, 13 * n + i) for i, k in enumerate(SOLVE_KAPPAS)]


def ls_problem(m, n, kappa, rho, k, seed):
    """(A, B, X_ld, residual norms): B = A X + r with r orthogonal to range(A) and ||r_j|| = rho ||A||_2 ||x_j|| (||A||_2 = 1)"""
    from scqr3_reference import ill_conditioned
    a = ill_conditioned(m, n, kappa, seed)
    rng = np.random.default_rng(seed + 1)
    x = rng.standard_normal((n, k))
    b = a @ x
    if rho > 0:
        qa, _ = np.linalg.qr(a)
        g = rng.standard_normal((m, k))
        r = g - qa @ (qa.T @ g)
        r *= rho * np.linalg.norm(x, axis=0) / np.linalg.norm(r, axis=0)
        b = b + r
    xl, res = lstsq_ld(a, b)
    return a, b, xl, res


def ls_rho(kappa, rho):
    return rho if kappa < 1e9 else rho * 1e-9


def ls_bound(a, xl, res, num_iter):
    """lstsq_bound of the problem (a, X_ld, residual norms from lstsq_ld)"""
    m, n = a.shape
    sv = np.linalg.svd(a, compute_uv=False)
    xn = np.linalg.norm(np.asarray(xl, dtype=np.float64).reshape(n, -1), axis=0)
    return lstsq_bound(m, n, num_iter, float(sv[0] / sv[-1]), float(sv[0]), float(xn.min()), float(np.max(res.astype(np.float64))))


# ---- chunk rules of the batched entry points (restated; change together with api.cu / dist.cu) -------------------------------------
WORKSPACE_CAP = 2 << 30   # BATCHED_WORKSPACE_CAP (api.cu) and QR_BATCHED_CAP (dist.cu), bytes
GRID_MAX = 65535          # grid y of the cluster kernel, grid z of the batched products
SOLVE_W = 32              # right-hand sides per panel
LEAF_MAX = 64


def _ru(x, k):
    return (x + k - 1) // k * k


def _cdiv(x, k):
    return (x + k - 1) // k


def factor_chunk(n, batch, aligned=True):
    """matrices per launch of capital_cholinv_factor_batched_f64: the leaf path (n <= 64) takes the whole batch (up to INT32_MAX);
    the cluster path holds W and Rinv^T per matrix, plus R and Rinv when it cannot write the outputs in place ("direct": n a multiple
    of 64 and R, Rinv 16-byte aligned)."""
    if n <= LEAF_MAX:
        return min(batch, 2 ** 31 - 1)
    nb = _ru(n, 64)
    direct = nb == n and aligned
    return min(batch, GRID_MAX, WORKSPACE_CAP // ((2 if direct else 4) * nb * nb * 8))


def solve_chunk(n, batch):
    """capital_cholinv_solve_batched_f64: the panel intermediate T (n x 32) and tri_apply's partials (roundup(n, 64) x 32) per matrix"""
    per = (n * SOLVE_W + _ru(n, 64) * SOLVE_W) * 8
    return min(batch, GRID_MAX, WORKSPACE_CAP // per)


def splitk_chunks(m, n, k, num_sms, c_upper=True):
    """gemm_splitk_chunks (gemm_tn.cu): the k chunks of the Gram product of an m x n output over k"""
    big = m >= 128 and n >= 128
    t = 128 if big else 64
    gm, gn = _cdiv(m, t), _cdiv(n, t)
    tiles = gm * (gm + 1) // 2 if (c_upper and gm == gn) else gm * gn
    ks = min(_cdiv(num_sms * (1 if big else 2), tiles), _cdiv(k, 16 * 32))
    return max(ks, 1)


def qr_per(m, n, num_iter, num_sms, in_place=None):
    """doubles per matrix that dist_cacqr_factor_batched holds; in_place: A read where it is (m even, 16-byte aligned)"""
    if in_place is None:
        in_place = m % 2 == 0
    need_q = num_iter > 1 or not in_place
    ldq, ldt = _ru(m, 16), _ru(n, 16)
    nr = _ru(n, 16) if n <= LEAF_MAX else _ru(n, 64)
    nb = _ru(n, 64)
    nfac = {1: 2, 2: 5, 3: 6}[num_iter]
    ks = splitk_chunks(n, n, m, num_sms)
    return ((ldq * n if need_q else 0) + ldt * m * (2 if num_iter > 1 else 1) + n * n + (ks * _ru(n, 2) * n if ks > 1 else 0) +
            nfac * nr * nr + (2 * nb * nb if n > LEAF_MAX else 0))


def qr_chunk(m, n, batch, num_iter, num_sms, in_place=None):
    """matrices per pass of capital_cacqr_factor_batched_f64"""
    return max(1, min(batch, GRID_MAX, WORKSPACE_CAP // (qr_per(m, n, num_iter, num_sms, in_place) * 8)))


def lstsq_chunk(m, n, batch):
    """capital_cacqr_lstsq_batched_f64: tri_apply's partials of Q^T B (64-row blocks x 1024-row k chunks x a 64 x 32 tile)"""
    per = _cdiv(n, 64) * _cdiv(_cdiv(m, 64), 16) * 64 * SOLVE_W * 8
    return max(1, min(batch, GRID_MAX, WORKSPACE_CAP // per))


def gram_grid_z(m, n, batch, num_iter, num_sms, in_place=None):
    """grid z that the batched Gram product of one chunk asks for (chunk x ks); launch_batched splits it only above 65535"""
    return qr_chunk(m, n, batch, num_iter, num_sms, in_place) * splitk_chunks(n, n, m, num_sms)
