"""Extended-precision references for the batched Jacobi eigensolver (capital_syevj_batched_f64): residuals in long double, reference
eigenvalues with a certified error far below u ||A||_2, and an a-posteriori gate on computed eigenvalues that needs no tuned constant.

  - ld_residual / ld_orth: R = A V - V diag(w) and V^T V - I in np.longdouble (64-bit significand on x86), so that their rounding
    (about n 2^-64 ||A||) stays far below the u ||A|| level the gates measure, even at n = 512.
  - mp_reference (n <= 64): mpmath.eigsy at 30 decimal digits on the exact double matrix.
  - rr_reference (any n): long-double Rayleigh-Ritz on scipy's eigenvectors.  A separated eigenvalue is the Rayleigh quotient rho of
    its normalised vector y, with |rho - lambda| <= ||A y - rho y||^2 / gap (Kato-Temple).  A cluster C (scipy eigenvalues closer than
    CLUSTER_TOL ||A||_2) is the Ritz block M = Y^T A Y of its orthonormalised basis Y; its eigenvalues are within ||A Y - Y M||_2^2 /
    gap of the cluster's (the quadratic residual bound), from mpmath when |C| <= MP_BLOCK, and otherwise only the trace is used.
    Each reference error also counts the long-double evaluation, 4 n 2^-64 ||A||_2.
  - Certified: Kahan's residual bound for a square, non-orthonormal basis.  For symmetric A, any nonsingular V and any w, the sorted
    eigenvalues satisfy |w_i - lambda_i| <= sqrt(2) ||A V - V diag(w)||_2 / sigma_min(V) (Kahan 1967; Stewart and Sun, Matrix
    Perturbation Theory, IV.4).  ||R||_2 is bounded from above and sigma_min(V) from below, both from long-double quantities, and
    the evaluation gets a slack of 2^-60 ||A||_2.

Because that bound holds for every (w, V), it cannot tell a wrong w from a right one on its own: moving w_i by d raises the residual
by d.  The gate therefore also requires the certified bound itself to lie within sqrt(2) 4 n u ||A||_F, what Kahan's bound gives
for a residual at the a-priori bound 4 n u ||A||_F of syevj_reference.Check and an orthonormal V, and the long-double residual and
orthogonality within their a-priori bounds."""
import math
import numpy as np

LD = np.longdouble
U = 2.0 ** -53
SLACK = 2.0 ** -60     # evaluation slack of the certified bound, relative to ||A||_2
CLUSTER_TOL = 1e-10    # scipy eigenvalues closer than this times ||A||_2 form one Ritz cluster
MP_BLOCK = 16          # Ritz blocks up to this order get their eigenvalues from mpmath; larger ones only their trace
MP_DPS = 30
ULD = 2.0 ** -64       # unit roundoff of np.longdouble (x86 extended precision)


def ld_residual(a, w, v):
    """R = A V - V diag(w) in long double"""
    V = np.asarray(v, dtype=LD)
    return np.asarray(a, dtype=LD) @ V - V * np.asarray(w, dtype=LD)[None, :]


def ld_orth(v):
    """V^T V - I in long double"""
    V = np.asarray(v, dtype=LD)
    return V.T @ V - np.eye(V.shape[1], dtype=LD)


def ld_fro(x) -> float:
    """||x||_F of a long-double array, summed at the scale of its largest entry"""
    mx = np.abs(x).max() if x.size else LD(0)
    if mx == 0:
        return 0.0
    y = x / mx
    return float(mx * np.sqrt(np.sum(y * y)))


def norm2_upper(x) -> float:
    """an upper bound on ||x||_2 of a long-double matrix: sigma_max of x rounded to double, times 1 + 2^-40.  Rounding changes each
    entry by at most 2^-53 relative, so ||x - fl(x)||_2 <= 2^-53 sqrt(n) ||x||_2, and LAPACK's sigma_max has a relative error of
    order n u; both are below 2^-40 for n <= 512."""
    mx = np.abs(x).max() if x.size else LD(0)
    if mx == 0:
        return 0.0
    e = int(np.frexp(float(mx))[1])
    s = np.linalg.norm(np.asarray(np.ldexp(x, -e), dtype=np.float64), 2)
    return math.ldexp(float(s) * (1 + 2.0 ** -40), e)


def sigma_min_lower(v) -> float:
    """a lower bound on sigma_min(V): sigma_min^2 = lambda_min(V^T V) >= 1 - ||V^T V - I||_2 >= 1 - ||V^T V - I||_F"""
    e = ld_fro(ld_orth(v))
    return math.sqrt(1.0 - e) if e < 1.0 else 0.0


def _mp():
    import mpmath
    return mpmath


def _to_mp(x):
    """an mpmath matrix holding a long-double matrix exactly (each entry as the sum of two doubles)"""
    mp = _mp()
    hi = np.asarray(x, dtype=np.float64)
    lo = np.asarray(np.asarray(x, dtype=LD) - hi, dtype=np.float64)
    m = mp.matrix(*hi.shape)
    for i in range(hi.shape[0]):
        for j in range(hi.shape[1]):
            m[i, j] = mp.mpf(float(hi[i, j])) + mp.mpf(float(lo[i, j]))
    return m


def _mp_eigvals(x):
    mp = _mp()
    with mp.workdps(MP_DPS):
        ev = mp.eigsy(_to_mp(x), eigvals_only=True)
        return np.array(sorted(LD(mp.nstr(e, MP_DPS, min_fixed=1, max_fixed=0)) for e in ev), dtype=LD)


class Reference:
    """Reference eigenvalues of one symmetric matrix, ascending: lam (long double) and err (an upper bound on |lam_i - lambda_i|)
    where known individually; `traces` lists (indices, trace, err) of clusters known only by the sum of their eigenvalues (those
    indices have err = inf)."""

    def __init__(self, lam, err, traces=()):
        self.lam, self.err, self.traces = np.asarray(lam, dtype=LD), np.asarray(err, dtype=np.float64), list(traces)


def mp_reference(a) -> Reference:
    """mpmath.eigsy at MP_DPS digits on the exact matrix: error far below 1e-25 ||A||_F"""
    a = np.asarray(a, dtype=np.float64)
    lam = _mp_eigvals(a)
    # mpmath's error, and the rounding of its result to long double
    return Reference(lam, a.shape[0] * 10.0 ** (3 - MP_DPS) * float(np.linalg.norm(a)) + ULD * np.abs(lam).astype(np.float64))


def _orthonormalise(X):
    """X G^{-1/2} in long double for a nearly orthonormal X, G = X^T X = I + E: G^{-1/2} = I - E/2 + 3 E^2 / 8 up to O(||E||^3)"""
    E = X.T @ X - np.eye(X.shape[1], dtype=LD)
    return X @ (np.eye(X.shape[1], dtype=LD) - E / 2 + 3 * (E @ E) / 8)


def rr_reference(a, tol=CLUSTER_TOL, mp_block=MP_BLOCK) -> Reference:
    """long-double Rayleigh-Ritz on scipy's eigenvectors (module docstring)"""
    import scipy.linalg as sl
    a = np.asarray(a, dtype=np.float64)
    n = a.shape[0]
    wr, xr = sl.eigh(a)
    an = float(np.abs(wr).max())
    if an == 0.0:
        return Reference(np.zeros(n), np.zeros(n))
    A = np.asarray(a, dtype=LD)
    Y = _orthonormalise(np.asarray(xr, dtype=LD))
    AY = A @ Y
    slop = 4 * n * U * an  # scipy's eigenvalues as neighbours: their error is below this
    ev = 4 * n * ULD * an   # the long-double evaluation of Y, A Y and Y^T A Y, per eigenvalue
    cuts = np.nonzero(np.diff(wr) > tol * an)[0] + 1
    lam = np.zeros(n, dtype=LD)
    err = np.full(n, np.inf)
    traces = []
    for c in np.split(np.arange(n), cuts):
        lo, hi = c[0], c[-1]
        Yc, AYc = Y[:, c], AY[:, c]
        M = Yc.T @ AYc
        M = (M + M.T) / 2
        R = AYc - Yc @ M
        r2 = ld_fro(R) ** 2
        left = wr[lo - 1] + slop if lo > 0 else -np.inf
        right = wr[hi + 1] - slop if hi + 1 < n else np.inf
        if len(c) == 1:
            rho = M[0, 0]
            gap = min(float(rho) - left, right - float(rho))
            lam[lo], err[lo] = rho, r2 / gap + ev
        elif len(c) <= mp_block:
            th = _mp_eigvals(M)
            gap = min(float(th[0]) - left, right - float(th[-1]))
            lam[c], err[c] = th, r2 / gap + len(c) * 10.0 ** (3 - MP_DPS) * an + ev
        else:
            lam[c] = np.diagonal(M)
            gap = min(float(np.diagonal(M).min()) - left, right - float(np.diagonal(M).max()))
            traces.append((c, np.trace(M), len(c) * (r2 / gap + ev)))
    return Reference(lam, err, traces)


class Certified:
    """The gate on one computed eigendecomposition (w ascending, V) of the symmetric a against a Reference:
      bound = sqrt(2) ||R||_2 / sigma_min(V) + 2^-60 ||A||_2   (Kahan; R = A V - V diag(w) in long double)
      |w_i - lam_i| <= bound + err_i for the individually known reference eigenvalues,
      |sum_C w - trace_C| <= |C| bound + err_C for the clusters known by their trace,
      bound <= sqrt(2) 4 n u ||A||_F, ||R||_F <= 4 n u ||A||_F, ||V^T V - I||_F <= 4 n u max(4, n) (long double), w ascending."""

    def __init__(self, a, w, v, ref: Reference):
        a = np.asarray(a, dtype=np.float64)
        w, v = np.asarray(w, dtype=np.float64), np.asarray(v, dtype=np.float64)
        n = a.shape[0]
        R = ld_residual(a, w, v)
        self.anorm_2 = float(np.linalg.norm(a, 2)) * (1 + 2.0 ** -40)
        self.anorm_f = float(np.linalg.norm(a))
        self.residual = ld_fro(R)
        self.orth = ld_fro(ld_orth(v))
        smin = sigma_min_lower(v)
        self.bound = math.sqrt(2) * norm2_upper(R) / smin + SLACK * self.anorm_2 if smin > 0 else math.inf
        dw = np.abs(np.asarray(w, dtype=LD) - ref.lam).astype(np.float64)
        known = np.isfinite(ref.err)
        self.werr = float(dw[known].max()) if known.any() else 0.0
        den = self.bound + ref.err[known]
        self.wratio = float(np.where(den > 0, dw[known] / np.where(den > 0, den, 1.0), 0.0).max()) if known.any() else 0.0
        self.trace_ok = all(abs(float(np.sum(np.asarray(w[c], dtype=LD)) - t)) <= len(c) * self.bound + e for c, t, e in ref.traces)
        self.eig_ok = bool((dw[known] <= self.bound + ref.err[known]).all()) and self.trace_ok
        self.apriori = (math.sqrt(2) * 4 * n * U * self.anorm_f, 4 * n * U * self.anorm_f, 4 * n * U * max(4, n))
        self.ascending = bool(np.all(np.diff(w) >= 0))
        self.ok = (self.eig_ok and self.bound <= self.apriori[0] and self.residual <= self.apriori[1] and self.orth <= self.apriori[2]
                   and self.ascending)

    def ratios(self):
        """(certified bound, long-double residual, long-double orthogonality) over their a-priori bounds"""
        return tuple(x / b if b > 0 else 0.0 for x, b in zip((self.bound, self.residual, self.orth), self.apriori))

    def __repr__(self):
        b, r, o = self.ratios()
        return (f"Certified(w err {self.werr:.3g} <= {self.wratio:.3g} x (bound + ref err), traces {self.trace_ok}, bound {b:.3g}, "
                f"residual {r:.3g}, orth {o:.3g} of a-priori, ascending {self.ascending})")


def reference(a) -> Reference:
    """mp_reference for n <= 64 (about 1.6 s per matrix at n = 64), rr_reference above"""
    return mp_reference(a) if np.asarray(a).shape[0] <= 64 else rr_reference(a)


def certify(a, w, v, ref=None) -> Certified:
    return Certified(a, w, v, reference(a) if ref is None else ref)
