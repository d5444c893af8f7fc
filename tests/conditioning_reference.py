"""Inputs and error bounds for the conditioning tests: seeded SPD generators (prescribed spectrum, power-of-two grading, uniform
power-of-two scaling), componentwise backward-error bounds for R and R^-1, and a scalar restatement of the Cholesky phase of
`warp_potrf_trtri_32` (capital_b200/csrc/leaf.cu), the two-pivot step of the cluster base case.

Plain numpy / torch: importing this module needs no GPU.  The bound functions take torch tensors on any device, so the GPU tests
evaluate them on the device in FP64."""
import math
from fractions import Fraction
import numpy as np
import torch

U = 2.0 ** -53                # unit roundoff of FP64
DBL_MAX = float(np.finfo(np.float64).max)


def gamma(k: int) -> float:
    """Higham's gamma_k = k u / (1 - k u)."""
    return k * U / (1 - k * U)


# ---- generators -------------------------------------------------------------------------------------------------------------
def spd_spectrum(n: int, kappa: float, seed: int, device="cpu") -> torch.Tensor:
    """Q diag(logspace(0, -log10 kappa, n)) Q^T, symmetrized; Q from the QR factorization of a seeded Gaussian matrix.  The Gaussian
    is drawn on the host (so that a seed names one matrix on every device) and factored on `device`."""
    g = torch.Generator().manual_seed(seed)
    q, _ = torch.linalg.qr(torch.randn(n, n, dtype=torch.float64, generator=g).to(device))
    lam = torch.logspace(0, -math.log10(kappa), n, dtype=torch.float64, device=device)
    a = (q * lam) @ q.T
    return 0.5 * (a + a.T)


def ramp_exponents(n: int, emax: int) -> torch.Tensor:
    """Integer exponent profile e_i rising linearly from -emax to +emax (int64)."""
    return torch.round(torch.linspace(-emax, emax, n, dtype=torch.float64)).to(torch.int64)


def pow2(e: torch.Tensor, device="cpu") -> torch.Tensor:
    """2^e (FP64) for an integer tensor e, formed exactly on the host"""
    return torch.from_numpy(np.ldexp(1.0, e.cpu().numpy().astype(np.int64))).to(device)


def graded(a: torch.Tensor, e: torch.Tensor) -> torch.Tensor:
    """D A D with D = diag(2^e): exact in FP64 as long as no entry leaves the normal range."""
    d = pow2(e, a.device)
    return a * d[:, None] * d[None, :]


def scaled(a: torch.Tensor, k: int) -> torch.Tensor:
    """2^(2k) A, exactly; R(2^(2k) A) = 2^k R(A) and R^-1(2^(2k) A) = 2^-k R^-1(A)."""
    return a * math.ldexp(1.0, 2 * k)


def pair_product_log2(a: torch.Tensor, e: torch.Tensor) -> tuple:
    """(min, max) over k even of log2(d_k d_{k+1}), d = diag(D A D): the range of the products a * b that the two-pivot step of
    `warp_potrf_trtri_32` forms for graded inputs (its pivot pairs are (k, k+1), k even), without forming D A D."""
    d = torch.log2(torch.diagonal(a).double().cpu()) + 2.0 * e.double().cpu()
    s = d[0:d.numel() - 1:2] + d[1::2]
    return float(s.min()), float(s.max())


# ---- componentwise bounds ---------------------------------------------------------------------------------------------------
def _worst(err: torch.Tensor, bound: torch.Tensor) -> float:
    """max of err / bound; an entry with a zero bound must be exact (ratio inf otherwise)"""
    pos = bound > 0
    r = (err[pos] / bound[pos]).max().item() if bool(pos.any()) else 0.0
    if bool((err[~pos] > 0).any()):
        return math.inf
    return float(r)


def chol_ratio(a: torch.Tensor, r: torch.Tensor) -> float:
    """Worst ratio of |A - R^T R| to gamma_{n+1} |R|^T |R| over the upper triangle (Higham, Accuracy and Stability of Numerical
    Algorithms, 2nd ed., Thm 10.3: the computed R of any standard Cholesky ordering satisfies R^T R = A + dA,
    |dA| <= gamma_{n+1} |R|^T |R|).  A factor of a correct implementation gives a ratio below 1.

    Evaluating A - R^T R in FP64 adds at most gamma_n |R|^T |R| + u |A| <= (gamma_n + u (1 + gamma_{n+1})) |R|^T |R|: about one more
    bound, folded into the gate constant c of `ratio <= c`.  The bound is invariant under grading: with D = diag(2^e),
    R(D A D) = R(A) D and both sides scale by D . D entrywise; so is the ratio."""
    n = a.shape[0]
    ra = r.abs()
    err = (a - r.T @ r).abs().triu()
    return _worst(err, (gamma(n + 1) * (ra.T @ ra)).triu())


def inv_ratio(r: torch.Tensor, x: torch.Tensor, n1: int = None) -> float:
    """Worst ratio of the left residual |X R - I| to gamma_n |X| |R| |X| |R|, X the computed inverse of the computed upper factor R.
    With n1, only the diagonal blocks [0, n1) and [n1, n) are checked (complete_inv = 0 leaves the top-level X12 block zero).

    Why |X||R||X||R|.  X is built by the recursive combine X12 = -(X11 R12) X22 on top of diagonal blocks with E_ii = X_ii R_ii - I.
    Write T = fl(X11 R12) = X11 R12 + F1, |F1| <= gamma_n |X11||R12|, and X12 = -fl(T X22) = -T X22 - F2, |F2| <= gamma_n |T||X22|.
    Then the off-diagonal block of E = X R - I is
        E12 = X11 R12 + X12 R22 = X11 R12 - (X11 R12 + F1) X22 R22 - F2 R22
            = -X11 R12 E22 - F1 (I + E22) - F2 R22,
    so, to first order in u,
        |E12| <= |X11||R12||E22| + gamma_n |X11||R12| + gamma_n |X11||R12||X22||R22|.
    By induction |E_ii| <= c_i gamma_n |X_ii||R_ii||X_ii||R_ii|, and |X||R| has a unit diagonal and is non-negative, so
    |X||R| <= |X||R||X||R| entrywise; every term above is then a multiple of gamma_n (|X||R||X||R|)_12, and
    |E| <= c gamma_n |X||R||X||R| with c growing with the depth of the recursion only.  The base case's substitution solves
    R X = I (residual <= gamma_n |R||X|); its left residual X R - I = X (R X - I) X^-1 is of the same form.  The plain |X||R|
    (the bound of a column-oriented trtri) does not hold for the recursive combine.  Evaluating X R - I in FP64 adds
    gamma_n |X||R| <= gamma_n |X||R||X||R|, folded into c.  Under grading X(D A D) = D^-1 X(A) and R(D A D) = R(A) D: the
    residual and the bound both scale by D^-1 . D entrywise."""
    def one(rb, xb):
        m = rb.shape[0]
        eye = torch.eye(m, dtype=rb.dtype, device=rb.device)
        xa, ra = xb.abs(), rb.abs()
        err = (xb @ rb - eye).abs().triu()
        return _worst(err, (gamma(m) * (xa @ (ra @ (xa @ ra)))).triu())
    if n1 is None:
        return one(r, x)
    return max(one(r[:n1, :n1], x[:n1, :n1]), one(r[n1:, n1:], x[n1:, n1:]))


# ---- the two-pivot step of warp_potrf_trtri_32, restated -----------------------------------------------------------------------
def fma(x: float, y: float, z: float) -> float:
    """x y + z with one rounding (IEEE fused multiply-add) for finite operands; overflow gives inf."""
    if not (math.isfinite(x) and math.isfinite(y) and math.isfinite(z)):
        return x * y + z
    v = Fraction(x) * Fraction(y) + Fraction(z)
    try:
        return float(v)
    except OverflowError:
        return math.inf if v > 0 else -math.inf


def fast_rsqrt(d: float) -> float:
    """leaf.cu fast_rsqrt: an FP32 seed and two FP64 Newton steps inside (1e-30, 1e30), the library rsqrt outside.  The FP32 seed
    here is the correctly rounded 1/sqrt, not the hardware's approximation, so results agree with the GPU to about 1 ulp, not bitwise."""
    if not (1e-30 < d < 1e30):
        if d == 0.0:
            return math.inf
        return 1.0 / math.sqrt(d) if d > 0 else math.nan
    y = float(np.float32(1.0) / np.sqrt(np.float32(d)))
    h = 0.5 * d
    y = y * fma(-h, y * y, 1.5)
    y = y * fma(-h, y * y, 1.5)
    return y


def _pivot_pair(a: float, l: float, b: float):
    """One step of the pivot pair (k, k+1) from a = A(k,k), l = A(k,k+1), b = A(k+1,k+1) (a already checked positive): det = a b - l^2
    in one fma, rsqrt(a) and rsqrt(det) side by side.  Returns (ra, lk, rs2, d1, second_ok): 1/R(k,k), R(k,k+1), 1/R(k+1,k+1),
    R(k+1,k+1) and whether the second pivot was positive."""
    det = fma(b, a, -(l * l))
    ok = True
    if not det > 0.0:
        ok, det = False, 1.0
    ra, rdet = fast_rsqrt(a), fast_rsqrt(det)
    sa, lk = a * ra, l * ra
    return ra, lk, sa * rdet, det * rdet * ra, ok


BLOCK_SAFE = (2.0 ** -400, 2.0 ** 400)


def warp_potrf_32(a: np.ndarray, guarded: bool = True):
    """The Cholesky phase of warp_potrf_trtri_32 (leaf.cu) on a 32 x 32 SPD block, operation for operation: lane j holds column j,
    c[i][j] = A(i, j); two pivots per step, then the rank-2 update c[i] -= R(k+1, i) R(k+1, j) + R(k, i) R(k, j) as two fmas.
    Without `guarded`, the kernel before the fix.  With it, the fixed kernel: unless every diagonal entry lies in [2^-400, 2^400]
    (BLOCK_SAFE), the block is first equilibrated to S = D^-1 A D^-1, D = diag(2^e), e_j = floor(log2(A(j,j)) / 2), and the factor is
    R = R(S) D.  Returns (R, info): R upper triangular, info the 1-based index of the first non-positive pivot (0: none)."""
    assert a.shape == (32, 32)
    c = [[float(a[i, j]) for j in range(32)] for i in range(32)]
    f = [1.0] * 32  # 2^-e
    if guarded and not all(BLOCK_SAFE[0] <= c[i][i] <= BLOCK_SAFE[1] for i in range(32)):
        f = [math.ldexp(1.0, -(math.frexp(c[j][j])[1] - 1 >> 1)) if 0.0 < c[j][j] <= DBL_MAX else 1.0 for j in range(32)]
        c = [[c[i][j] * f[i] * f[j] for j in range(32)] for i in range(32)]
    info = 0
    for k in range(0, 32, 2):
        pa, pl, pb = c[k][k], c[k][k + 1], c[k + 1][k + 1]
        if not pa > 0.0:
            info = info or k + 1
            pa = 1.0
        ra, lk, rs2, d1, ok = _pivot_pair(pa, pl, pb)
        if not ok:
            info = info or k + 2
        u0 = [c[k][j] * ra if j > k else (pa * ra if j == k else 0.0) for j in range(32)]
        u1 = [0.0] * 32
        for j in range(k + 1, 32):
            u1[j] = d1 if j == k + 1 else fma(-lk, u0[j], c[k + 1][j]) * rs2
        c[k], c[k + 1] = u0, u1
        for i in range(k + 2, 32):
            ci = c[i]
            for j in range(i, 32):  # lanes j < i hold R's zero lower part at the end; nothing reads them
                ci[j] = fma(-u1[i], u1[j], fma(-u0[i], u0[j], ci[j]))
    r = np.triu(np.array(c))
    return r / np.array(f)[None, :], info
