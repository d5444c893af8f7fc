"""A numpy model of the batched Jacobi eigensolver's exact schedule (capital_b200/csrc/syevj.cu), the test matrices with known spectra,
and the accuracy bounds the GPU tests gate on.

The model follows the kernels' decisions: the circle-method pairing, the padding of n to an even order (n <= 64) or to Np =
roundup(n, 64) (n > 64), the skip threshold |a_pq| <= max(u sqrt|a_pp| sqrt|a_qq|, u ||A||_F), the inner sweeps on 64 x 64
subproblems with their "quiet" flag (no rotation in the first inner sweep), the block step A <- Q^T A Q, V <- V Q over the pairs of
one outer step, and convergence after an outer sweep in which every subproblem was quiet.  It does not model the last bits: the
block update is a dense product here, and the 2 x 2 updates run as whole-row and whole-column passes."""
import numpy as np

U = 2.0 ** -53
SWEEPS = 30            # the sweep bound of syevj.cu (inner and outer)
WORKSPACE_CAP = 2 << 30
FAMILIES = ("random", "cluster", "repeated", "rankdef", "negdef", "graded", "diagonal", "zero")


def pairing(m: int, s: int):
    """pairs (p, q), p < q, of circle-method step s in [0, m - 1) over m (even) players: (s, m - 1) and ((s + k) mod (m - 1),
    (s - k) mod (m - 1)) for k = 1 .. m / 2 - 1"""
    out = [(s, m - 1)]
    for k in range(1, m // 2):
        a, b = (s + k) % (m - 1), (s - k) % (m - 1)
        out.append((min(a, b), max(a, b)))
    return out


def chunk(n: int, batch: int) -> int:
    """matrices per chunk of capital_syevj_batched_f64: at most 65535; for n > 64 the 2 GiB workspace cap over A, V (Np x Np each)
    and the Np / 64 subproblem Q tiles of 64 x 64 per matrix"""
    if n <= 64:
        return min(batch, 65535)
    Np = -(-n // 64) * 64
    return min(batch, 65535, WORKSPACE_CAP // ((2 * Np * Np + Np // 64 * 4096) * 8))


def _threshold(app, aqq, floor):
    return np.maximum(U * (np.sqrt(np.abs(app)) * np.sqrt(np.abs(aqq))), floor)


def jacobi(A, V, floor, sweeps=SWEEPS):
    """Cyclic Jacobi in circle-method order on a batch A (B, m, m), m even, accumulating into V (B, m, m), in place.  floor: (B,).
    Returns (sweeps run up to and including the first sweep without a rotation, first sweep rotated, converged), each (B,)."""
    B, m, _ = A.shape
    steps = [np.array(pairing(m, s)).T for s in range(m - 1)]
    ar = np.arange(B)[:, None]
    first = np.zeros(B, bool)
    conv = np.zeros(B, bool)
    count = np.zeros(B, int)
    for sweep in range(sweeps):
        rot = np.zeros(B, bool)
        for p, q in steps:
            app, aqq, apq = A[:, p, p], A[:, q, q], A[:, p, q]
            fire = ~(np.abs(apq) <= _threshold(app, aqq, floor[:, None]))
            if not fire.any():
                continue
            rot |= fire.any(1)
            with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
                tau = np.where(fire, (aqq - app) / (2.0 * apq), 0.0)
                t = np.where(np.abs(tau) > 2.0 ** 60, 0.5 / tau,
                             np.copysign(1.0, tau) / (np.abs(tau) + np.sqrt(tau * tau + 1.0)))
            t = np.where(fire, t, 0.0)
            c = np.where(fire, 1.0 / np.sqrt(t * t + 1.0), 1.0)
            s = t * c
            for M in (A, V):  # columns
                Mp, Mq = M[:, :, p].copy(), M[:, :, q].copy()
                M[:, :, p] = Mp * c[:, None, :] - Mq * s[:, None, :]
                M[:, :, q] = Mp * s[:, None, :] + Mq * c[:, None, :]
            Ap, Aq = A[:, p, :].copy(), A[:, q, :].copy()  # rows
            A[:, p, :] = c[:, :, None] * Ap - s[:, :, None] * Aq
            A[:, q, :] = s[:, :, None] * Ap + c[:, :, None] * Aq
            A[ar, p, p] = np.where(fire, app - t * apq, A[ar, p, p])
            A[ar, q, q] = np.where(fire, aqq + t * apq, A[ar, q, q])
            A[ar, p, q] = np.where(fire, 0.0, A[ar, p, q])
            A[ar, q, p] = np.where(fire, 0.0, A[ar, q, p])
        if sweep == 0:
            first = rot.copy()
        count += ~conv
        conv |= ~rot
        if conv.all():
            break
    return count, first, conv


def fro(a):
    return float(np.linalg.norm(a))


def _finish(Aw, V, n):
    """w = the real diagonal, ascending by rank counting (ties by index); V's real columns permuted alike, real rows"""
    d = np.diagonal(Aw, axis1=1, axis2=2)[:, :n]
    order = np.argsort(d, axis=1, kind="stable")
    w = np.take_along_axis(d, order, 1)
    Vr = np.stack([V[b][:n][:, order[b]] for b in range(V.shape[0])])
    return w, Vr


def syevj(A, snapshots=False):
    """The model on a batch A (B, n, n) of symmetric matrices.  Returns a dict: w, V, info, sweeps (per matrix: outer sweeps for
    n > 64, sweeps for n <= 64), the padded iterate Aw and Vw, and for n > 64 with `snapshots`, steps: the finished (w, V) after every
    outer step."""
    A = np.asarray(A, dtype=np.float64)
    B, n, _ = A.shape
    floor = np.array([U * fro(a) for a in A])
    if n <= 64:
        m = n + (n & 1)
        Aw = np.zeros((B, m, m))
        Aw[:, :n, :n] = A
        Vw = np.tile(np.eye(m), (B, 1, 1))
        count, _, conv = jacobi(Aw, Vw, floor)
        w, V = _finish(Aw, Vw, n)
        return dict(w=w, V=V, info=(~conv).astype(int), sweeps=count, Aw=Aw, Vw=Vw)
    Np = -(-n // 64) * 64
    N, h = Np // 32, Np // 64
    Aw = np.zeros((B, Np, Np))
    Aw[:, :n, :n] = A
    Vw = np.tile(np.eye(Np), (B, 1, 1))
    active = np.ones(B, bool)
    sweeps = np.zeros(B, int)
    steps = []
    for sweep in range(SWEEPS):
        dirty = np.zeros(B, bool)
        for s in range(N - 1):
            idx = np.array([np.r_[32 * I:32 * I + 32, 32 * J:32 * J + 32] for I, J in pairing(N, s)])  # (h, 64)
            act = np.nonzero(active)[0]
            if len(act) == 0:
                break
            S = Aw[act][:, idx[:, :, None], idx[:, None, :]].reshape(-1, 64, 64).copy()
            Q = np.tile(np.eye(64), (S.shape[0], 1, 1))
            _, first, _ = jacobi(S, Q, np.repeat(floor[act], h))
            quiet = ~first.reshape(len(act), h)
            S, Q = S.reshape(len(act), h, 64, 64), Q.reshape(len(act), h, 64, 64)
            for ai, b in enumerate(act):
                if quiet[ai].all():
                    continue
                Qb = np.zeros((Np, Np))
                for P in range(h):
                    Qb[np.ix_(idx[P], idx[P])] = Q[ai, P]
                An = Qb.T @ Aw[b] @ Qb
                An = (An + An.T) / 2
                for P in range(h):
                    if not quiet[ai, P]:
                        An[np.ix_(idx[P], idx[P])] = S[ai, P]
                Aw[b] = An
                Vw[b] = Vw[b] @ Qb
                dirty[b] = True
            if snapshots:
                steps.append(_finish(Aw, Vw, n))
        sweeps += active
        active &= dirty
        if not active.any():
            break
    w, V = _finish(Aw, Vw, n)
    return dict(w=w, V=V, info=active.astype(int), sweeps=sweeps, Aw=Aw, Vw=Vw, steps=steps)


# ---- test matrices with known spectra -----------------------------------------------------------------------------------------------
def family(name: str, n: int, seed: int):
    """(A, eigenvalues ascending): A = Q diag(lam) Q^T with a random orthogonal Q, exactly symmetric, for the families
      random    lam uniform in [-1, 1]
      cluster   half of lam at 1 +- 1e-12, the rest in [-1, 0.5]
      repeated  a 10-fold eigenvalue 0.5 (n-fold when n < 10), the rest in [-1, 1]
      rankdef   half of lam exactly zero
      negdef    lam in [-1, -0.1]
      graded    lam logarithmically spaced over [1e-15, 1]
      diagonal  A = diag(lam), lam standard normal (no rotation)
      zero      A = 0"""
    g = np.random.default_rng(seed)
    if name == "zero":
        return np.zeros((n, n)), np.zeros(n)
    if name == "diagonal":
        lam = g.standard_normal(n)
        return np.diag(lam), np.sort(lam)
    k = n // 2
    if name == "random":
        lam = g.uniform(-1, 1, n)
    elif name == "cluster":
        lam = np.r_[1 + 1e-12 * g.uniform(-1, 1, max(k, 1)), g.uniform(-1, 0.5, n - max(k, 1))]
    elif name == "repeated":
        m = min(10, n)
        lam = np.r_[np.full(m, 0.5), g.uniform(-1, 1, n - m)]
    elif name == "rankdef":
        lam = np.r_[np.zeros(k), g.uniform(-1, 1, n - k)]
    elif name == "negdef":
        lam = -g.uniform(0.1, 1, n)
    elif name == "graded":
        lam = np.logspace(-15, 0, n) if n > 1 else np.ones(1)
    else:
        raise ValueError(name)
    Q, _ = np.linalg.qr(g.standard_normal((n, n)))
    a = (Q * lam) @ Q.T
    a = np.tril(a) + np.tril(a, -1).T
    return a, np.sort(lam)


# ---- bounds ---------------------------------------------------------------------------------------------------------------------------
class Check:
    """The gated quantities of one eigendecomposition against their bounds (u = 2^-53):
      ||A V - V diag(w)||_F <= 4 n u ||A||_F,  max |w - w_scipy| <= 4 n u ||A||_2,  w ascending,
      ||V^T V - I||_F <= 4 n u max(4, n).
    The orthogonality bound is wider than 4 n u on purpose.  Every rotation applied to V leaves a rounding of order u in the two
    columns it mixes, and Jacobi applies many: up to s (n - 1) per column over s sweeps for n <= 64, and for n > 64 every outer step
    applies a 64 x 64 Q that itself accumulated the rotations of a whole inner solve.  Measured on an H100, ||V^T V - I||_F reached
    4.4 x 4 n u at n = 64 and grew about linearly in n beyond (up to about 280 x 4 n u at n = 512, graded spectrum, before the
    floor of the threshold was raised to u ||A||_F), so 4 n u max(4, n) is the bound."""

    def __init__(self, a, w, v):
        import scipy.linalg as sl
        n = a.shape[0]
        self.anorm_f, self.anorm_2 = fro(a), float(np.linalg.norm(a, 2))
        self.residual = fro(a @ v - v * w)
        self.orth = fro(v.T @ v - np.eye(n))
        self.wref = sl.eigh(a, eigvals_only=True)
        self.werr = float(np.abs(w - self.wref).max())
        self.ascending = bool(np.all(np.diff(w) >= 0))
        self.bounds = (4 * n * U * self.anorm_f, 4 * n * U * max(4, n), 4 * n * U * self.anorm_2)
        self.ok = (self.residual <= self.bounds[0] and self.orth <= self.bounds[1] and self.werr <= self.bounds[2] and self.ascending)

    def __repr__(self):
        return (f"Check(residual {self.residual:.3g} / {self.bounds[0]:.3g}, orth {self.orth:.3g} / {self.bounds[1]:.3g}, "
                f"w {self.werr:.3g} / {self.bounds[2]:.3g}, ascending {self.ascending})")


def check(a, w, v) -> Check:
    return Check(np.asarray(a), np.asarray(w), np.asarray(v))


def vectors_ok(a, w, v, tol_cluster=1e-6) -> bool:
    """Eigenvectors against scipy's, cluster by cluster: eigenvalues of scipy's spectrum closer than tol_cluster ||A||_2 form one
    cluster C with gap g_C to the rest.  The computed columns of C must lie in scipy's invariant subspace of C up to
    ||V_C - P_C V_C||_F <= (4 n + 64) u ||A||_2 |C| / g_C (for a single eigenvalue: the eigenvector within that bound of scipy's,
    up to sign).  n u ||A|| / g_C is the first-order error of one backward stable solver; the comparison holds two (4 n), and the 64 u
    covers the rounding every eigenvector carries whatever n (at n = 2 .. 7, n u alone was exceeded on an H100).  The factor |C|
    rather than sqrt(|C|): a 15-fold cluster at n = 31 was 1.9 times over the sqrt(|C|) form, in the numpy model and on the GPU.
    Clusters whose bound is not below 0.1 (gap at the rounding level) are not checked."""
    import scipy.linalg as sl
    n = a.shape[0]
    wr, vr = sl.eigh(a)
    an = float(np.linalg.norm(a, 2))
    if n == 1 or an == 0.0:
        return True
    cuts = np.nonzero(np.diff(wr) > tol_cluster * an)[0] + 1
    for c in np.split(np.arange(n), cuts):
        lo, hi = c[0], c[-1]
        gap = min(wr[lo] - wr[lo - 1] if lo > 0 else np.inf, wr[hi + 1] - wr[hi] if hi + 1 < n else np.inf)
        if len(c) == n:
            continue  # one cluster holds the whole spectrum: every orthonormal basis spans it
        bound = (4 * n + 64) * U * an * len(c) / gap
        if not bound < 0.1:
            continue
        Vc, Rc = v[:, c], vr[:, c]
        if fro(Vc - Rc @ (Rc.T @ Vc)) > bound:
            return False
    return True
