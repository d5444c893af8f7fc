"""Batched Jacobi eigensolver (eig.syevj_batched) against extended-precision references, over the whole exponent range, at the chunk
and loop edges of its launches, on poisoned workspaces, and inside eigh_batched on ill-conditioned pencils.

  - accuracy: every family of syevj_reference at each n of ACCURACY_N; eigenvalues gated by the certified bound of
    syevj_ld_reference against mpmath (n <= 64) or long-double Rayleigh-Ritz references, residual and orthogonality in long double;
    the bits of (w, V, info) pinned by tests/golden/syevj_sha256.json, recorded before the solver normalised each matrix by a power
    of 4 (tools/syevj_sha256.py), so the normalisation is shown to change no bit of an in-range matrix;
  - exponent range: A_j = 4^j A from a largest entry of about 2^-1070 to ||A||_2 just below DBL_MAX: V bit for bit and w = 4^j w of
    the exactly scaled-back B_j = 4^-j A_j, info 0; odd powers of two gated by the certified bound; crafted matrices at the top;
    NaN and Inf matrices stay local;
  - the small path's second launch (batch > 65535) and a chunk of more than 1024 matrices at n > 64 (the sweep-end loop);
  - every batched entry point on poisoned workspaces, and stale syevj workspace of a larger n on one context;
  - eigh_batched with eigensolver="jacobi" at kappa(B) = 1e8 and on a graded D B D."""
import hashlib, json, os
import numpy as np
import pytest
import scipy.linalg as sl
import torch
import capital_b200 as cb
from capital_b200 import _lib
import batched_sygst_reference as bs
import syevj_ld_reference as lr
import syevj_reference as sr

pytestmark = pytest.mark.gpu

F64 = torch.float64
U = 2.0 ** -53
DBL_MAX = float(np.finfo(np.float64).max)
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "syevj_sha256.json")
ACCURACY_N = [1, 2, 3, 7, 31, 32, 33, 63, 64, 65, 100, 127, 128, 129, 255, 256, 257, 383, 511, 512]
LARGE_N_FAMILIES = ("cluster", "graded")  # the certified families at n >= 257 (long-double products take ~1 s each there)


@pytest.fixture(scope="module")
def topo():
    t = cb.topo.square(1, 0, 1)
    yield t
    # the batches here leave workspace and cached blocks behind; the multi-rank tests that run later share this GPU
    t.context().release_workspace()
    torch.cuda.empty_cache()


def _same(x, y):
    return torch.equal(x.contiguous().view(torch.int64), y.contiguous().view(torch.int64))


def _batch(mats):
    return torch.from_numpy(np.stack(mats)).cuda()


def _sha(t):
    return hashlib.sha256(t.cpu().contiguous().numpy().tobytes()).hexdigest()


# ---- accuracy against extended-precision references --------------------------------------------------------------------------------

@pytest.mark.parametrize("n", ACCURACY_N)
def test_certified_accuracy_and_pinned_bits(topo, n):
    fams = list(sr.FAMILIES)
    mats = [sr.family(f, n, 1000 * n + i)[0] for i, f in enumerate(fams)]  # the inputs of tools/syevj_sha256.py
    w, V, info = cb.eig.syevj_batched(_batch(mats), topo)
    golden = {r["n"]: r for r in json.load(open(GOLDEN))}[n]
    assert (_sha(w), _sha(V), _sha(info)) == (golden["w"], golden["V"], golden["info"])
    graded = fams.index("graded")  # may end with info = 1 at n >= 511 (DESIGN.md 5h); its last iterate meets every bound
    assert [x for i, x in enumerate(info.tolist()) if i != graded or n < 511] == [0] * (len(fams) - (n >= 511))
    wn, vn = w.cpu().numpy(), V.cpu().numpy()
    for i, f in enumerate(fams):
        if n >= 257 and f not in LARGE_N_FAMILIES:
            continue
        c = lr.certify(mats[i], wn[i], vn[i])
        assert c.ok, (f, c)
        rat = c.ratios()
        print(f"n={n} {f}: w err / (bound + ref err) {c.wratio:.3g}; bound {rat[0]:.3g}, residual {rat[1]:.3g}, orth {rat[2]:.3g}"
              " of the a-priori bounds")


# ---- the exponent range -----------------------------------------------------------------------------------------------------------
RANGE_N = [2, 7, 33, 64, 65, 129, 512]
RANGE_FAMILIES = ("random", "graded", "rankdef", "diagonal")


def _powers(a):
    """j of the scalings 4^j A: largest entry about 2^-1070 (most entries subnormal), near the bottom of the normal range, 1, ||A||_F
    just below DBL_MAX, and ||A||_2 just below DBL_MAX (||A||_F above it when the two differ by more than a factor 4)"""
    e = int(np.frexp(np.abs(a).max())[1]) - 1
    f, s2 = sr.fro(a), float(np.linalg.norm(a, 2))
    jf = int(np.floor((np.log2(DBL_MAX) - np.log2(f)) / 2))
    j2 = int(np.floor((np.log2(DBL_MAX) - np.log2(s2) - 1e-9) / 2))
    return sorted({(-1070 - e) // 2, (-1020 - e) // 2, 0, jf, j2})


def _crafted(n):
    """(name, matrix) at the top of the range, finite entries"""
    out = []
    d = np.zeros(n)
    d[0], d[n // 2] = DBL_MAX, -DBL_MAX
    out.append(("diag_dbl_max", np.diag(d)))
    ones = np.ones((n, n)) * (DBL_MAX / (n - 1)) if n > 2 else np.full((n, n), 0.75 * DBL_MAX)
    out.append(("ones_over", ones))                  # eigenvalue n DBL_MAX / (n - 1) > DBL_MAX: +Inf
    out.append(("neg_ones_over", -ones))
    out.append(("diag_1e307", np.diag(np.full(n, 1e307))))  # ||A||_F > DBL_MAX once n > 3
    return out


@pytest.mark.parametrize("n", RANGE_N)
def test_exponent_range_matches_the_scaled_back_matrix(topo, n):
    A, B, keys = [], [], []
    for i, f in enumerate(RANGE_FAMILIES):
        a = sr.family(f, n, 17 * n + i)[0]
        for j in _powers(a):
            aj = np.ldexp(a, 2 * j)
            A.append(aj)
            B.append(np.ldexp(aj, -2 * j))  # exact
            keys.append((f, j))
    for name, c in _crafted(n):
        A.append(c)
        B.append(c)
        keys.append((name, 0))
    pos_nan, pos_inf = 1, len(A) // 2
    An = [x.copy() for x in A]
    An[pos_nan][n - 1, 0] = np.nan
    An[pos_inf][0, 0] = np.inf
    w, V, info = cb.eig.syevj_batched(_batch(A), topo)
    wb, Vb, infob = cb.eig.syevj_batched(_batch(B), topo)
    assert info.equal(infob)
    # the graded spectrum may end with info = 1 at n >= 511 (DESIGN.md 5h), at every scaling alike
    assert [x for k, x in zip(keys, info.tolist()) if k[0] != "graded" or n < 511] == [0] * sum(k[0] != "graded" or n < 511 for k in keys)
    assert not torch.isnan(w).any() and not torch.isnan(V).any() and torch.isfinite(V).all()
    assert _same(V, Vb)
    wn, wbn = w.cpu().numpy(), wb.cpu().numpy()
    for k, (f, j) in enumerate(keys):
        with np.errstate(over="ignore"):
            assert np.array_equal(wn[k], np.ldexp(wbn[k], 2 * j)), (f, j)
    for k, (f, j) in enumerate(keys):
        if f in RANGE_FAMILIES and j == 0:
            chk = sr.check(B[k], wbn[k], Vb[k].cpu().numpy())
            assert chk.ok, (f, chk)
    vn = V.cpu().numpy()
    for k, (name, _) in enumerate(keys):
        if name == "diag_dbl_max":
            assert wn[k][0] == -DBL_MAX and wn[k][-1] == DBL_MAX and not wn[k][1:-1].any()
        elif name in ("ones_over", "neg_ones_over"):
            top = -1 if name == "ones_over" else 0
            assert wn[k][top] == (np.inf if top == -1 else -np.inf)
            others = np.delete(wn[k], top)
            assert np.abs(others).max() / DBL_MAX <= 8 * n * U  # zero eigenvalues, to n u ||A||
            assert np.abs(np.abs(vn[k][:, top]) - 1 / np.sqrt(n)).max() <= 4 * n * U
        elif name == "diag_1e307":
            assert (wn[k] == 1e307).all() and np.array_equal(vn[k], np.eye(n))
    # NaN and Inf stay local: info 1, NaN outputs, and the other matrices keep their bits
    w2, V2, info2 = cb.eig.syevj_batched(_batch(An), topo)
    expect = info.tolist()
    expect[pos_nan] = expect[pos_inf] = 1
    assert info2.tolist() == expect
    keep = [k for k in range(len(A)) if k not in (pos_nan, pos_inf)]
    assert _same(w2[keep], w[keep]) and _same(V2[keep], V[keep])
    assert torch.isnan(w2[[pos_nan, pos_inf]]).all() and torch.isnan(V2[[pos_nan, pos_inf]]).all()


@pytest.mark.parametrize("n", RANGE_N)
def test_odd_powers_of_two_meet_the_certified_bound(topo, n):
    """2^(2j+1) A with its largest entry near 2^-1019 (the bottom of the normal range, where the floor u ||A||_F is subnormal) and with
    ||A||_2 just below DBL_MAX: not an exact power-of-4 image of an in-range matrix, so gated by the certified bound on the scaled-back
    B = 2^-(2j+1) A_j (exact), w scaled back alike.  Lower down, w itself is subnormal and holds only a few bits."""
    fams = RANGE_FAMILIES if n < 512 else ("random",)
    A, keys = [], []
    for i, f in enumerate(fams):
        a = sr.family(f, n, 23 * n + i)[0]
        js = _powers(a)
        for p in (2 * js[1] + 1, 2 * js[-1] - 1):
            A.append(np.ldexp(a, p))
            keys.append((f, p))
    w, V, info = cb.eig.syevj_batched(_batch(A), topo)
    assert info.tolist() == [0] * len(A)
    assert torch.isfinite(w).all() and torch.isfinite(V).all()
    wn, vn = w.cpu().numpy(), V.cpu().numpy()
    for k, (f, p) in enumerate(keys):
        b = np.ldexp(A[k], -p)
        c = lr.certify(b, np.ldexp(wn[k], -p), vn[k])
        assert c.ok, (f, p, c)


def test_overflowing_pencil(topo):
    """[[d, x], [x, -d]], x = 0.6 DBL_MAX, d = 0.5 DBL_MAX: tau overflows without the normalisation; eigenvalues +-0.78 DBL_MAX"""
    d, x = 0.5 * DBL_MAX, 0.6 * DBL_MAX
    a = np.array([[d, x], [x, -d]])
    for n in (2, 65):
        m = np.zeros((n, n))
        m[:2, :2] = a
        w, V, info = cb.eig.syevj_batched(_batch([m]), topo)
        assert info.item() == 0 and torch.isfinite(w).all() and torch.isfinite(V).all()
        b = np.ldexp(m, -1024)
        c = lr.certify(b, np.ldexp(w[0].cpu().numpy(), -1024), V[0].cpu().numpy())
        assert c.ok, (n, c)
        assert abs(float(w[0, -1]) / DBL_MAX - np.hypot(0.5, 0.6)) <= 8 * U


# ---- chunk and loop edges ----------------------------------------------------------------------------------------------------------
def _launches(topo, fn):
    ctx = topo.context()
    torch.cuda.synchronize()
    ctx.reset_counters()
    out = fn()
    torch.cuda.synchronize()
    return ctx.counters().kernel_launches, out


def test_small_path_second_launch(topo):
    n, b = 8, 65535 + 5
    base = _batch([sr.family("random", n, 40 + i)[0] for i in range(7)])
    A = base[torch.arange(b, device="cuda") % 7]
    cnt, (w, V, info) = _launches(topo, lambda: cb.eig.syevj_batched(A, topo))
    assert cnt == 2
    assert info.eq(0).all()
    t0 = 65535 - 3
    wt, Vt, it = cb.eig.syevj_batched(A[t0:].contiguous(), topo)
    assert _same(wt, w[t0:]) and _same(Vt, V[t0:]) and it.equal(info[t0:])


def test_chunk_of_more_than_1024_matrices(topo):
    """n = 100, 1500 matrices in one chunk: syevj_sweep_end_kernel walks them in strides of 1024.  Matrices 0 .. 1199 are diagonal
    (one sweep), 1200 .. 1499 random: a miscount beyond index 1023 would stop the host early and leave these unconverged."""
    n, b = 100, 1500
    assert sr.chunk(n, b) == b
    diag = torch.diag_embed(torch.from_numpy(np.random.default_rng(5).standard_normal((1200, n)))).cuda()
    rand = _batch([sr.family("random", n, 300 + i)[0] for i in range(4)])[torch.arange(300, device="cuda") % 4]
    A = torch.cat([diag, rand])
    w, V, info = cb.eig.syevj_batched(A, topo)
    assert info.tolist() == [0] * b
    for k in (0, 1023, 1024, 1199, 1200, 1300, 1499):
        w1, V1, i1 = cb.eig.syevj_batched(A[k:k + 1], topo)
        assert _same(w1[0], w[k]) and _same(V1[0], V[k]) and i1.item() == 0, k
    chk = sr.check(A[1499].cpu().numpy(), w[1499].cpu().numpy(), V[1499].cpu().numpy())
    assert chk.ok, chk


# ---- poisoned workspaces ----------------------------------------------------------------------------------------------------------
class _Poisoned:
    """topo stand-in with its own context made under CAPITAL_POISON_WORKSPACE=1: every workspace it (re)allocates starts as NaN.
    context() frees the workspaces first (unless `keep`), so that every call of an entry point runs on fresh, poisoned buffers."""

    def __init__(self, topo, keep=False):
        self.grid, self.keep = topo.grid, keep
        old = os.environ.get("CAPITAL_POISON_WORKSPACE")
        os.environ["CAPITAL_POISON_WORKSPACE"] = "1"
        try:
            self.ctx = _lib.Context(topo.grid, torch.cuda.current_device(), torch.cuda.current_stream().cuda_stream or 0x1)
        finally:
            if old is None:
                del os.environ["CAPITAL_POISON_WORKSPACE"]
            else:
                os.environ["CAPITAL_POISON_WORKSPACE"] = old

    def context(self):
        if not self.keep:
            self.ctx.release_workspace()
        return self.ctx


@pytest.fixture(scope="module")
def poisoned(topo):
    p = _Poisoned(topo)
    yield p
    p.ctx.close()


def _all_same(xs, ys):
    for x, y in zip(xs, ys):
        assert torch.isfinite(x).all()
        assert _same(x, y)


@pytest.mark.parametrize("n", [33, 65, 100, 512])
def test_syevj_on_poisoned_workspace(topo, poisoned, n):
    A = _batch([sr.family(f, n, 3 * n + i)[0] for i, f in enumerate(("random", "cluster", "graded"))])
    _all_same(cb.eig.syevj_batched(A, poisoned)[:2], cb.eig.syevj_batched(A, topo)[:2])


def _pencil(n, seed):
    g = torch.Generator().manual_seed(seed)
    G = torch.randn(2, n, n, dtype=F64, generator=g)
    Bm = torch.stack([bs.spd_spectrum(n, 10.0 ** (2 + 2 * j), seed + j) for j in range(2)])
    return (G + G.mT).cuda(), Bm.cuda()


@pytest.mark.parametrize("n", [65, 200])
def test_batched_entry_points_on_poisoned_workspace(topo, poisoned, n):
    A, Bm = _pencil(n, 7 * n)
    rhs = torch.randn(2, n, 5, dtype=F64, generator=torch.Generator().manual_seed(n)).cuda()
    tall = torch.randn(2, 3 * n, n, dtype=F64, generator=torch.Generator().manual_seed(n + 1)).cuda()
    tall_rhs = torch.randn(2, 3 * n, 3, dtype=F64, generator=torch.Generator().manual_seed(n + 2)).cuda()

    def run(t):
        out = []
        for solver in ("torch", "jacobi"):
            for it in (1, 2, 3):
                out += cb.cholinv.eigh_batched(A, Bm, t, itype=it, eigensolver=solver)[:2]
        R, Ri, info = cb.cholinv.factor_batched(Bm, t)
        assert info.tolist() == [0, 0]
        out += [R, Ri, cb.cholinv.solve_batched(Ri, rhs, t), cb.cholinv.inverse_batched(Ri, t)]
        out += [cb.cholinv.sygst_batched(A, R, Ri, t, itype=it) for it in (1, 2, 3)]
        out += [cb.cholinv.apply_Rinv_batched(Ri, rhs, t), cb.cholinv.apply_RinvT_batched(Ri, rhs, t),
                cb.cholinv.apply_R_batched(R, rhs, t), cb.cholinv.apply_RT_batched(R, rhs, t)]
        for k in (1, 2, 3):
            Q, Rq, qi = cb.cacqr.factor_batched(tall, t, num_iter=k)
            assert qi.tolist() == [0, 0]
            out += [Q, Rq, cb.cacqr.lstsq_batched(Q, Rq, tall_rhs, t)]
        return out

    _all_same(run(poisoned), run(topo))


def test_stale_syevj_workspace_of_a_larger_n(topo):
    """512, then 65, then 512 on one context that keeps its (poisoned) workspace: each result equals a fresh context's"""
    held = _Poisoned(topo, keep=True)
    try:
        As = {n: _batch([sr.family(f, n, 5 * n + i)[0] for i, f in enumerate(("random", "rankdef", "graded"))]) for n in (512, 65)}
        for n in (512, 65, 512):
            fresh = _Poisoned(topo)
            try:
                _all_same(cb.eig.syevj_batched(As[n], held)[:2], cb.eig.syevj_batched(As[n], fresh)[:2])
            finally:
                fresh.ctx.close()
    finally:
        held.ctx.close()


# ---- eigh_batched with the Jacobi solver on ill-conditioned pencils -------------------------------------------------------------------
@pytest.mark.parametrize("itype", [1, 2, 3])
@pytest.mark.parametrize("n", [17, 129, 512])
def test_eigh_batched_jacobi_ill_conditioned(topo, n, itype):
    """kappa(B) = 1e8, and a graded D B D (D = diag(2^e), e from -6 to 6, of a kappa = 10 matrix; kappa about 1e5, so that the
    reference's eigvalsh still resolves B's smallest eigenvalue): the bounds the torch solver is gated on"""
    b8 = bs.spd_spectrum(n, 1e8, 5 * n + 1)
    e = bs.ramp_exponents(n, 6)
    d = torch.from_numpy(np.ldexp(1.0, e.numpy()))
    bg = bs.spd_spectrum(n, 10.0, 5 * n + 2) * d[:, None] * d[None, :]
    Bm = torch.stack([b8, bg]).cuda()
    G = torch.randn(2, n, n, dtype=F64, generator=torch.Generator().manual_seed(19 * n))
    A = (G + G.mT).cuda()
    w, X, info = cb.cholinv.eigh_batched(A, Bm, topo, itype=itype, eigensolver="jacobi")
    assert info.tolist() == [0, 0]
    a, bm, wn, xn = A.cpu().numpy(), Bm.cpu().numpy(), w.cpu().numpy(), X.cpu().numpy()
    for i in range(2):
        wr = sl.eigh(a[i], bm[i], type=itype, eigvals_only=True)
        eb = bs.EighBounds(a[i], bm[i], itype)
        assert (np.abs(wn[i] - wr) <= eb.eigenvalues(wr)).all(), (i, float(np.abs(wn[i] - wr).max()))
        assert bs.eigh_residual(a[i], bm[i], wn[i], xn[i], itype) <= eb.residual(wn[i], xn[i]), i
        assert bs.eigh_orthonormality(bm[i], xn[i], itype) <= eb.orthonormality(), i
