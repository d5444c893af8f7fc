"""CholInv and CholeskyQR on scaled, graded and ill-conditioned inputs given as data.

Cholesky is exactly equivariant under power-of-two scaling: R(2^(2k) A) = 2^k R(A), R(D A D) = R(A) D, R^-1(D A D) = D^-1 R^-1(A),
and every product of the schedule then scales by a uniform power of two.  So the factors of a scaled or graded input are checked
against the factors of the unscaled one from the same call path; ill-conditioned inputs against componentwise backward-error
bounds (conditioning_reference.py), which are scale-invariant and do not hide errors in small entries.  The scales are chosen so
that the products of neighbouring pivots, which the cluster base case forms two at a time, leave the double range on both sides.

The factors' own validators sum plain squares and overflow for entries above about 1e154, so these tests compute their own checks
on rescaled outputs instead."""
import math, os, subprocess, sys
import numpy as np
import pytest
import torch
import capital_b200 as cb
from capital_b200 import _lib
from oracle import capital_oracle as co
import conditioning_reference as cr

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GATE = 1.0  # both bound ratios: a correct factor stays below its bound (c = 1); LAPACK's stays below 0.03 (test_conditioning_cpu)


@pytest.fixture(scope="module")
def topo():
    return cb.topo.square(1, 0, 1)


def _rel(x, ref):
    return ((x - ref).abs().max() / ref.abs().max()).item()


def _potrf_trtri(ctx, a):
    """(status, R, Rinv) of capital_lapack_potrf_trtri_f64 on the symmetric n x n CUDA tensor a"""
    n = a.shape[0]
    ld = n + (n & 1)
    R = torch.zeros((n, ld), dtype=torch.float64, device="cuda")
    Ri = torch.zeros_like(R)
    acm = a.t().contiguous()
    st = _lib.lib().capital_lapack_potrf_trtri_f64(ctx.handle, n, acm.data_ptr(), n, R.data_ptr(), ld, Ri.data_ptr(), ld)
    torch.cuda.synchronize()
    return st, R.t()[:n], Ri.t()[:n]


# diagonal entries n 4^k from about 1e-250 to 1e250; |k| >= 270 puts a b and l^2 of the pivot pairs outside the double range
SCALES = [-412, -330, -270, -12, 12, 270, 330, 412]
SMALL = (-12, 12)  # every pivot, and every pair's det, inside fast_rsqrt's FP32-seeded range


@pytest.mark.parametrize("n", [64, 96, 128, 256, 512, 640, 777])
def test_potrf_trtri_uniform_scaling(topo, n):
    """The base-case factor (leaf kernel n <= 64, cluster kernel 128..512, and mixed recursions) of 2^(2k) A against that of A."""
    ctx = topo.context()
    a = torch.from_numpy(co.spd_global(n)).cuda()
    st, R0, X0 = _potrf_trtri(ctx, a)
    assert st == _lib.OK
    bad, lines = [], []
    for k in SCALES:
        st, R, X = _potrf_trtri(ctx, cr.scaled(a, k))
        Rs, Xs = R * math.ldexp(1.0, -k), X * math.ldexp(1.0, k)
        eR, eX = _rel(Rs, R0), _rel(Xs, X0)
        same = torch.equal(Rs, R0) and torch.equal(Xs, X0)
        lines.append(f"k={k}: status={st} errR={eR:.1e} errRinv={eX:.1e} bit-identical={same}")
        # in fast_rsqrt's range the FP32 seed of the H100 (MUFU.RSQ) is exactly equivariant under 4^k: the same bits
        if st != _lib.OK or not (eR <= 1e-14 and eX <= 1e-14) or (k in SMALL and not same):
            bad.append(lines[-1])
    print(f"\n[scaling] n={n}: " + " | ".join(lines))
    assert not bad, bad


@pytest.mark.parametrize("n,kernel", [(64, "leaf"), (256, "cluster")])
@pytest.mark.parametrize("k", [-412, 0, 412])
def test_not_spd_still_reported_at_extreme_scales(topo, n, kernel, k):
    """A negative diagonal entry, and a zero row and column at an even and at an odd pivot, are CAPITAL_ERR_NOT_SPD at any scale."""
    ctx = topo.context()
    base = torch.from_numpy(co.spd_global(n)).cuda()
    cases = {}
    a = base.clone(); a[40, 40] = -5.0; cases["A[40,40]=-5"] = a
    for p in (40, 41):
        a = base.clone(); a[p, :] = 0.0; a[:, p] = 0.0; cases[f"zero pivot {p}"] = a
    for name, a in cases.items():
        st, _, _ = _potrf_trtri(ctx, cr.scaled(a, k))
        assert st == _lib.ERR_NOT_SPD, (kernel, name, k, st)


# ---- cholinv.factor with user data --------------------------------------------------------------------------------------------
_CACHE = {}


def _spectrum(n, kappa):
    if (n, kappa) not in _CACHE:
        _CACHE[(n, kappa)] = cr.spd_spectrum(n, kappa, 1234, device="cuda")
    return _CACHE[(n, kappa)]


def _bc_mult(n):
    """bc_mult_dim that makes the base case 512 on one GPU"""
    return -int(np.log2(n // 512)) if n % 512 == 0 else 0


def _factor(topo, a, ci, split, serialize=False):
    n = a.shape[0]
    A = cb.matrix(n, n, 1, 1, data=a.t().contiguous().view(-1))
    args = cb.cholinv.info(ci, split, _bc_mult(n), "U", serialize=serialize)
    cb.cholinv.factor(A, args, topo)
    return args, cb.cholinv.construct_R(args), cb.cholinv.construct_Rinv(args)


def _skipped_split(n, ci, split):
    """the top-level split point when complete_inv = 0 leaves Rinv12 zero, else None"""
    return n >> split if ci == 0 and n > 512 else None


@pytest.mark.parametrize("n", [512, 777, 2048, 4096])
@pytest.mark.parametrize("ci", [0, 1])
@pytest.mark.parametrize("split", [1, 2])
def test_cholinv_prescribed_spectrum_bounds(topo, n, ci, split):
    lines = []
    for kappa in (1e2, 1e7, 1e11):
        a = _spectrum(n, kappa)
        _, R, X = _factor(topo, a, ci, split)
        rc, ri = cr.chol_ratio(a, R), cr.inv_ratio(R, X, _skipped_split(n, ci, split))
        lines.append(f"kappa={kappa:.0e}: R ratio {rc:.2e}, Rinv ratio {ri:.2e}")
        assert rc <= GATE and ri <= GATE, lines[-1]
    print(f"\n[spectrum] n={n} ci={ci} split={split}: " + " | ".join(lines))


def _ramp(n):
    """the exponent profile and 2^e on the device"""
    e = cr.ramp_exponents(n, 300)
    return e, cr.pow2(e, "cuda")


@pytest.mark.parametrize("n", [512, 777, 2048, 4096])
@pytest.mark.parametrize("ci", [0, 1])
@pytest.mark.parametrize("split", [1, 2])
def test_cholinv_graded(topo, n, ci, split):
    """D A D with D = diag(2^e), e rising from -300 to 300: R(D A D) D^-1 and D R^-1(D A D) against R(A) and R^-1(A) of the same
    path, and a graded kappa = 1e7 core against the bounds."""
    a = torch.from_numpy(co.spd_global(n)).cuda()
    e, d = _ramp(n)
    lo, hi = cr.pair_product_log2(a, e)
    assert lo < -1022 and hi > 1024, (lo, hi)  # neighbouring diagonal products leave the double range on both sides
    _, R0, X0 = _factor(topo, a, ci, split)
    _, R, X = _factor(topo, cr.graded(a, e), ci, split)
    eR = _rel(R / d[None, :], R0)
    eX = _rel(X * d[:, None], X0)
    core = _spectrum(n, 1e7)
    ag = cr.graded(core, e)
    _, Rg, Xg = _factor(topo, ag, ci, split)
    rc, ri = cr.chol_ratio(ag, Rg), cr.inv_ratio(Rg, Xg, _skipped_split(n, ci, split))
    print(f"\n[graded] n={n} ci={ci} split={split}: errR={eR:.1e} errRinv={eX:.1e} | kappa=1e7 core: R ratio {rc:.2e}, "
          f"Rinv ratio {ri:.2e}")
    assert eR <= 1e-14 and eX <= 1e-14
    assert rc <= GATE and ri <= GATE


@pytest.mark.parametrize("n", [777, 2048])
def test_solve_and_inverse_of_a_graded_factor(topo, n):
    """(D A D)^-1 = D^-1 A^-1 D^-1: D X(D A D, D B) against X(A, B), and D inverse(D A D) D against inverse(A)."""
    a = torch.from_numpy(co.spd_global(n)).cuda()
    e, d = _ramp(n)
    B =torch.from_numpy(np.random.default_rng(n).standard_normal((n, 3))).cuda()
    out = []
    for mat, rhs in ((a, B), (cr.graded(a, e), B * d[:, None])):
        args, _, _ = _factor(topo, mat, 0, 1, serialize=True)
        out.append((cb.cholinv.solve(args, rhs, topo), cb.cholinv._expand(cb.cholinv.inverse(args, topo), n, True)))
    (X0, I0), (X, I) = out
    eX = _rel(X * d[:, None], X0)
    eI = _rel(I * d[:, None] * d[None, :], I0)
    print(f"\n[graded solve/inverse] n={n}: errX={eX:.1e} errInv={eI:.1e}")
    assert eX <= 1e-13 and eI <= 1e-13


# ---- CholeskyQR --------------------------------------------------------------------------------------------------------------
def _cacqr(A_data, m, n, num_iter):
    topo = cb.topo.rect(1, 0, 1)
    A = cb.matrix(n, m, 1, 1, data=A_data.contiguous())
    args = cb.cacqr.info(num_iter, cb.cholinv.info(0, 1, 0, "U"))
    cb.cacqr.factor(A, args, topo)
    B = torch.from_numpy(np.random.default_rng(m).standard_normal((m, 2))).cuda()
    return cb.cacqr.construct_Q(args).clone(), cb.cacqr.construct_R(args), cb.cacqr.lstsq(args, B, topo)


# Gram diagonal ~ m 4^k / 3: its neighbouring products leave the double range for k <= -264 and k >= 249 at m = 2^17
@pytest.mark.parametrize("m,n", [(4096, 64), (1 << 17, 256)])
@pytest.mark.parametrize("num_iter", [1, 2, 3])
def test_cacqr_uniform_scaling(m, n, num_iter):
    """Q(A 2^k) against Q(A), R against 2^k R(A), and the least-squares solution against 2^-k X(A)."""
    topo = cb.topo.rect(1, 0, 1)
    A = cb.matrix(n, m, 1, 1).distribute_random(topo, 0)
    Q0, R0, X0 = _cacqr(A.data, m, n, num_iter)
    lines = []
    for k in (-300, 270):
        Q, R, X = _cacqr(A.data * math.ldexp(1.0, k), m, n, num_iter)
        eQ, eR, eX = _rel(Q, Q0), _rel(R * math.ldexp(1.0, -k), R0), _rel(X * math.ldexp(1.0, k), X0)
        lines.append(f"k={k}: errQ={eQ:.1e} errR={eR:.1e} errX={eX:.1e}")
        assert eQ <= 1e-13 and eR <= 1e-13 and eX <= 1e-12, lines[-1]
    print(f"\n[cacqr scaling] m={m} n={n} num_iter={num_iter}: " + " | ".join(lines))


@pytest.mark.parametrize("m,n", [(4096, 64), (1 << 17, 256)])
@pytest.mark.parametrize("num_iter", [1, 2])
def test_cacqr_column_grading(m, n, num_iter):
    """A D with D = diag(2^e), e from -300 to 300: Q unchanged, R = R(A) D, X = D^-1 X(A).  (Shifted CholeskyQR3 is left out: its
    shift is meant for kappa(A) < 1/u, and a graded A is far past that.)"""
    topo = cb.topo.rect(1, 0, 1)
    A = cb.matrix(n, m, 1, 1).distribute_random(topo, 0)
    e, d = _ramp(n)
    Q0, R0, X0 = _cacqr(A.data, m, n, num_iter)
    G = A.view2d().t() @ A.view2d()
    lo, hi = cr.pair_product_log2(G, e)
    assert lo < -1022 and hi > 1024, (lo, hi)
    AD = (A.data.view(n, m) * d[:, None]).view(-1)  # column-major: row j of the view is column j
    Q, R, X = _cacqr(AD, m, n, num_iter)
    eQ, eR, eX = _rel(Q, Q0), _rel(R / d[None, :], R0), _rel(X * d[:, None], X0)
    print(f"\n[cacqr graded] m={m} n={n} num_iter={num_iter}: errQ={eQ:.1e} errR={eR:.1e} errX={eX:.1e}")
    assert eQ <= 1e-13 and eR <= 1e-13 and eX <= 1e-12


# ---- grids ---------------------------------------------------------------------------------------------------------------------
def test_grids_at_an_extreme_scale_with_ranks_sharing_one_gpu():
    """cholinv on the 2x1x1 grid and CholeskyQR2 on the 2-rank 1D grid, inputs scaled past the pivot pairs' range, every rank on
    cuda:0 (tests/mp_worker_conditioning.py)."""
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1",
           "--master-port", "29881", os.path.join(ROOT, "tests", "mp_worker_conditioning.py")]
    env = dict(os.environ, CAPITAL_MP_SAME_DEVICE="1")
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=600, env=env)
    assert r.returncode == 0 and "MP_OK" in r.stdout, r.stdout[-3000:] + r.stderr[-3000:]
    print("\n" + r.stdout.strip()[-1500:])
