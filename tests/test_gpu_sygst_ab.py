"""cholinv::sygst for itype 2 and 3 on the GPU: A B x = lambda x and B A x = lambda x reduced to C = R A R^T with the CholInv factor of
B (capital_cholinv_sygst_ab_f64), and the products with the factor, X = R B and X = R^T B (capital_cholinv_apply_r_f64), on one GPU
and on the square grids."""
import ctypes as C
import os, subprocess, sys
import numpy as np
import pytest
import scipy.linalg as sla
import torch
import capital_b200 as cb
from capital_b200 import _lib
from sygst_reference import U
from sygst_ab_reference import dsygst_full

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def topo():
    return cb.topo.square(1, 0, 1)


def _full(Cl, n, serialize):
    """n x n view of the output: the upper triangle (zeros below) when packed, the full block when rect"""
    if not serialize:
        return Cl.view(n, n).t()
    out = torch.zeros(n, n, dtype=torch.float64, device=Cl.device)
    iu = torch.triu_indices(n, n, device=Cl.device)
    out[iu[0], iu[1]] = Cl[(iu[1] * (iu[1] + 1)) // 2 + iu[0]]
    return out


def _random_symmetric(n, seed):
    g = torch.randn(n, n, dtype=torch.float64, device="cuda", generator=torch.Generator("cuda").manual_seed(seed))
    a = g + g.t()
    return cb.matrix(n, n, 1, 1, data=a.t().contiguous().view(-1))


def _bound(a, r):
    """the elementwise first-order rounding bound of the n^3 form (sygst_ab_reference.bound), on the device"""
    m = r.abs()
    return 2 * a.shape[0] * U * (m @ a.abs() @ m.t())


_refs = {}


def _reference(n, seed):
    """B = the generator's SPD matrix, its R from the library, A random symmetric; dsygst's C and the bound, once per (n, seed)"""
    if (n, seed) not in _refs:
        topo = cb.topo.square(1, 0, 1)
        B = cb.matrix(n, n, 1, 1).distribute_symmetric(topo)
        args = cb.cholinv.info(1, 1, -2, "U")
        cb.cholinv.factor(B, args, topo)
        R = cb.cholinv.construct_R(args)
        A = _random_symmetric(n, seed)
        a = A.view2d()
        ref = torch.from_numpy(dsygst_full(a.cpu().numpy(), R.cpu().numpy(), 2)).cuda()
        _refs[(n, seed)] = (B, A, ref, _bound(a, R))
    return _refs[(n, seed)]


@pytest.mark.parametrize("n", [96, 1000, 4096])
@pytest.mark.parametrize("ci", [0, 1])
@pytest.mark.parametrize("serialize", [True, False])
def test_sygst_ab_matches_dsygst(topo, n, ci, serialize):
    B, A, ref, bnd = _reference(n, 5)
    args = cb.cholinv.info(ci, 1, -2, "U", serialize=serialize)
    cb.cholinv.factor(B, args, topo)
    Cl = cb.cholinv.sygst(A, args, topo, itype=2)
    assert Cl.is_cuda and Cl.shape == args.Rinv.shape
    assert torch.equal(cb.cholinv.sygst(A, args, topo, itype=3), Cl)  # the same C, deterministic
    M = _full(Cl, n, serialize)
    if serialize:
        err, lim = (M - torch.triu(ref)).abs(), torch.triu(bnd)
    else:
        assert torch.equal(M, M.t())  # exactly symmetric
        err, lim = (M - ref).abs(), bnd
    assert bool((err <= lim).all()), float((err / lim).max())
    # host pointers: R, A and C on the host give the same bits
    h = cb.cholinv.info(ci, 1, -2, "U", serialize=serialize)
    h.R, h.Rinv, h.local_dim, h.global_dim = args.R.cpu(), args.Rinv.cpu(), n, n
    Ch = cb.cholinv.sygst(cb.matrix(n, n, 1, 1, data=A.data.cpu()), h, topo, itype=2)
    assert not Ch.is_cuda and Ch.is_pinned() and torch.equal(Ch, Cl.cpu())


@pytest.mark.parametrize("serialize", [True, False])
def test_upper_triangle_of_A_is_never_read(topo, serialize):
    n = 1000
    B = cb.matrix(n, n, 1, 1).distribute_symmetric(topo)
    A = _random_symmetric(n, 3)
    poisoned = A.view2d().clone()
    poisoned[torch.triu(torch.ones(n, n, dtype=torch.bool, device="cuda"), 1)] = float("nan")
    Ap = cb.matrix(n, n, 1, 1, data=poisoned.t().contiguous().view(-1))
    args = cb.cholinv.info(1, 1, -2, "U", serialize=serialize)
    cb.cholinv.factor(B, args, topo)
    assert torch.equal(cb.cholinv.sygst(Ap, args, topo, itype=2), cb.cholinv.sygst(A, args, topo, itype=2))


@pytest.mark.parametrize("ci", [0, 1])
def test_flop_count_is_n_cubed(topo, ci):
    """W = R U counts n^3 / 3 (two triangular operands, upper output), the two-class product 2 n^3 / 3 (gemm_tn.cu's counter, exact in
    the structure).  Only R is read, so a skipped Rinv12 adds nothing; the dense R A R^T would count 4 n^3."""
    n = 4096
    B = cb.matrix(n, n, 1, 1).distribute_symmetric(topo)
    args = cb.cholinv.info(ci, 1, -3, "U")
    cb.cholinv.factor(B, args, topo)
    A = _random_symmetric(n, 7)
    ctx = topo.context()
    ctx.reset_counters()
    cb.cholinv.sygst(A, args, topo, itype=3)
    torch.cuda.synchronize()
    assert abs(ctx.counters().gemm_flops / n ** 3 - 1) <= 1e-9


def test_large_matches_torch(topo):
    """n = 16384 against torch's dense R @ A @ R.T.  Bound: twice the largest entry of the first-order rounding bound 2 n u |R| |A| |R|^T
    (one bound for each of the two computations), on the largest difference."""
    n = 16384
    B = cb.matrix(n, n, 1, 1).distribute_symmetric(topo)
    args = cb.cholinv.info(1, 1, -5, "U")
    cb.cholinv.factor(B, args, topo)
    A = _random_symmetric(n, 13)
    ctx = topo.context()
    ctx.reset_counters()
    Cl = cb.cholinv.sygst(A, args, topo, itype=2)
    torch.cuda.synchronize()
    assert abs(ctx.counters().gemm_flops / n ** 3 - 1) <= 1e-9
    M = _full(Cl, n, True)
    del Cl
    R = cb.cholinv.construct_R(args)
    a = A.view2d()
    ref = R @ a @ R.t()
    lim = 2 * _bound(a, R).max().item()
    err = (M - torch.triu(ref)).abs().max().item()
    print(f"\n[sygst_ab] n={n}: max |C - C_torch| = {err:.2e} (bound {lim:.2e}), max |C| = {ref.abs().max().item():.2e}")
    assert err <= lim


@pytest.mark.parametrize("itype", [2, 3])
def test_eigenpairs_end_to_end(topo, itype):
    """factor B, sygst A, torch.linalg.eigh(C), back-transform: itype 2 (A B x = lambda x) with x = apply_Rinv(y), normalised
    X^T B X = I; itype 3 (B A x = lambda x) with x = apply_RT(y), normalised X^T B^-1 X = I."""
    n = 1000
    Bm = cb.matrix(n, n, 1, 1).distribute_symmetric(topo)
    Am = cb.matrix(n, n, 1, 1).distribute_symmetric(topo, False)
    args = cb.cholinv.info(0, 1, -2, "U", serialize=False)
    cb.cholinv.factor(Bm, args, topo)
    Cm = cb.cholinv.sygst(Am, args, topo, itype=itype).view(n, n).t()
    lam, Y = torch.linalg.eigh(Cm)
    Y = Y.contiguous()
    a, b = Am.view2d(), Bm.view2d()
    scale = torch.linalg.matrix_norm(a, 2) * torch.linalg.matrix_norm(b, 2)  # ||A B||, ||B A|| <= ||A|| ||B||
    if itype == 2:
        X = cb.cholinv.apply_Rinv(args, Y, topo)
        res = (a @ (b @ X) - X * lam).abs().max() / (scale * X.abs().max())
        G = X.t() @ b @ X
    else:
        X = cb.cholinv.apply_RT(args, Y, topo)
        res = (b @ (a @ X) - X * lam).abs().max() / (scale * X.abs().max())
        W = cb.cholinv.apply_RinvT(args, X, topo)  # R^-T X: X^T B^-1 X = W^T W
        G = W.t() @ W
    ref = sla.eigh(a.cpu().numpy(), b.cpu().numpy(), type=itype, eigvals_only=True)
    assert np.abs(lam.cpu().numpy() - ref).max() <= 1e-13 * np.abs(ref).max() * n ** 0.5
    orth = (G - torch.eye(n, dtype=torch.float64, device="cuda")).abs().max()
    print(f"\n[sygst_ab] itype {itype} eigenpairs n={n}: residual {res.item():.1e}, |normalisation - I| = {orth.item():.1e}")
    assert res <= 1e-13 and orth <= 1e-12


@pytest.mark.parametrize("ci", [0, 1])
@pytest.mark.parametrize("serialize", [True, False])
@pytest.mark.parametrize("k", [1, 33])
def test_apply_r_matches_torch(topo, ci, serialize, k):
    n = 3000
    B = cb.matrix(n, n, 1, 1).distribute_symmetric(topo)
    args = cb.cholinv.info(ci, 1, -3, "U", serialize=serialize)
    cb.cholinv.factor(B, args, topo)
    R = cb.cholinv.construct_R(args)
    rhs = torch.randn(n, k, dtype=torch.float64, device="cuda", generator=torch.Generator("cuda").manual_seed(k))
    X = cb.cholinv.apply_R(args, rhs, topo)
    XT = cb.cholinv.apply_RT(args, rhs, topo)
    for got, F in ((X, R), (XT, R.t())):
        # each entry is a dot product of at most n terms: both results lie within n u |F| |rhs| of the exact one, to first order
        lim = 2 * n * U * (F.abs() @ rhs.abs())
        assert bool(((got - F @ rhs).abs() <= lim).all())
    assert torch.equal(cb.cholinv.apply_R(args, rhs[:, 0], topo), cb.cholinv.apply_R(args, rhs[:, :1], topo)[:, 0])  # a vector
    # in place (X = B) through the C ABI, and host pointers: the same bits
    ctx = topo.context()
    ca = args._c()
    P = _lib.UPPERTRI_PACKED if serialize else _lib.RECT
    for trans, want in ((0, X), (1, XT)):
        buf = rhs.t().clone(memory_format=torch.contiguous_format)  # a copy: for k = 1 .t() is already contiguous
        ctx.check(_lib.lib().capital_cholinv_apply_r_f64(ctx.handle, n, C.byref(ca), P, args.R.data_ptr(), trans, k, buf.data_ptr(), n,
                                                         buf.data_ptr(), n))
        assert torch.equal(buf.t(), want)
    h = cb.cholinv.info(ci, 1, -3, "U", serialize=serialize)
    h.R, h.Rinv, h.local_dim, h.global_dim = args.R.cpu(), args.Rinv.cpu(), n, n
    assert torch.equal(cb.cholinv.apply_R(h, rhs.cpu(), topo), X.cpu())
    assert torch.equal(cb.cholinv.apply_RT(h, rhs.cpu(), topo), XT.cpu())
    # R (R^-1 B) = B and R^T (R^-T B) = B
    for fwd, back in ((cb.cholinv.apply_Rinv, cb.cholinv.apply_R), (cb.cholinv.apply_RinvT, cb.cholinv.apply_RT)):
        Z = back(args, fwd(args, rhs, topo), topo)
        assert ((Z - rhs).abs().max() <= 1e-10 * rhs.abs().max()).item()


def test_c_abi_rejects_bad_arguments(topo):
    n = 512
    B = cb.matrix(n, n, 1, 1).distribute_symmetric(topo)
    A = _random_symmetric(n, 1)
    args = cb.cholinv.info(0, 1, -2, "U")
    cb.cholinv.factor(B, args, topo)
    out = torch.empty_like(args.R)
    ctx = topo.context()
    ca = args._c()
    L = _lib.lib()
    P = _lib.UPPERTRI_PACKED
    assert L.capital_cholinv_sygst_ab_f64(ctx.handle, n, C.byref(ca), P, None, A.data.data_ptr(), out.data_ptr()) == _lib.ERR_INVALID
    assert L.capital_cholinv_sygst_ab_f64(ctx.handle, n, C.byref(ca), P, args.R.data_ptr(), None, out.data_ptr()) == _lib.ERR_INVALID
    for bad_out in (args.R.data_ptr() + 8, A.data.data_ptr() + 8 * n):
        assert L.capital_cholinv_sygst_ab_f64(ctx.handle, n, C.byref(ca), P, args.R.data_ptr(), A.data.data_ptr(), bad_out) \
            == _lib.ERR_INVALID
    # Rinv is not an argument: C may overlap it
    assert L.capital_cholinv_sygst_ab_f64(ctx.handle, n, C.byref(ca), P, args.R.data_ptr(), A.data.data_ptr(),
                                          args.Rinv.data_ptr()) == _lib.OK
    for bad in (_lib.CholinvArgs(0, 0, -2, b"U"), _lib.CholinvArgs(0, 1, -2, b"L")):
        assert L.capital_cholinv_sygst_ab_f64(ctx.handle, n, C.byref(bad), P, args.R.data_ptr(), A.data.data_ptr(), out.data_ptr()) \
            == _lib.ERR_INVALID
    assert L.capital_cholinv_sygst_ab_f64(ctx.handle, n, C.byref(ca), 7, args.R.data_ptr(), A.data.data_ptr(), out.data_ptr()) \
        == _lib.ERR_INVALID
    x = torch.zeros(n, dtype=torch.float64, device="cuda")
    for trans in (-1, 2):
        assert L.capital_cholinv_apply_r_f64(ctx.handle, n, C.byref(ca), P, args.R.data_ptr(), trans, 1, x.data_ptr(), n, x.data_ptr(),
                                             n) == _lib.ERR_INVALID
    assert L.capital_cholinv_apply_r_f64(ctx.handle, n, C.byref(ca), P, None, 0, 1, x.data_ptr(), n, x.data_ptr(), n) == _lib.ERR_INVALID
    assert L.capital_cholinv_apply_r_f64(ctx.handle, n, C.byref(ca), P, args.R.data_ptr(), 0, 1, x.data_ptr(), n - 1, x.data_ptr(), n) \
        == _lib.ERR_INVALID


def _run_grid(nproc, same_device, timeout=1500):
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={nproc}", "--master-addr", "127.0.0.1",
           "--master-port", str(29781 + nproc), os.path.join(ROOT, "tests", "mp_worker_sygst_ab.py")]
    env = dict(os.environ)
    if same_device:
        env["CAPITAL_MP_SAME_DEVICE"] = "1"
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=timeout, env=env)
    assert r.returncode == 0 and "MP_OK" in r.stdout, r.stdout[-3000:] + r.stderr[-3000:]
    print("\n" + r.stdout.strip()[-2000:])


@pytest.mark.parametrize("nproc", [2, 4, 8])
def test_grid_sygst_ab_with_ranks_sharing_one_gpu(nproc):
    """2x1x1, 1x2x2 and 2x2x2 with every rank on cuda:0 (mp_worker_sygst_ab.py)."""
    _run_grid(nproc, True)


@pytest.mark.parametrize("nproc", [2, 4, 8])
def test_grid_sygst_ab_on_separate_gpus(nproc):
    if torch.cuda.device_count() < nproc:
        pytest.skip(f"needs {nproc} GPUs")
    _run_grid(nproc, False)
