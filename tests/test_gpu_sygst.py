"""cholinv::sygst on the GPU: A x = lambda B x reduced to C = R^-T A R^-1 with the CholInv factors of B (capital_cholinv_sygst_f64),
and the two halves of the solve (capital_cholinv_apply_rinv_f64), on one GPU and on the square grids."""
import ctypes as C
import os, subprocess, sys
import numpy as np
import pytest
import scipy.linalg as sla
import torch
import capital_b200 as cb
from capital_b200 import _lib
from sygst_reference import U, dsygst_full

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


def _bound(a, ri):
    """the elementwise first-order rounding bound of the n^3 form (sygst_reference.bound), on the device"""
    m = ri.abs()
    return 2 * a.shape[0] * U * (m.t() @ a.abs() @ m)


_refs = {}


def _reference(n, split, seed):
    """B = the generator's SPD matrix, its R from the library, A random symmetric; dsygst's C and the bound, once per (n, split, seed)"""
    if (n, split, seed) not in _refs:
        topo = cb.topo.square(1, 0, 1)
        B = cb.matrix(n, n, 1, 1).distribute_symmetric(topo)
        args = cb.cholinv.info(1, split, -2, "U")
        cb.cholinv.factor(B, args, topo)
        R = cb.cholinv.construct_R(args)
        A = _random_symmetric(n, seed)
        a = A.view2d()
        ref = torch.from_numpy(dsygst_full(a.cpu().numpy(), R.cpu().numpy())).cuda()
        _refs[(n, split, seed)] = (B, A, ref, _bound(a, torch.linalg.inv(R)))
    return _refs[(n, split, seed)]


@pytest.mark.parametrize("n", [96, 1000, 4096])
@pytest.mark.parametrize("ci", [0, 1])
@pytest.mark.parametrize("split", [1, 2])
@pytest.mark.parametrize("serialize", [True, False])
def test_sygst_matches_dsygst(topo, n, ci, split, serialize):
    B, A, ref, bnd = _reference(n, split, 5)
    args = cb.cholinv.info(ci, split, -2, "U", serialize=serialize)
    cb.cholinv.factor(B, args, topo)
    Cl = cb.cholinv.sygst(A, args, topo)
    assert Cl.is_cuda and Cl.shape == args.Rinv.shape
    M = _full(Cl, n, serialize)
    if serialize:
        err, lim = (M - torch.triu(ref)).abs(), torch.triu(bnd)
    else:
        assert torch.equal(M, M.t())  # exactly symmetric
        err, lim = (M - ref).abs(), bnd
    assert bool((err <= lim).all()), float((err / lim).max())
    # host pointers: factors, A and C on the host give the same bits
    h = cb.cholinv.info(ci, split, -2, "U", serialize=serialize)
    h.R, h.Rinv, h.local_dim, h.global_dim = args.R.cpu(), args.Rinv.cpu(), n, n
    Ch = cb.cholinv.sygst(cb.matrix(n, n, 1, 1, data=A.data.cpu()), h, topo)
    assert not Ch.is_cuda and Ch.is_pinned() and torch.equal(Ch, Cl.cpu())


@pytest.mark.parametrize("split", [1, 2])
@pytest.mark.parametrize("serialize", [True, False])
def test_complete_and_rebuilt_rinv12_give_the_same_bits(topo, split, serialize):
    n = 3000
    B = cb.matrix(n, n, 1, 1).distribute_symmetric(topo)
    A = _random_symmetric(n, 11)
    outs = []
    for ci in (0, 1):
        args = cb.cholinv.info(ci, split, -3, "U", serialize=serialize)
        cb.cholinv.factor(B, args, topo)
        outs.append(cb.cholinv.sygst(A, args, topo))
    assert torch.equal(outs[0], outs[1])


@pytest.mark.parametrize("ci", [0, 1])
@pytest.mark.parametrize("serialize", [True, False])
def test_upper_triangle_of_A_is_never_read(topo, ci, serialize):
    n = 1000
    B = cb.matrix(n, n, 1, 1).distribute_symmetric(topo)
    A = _random_symmetric(n, 3)
    poisoned = A.view2d().clone()
    poisoned[torch.triu(torch.ones(n, n, dtype=torch.bool, device="cuda"), 1)] = float("nan")
    Ap = cb.matrix(n, n, 1, 1, data=poisoned.t().contiguous().view(-1))
    args = cb.cholinv.info(ci, 1, -2, "U", serialize=serialize)
    cb.cholinv.factor(B, args, topo)
    assert torch.equal(cb.cholinv.sygst(Ap, args, topo), cb.cholinv.sygst(A, args, topo))


def _expected_flops(n, ci, split):
    """what the gemm_flops counter adds for one sygst call, from its formula (gemm_tn.cu: a product of two triangular operands counts
    2 m n k / 3, halved for C_UPPER on a square output; per operand class): V = U Rinv n^3 / 3, then the two-class product 2 n^3 / 3.
    A rebuilt Rinv12 adds the factor's two products, s2 s1 (s1 + 1) and s1 s2 (s2 + 1).  The counter is exact in the structure, not
    tile-rounded, so the only slack allowed is floating-point rounding of the sums; the 4 n^3 / 3 form would count a third more."""
    f = n ** 3 / 3 + 2 * n ** 3 / 3
    if not ci:
        s1 = n >> split
        s2 = n - s1
        f += s2 * s1 * (s1 + 1) + s1 * s2 * (s2 + 1)
    return f


@pytest.mark.parametrize("ci", [0, 1])
def test_flop_count_is_n_cubed(topo, ci):
    n = 4096
    B = cb.matrix(n, n, 1, 1).distribute_symmetric(topo)
    args = cb.cholinv.info(ci, 1, -3, "U")
    cb.cholinv.factor(B, args, topo)
    A = _random_symmetric(n, 7)
    ctx = topo.context()
    ctx.reset_counters()
    cb.cholinv.sygst(A, args, topo)
    torch.cuda.synchronize()
    flops = ctx.counters().gemm_flops
    expect = _expected_flops(n, ci, 1)
    assert abs(flops - expect) <= 1e-9 * expect, (flops, expect)
    if ci:
        assert abs(flops / n ** 3 - 1) <= 1e-9


@pytest.mark.parametrize("ci", [0, 1])
def test_large_matches_torch_trsm(topo, ci):
    """n = 16384 against torch's TRSM reference R^-T (A R^-1).  Bound: twice the largest entry of the first-order rounding bound
    2 n u |Rinv|^T |A| |Rinv| of the n^3 form (one bound for each of the two computations), on the largest difference."""
    n = 16384
    B = cb.matrix(n, n, 1, 1).distribute_symmetric(topo)
    args = cb.cholinv.info(ci, 1, -5, "U")
    cb.cholinv.factor(B, args, topo)
    A = _random_symmetric(n, 13)
    ctx = topo.context()
    ctx.reset_counters()
    Cl = cb.cholinv.sygst(A, args, topo)
    torch.cuda.synchronize()
    assert abs(ctx.counters().gemm_flops - _expected_flops(n, ci, 1)) <= 1e-9 * n ** 3
    M = _full(Cl, n, True)
    del Cl
    R = cb.cholinv.construct_R(args)
    a = A.view2d()
    T = torch.linalg.solve_triangular(R, a, upper=True, left=False)     # A R^-1
    ref = torch.linalg.solve_triangular(R.t(), T, upper=False)          # R^-T A R^-1
    del T
    lim = 2 * _bound(a, torch.linalg.solve_triangular(R, torch.eye(n, dtype=torch.float64, device="cuda"), upper=True)).max().item()
    err = (M - torch.triu(ref)).abs().max().item()
    print(f"\n[sygst] n={n} ci={ci}: max |C - C_torch| = {err:.2e} (bound {lim:.2e}), max |C| = {ref.abs().max().item():.2e}")
    assert err <= lim


def test_eigenpairs_end_to_end(topo):
    """factor B, sygst A, torch.linalg.eigh(C), back-transform with apply_Rinv: the generalized eigenpairs of (A, B)."""
    n = 1000
    Bm = cb.matrix(n, n, 1, 1).distribute_symmetric(topo)
    Am = cb.matrix(n, n, 1, 1).distribute_symmetric(topo, False)
    args = cb.cholinv.info(0, 1, -2, "U", serialize=False)
    cb.cholinv.factor(Bm, args, topo)
    Cm = cb.cholinv.sygst(Am, args, topo).view(n, n).t()
    lam, Y = torch.linalg.eigh(Cm)
    X = cb.cholinv.apply_Rinv(args, Y.contiguous(), topo)
    a, b = Am.view2d(), Bm.view2d()
    ref = sla.eigh(a.cpu().numpy(), b.cpu().numpy(), eigvals_only=True)
    scale = np.abs(ref).max()
    assert np.abs(lam.cpu().numpy() - ref).max() <= 1e-13 * scale * n ** 0.5
    res = (a @ X - (b @ X) * lam).abs().max() / ((a.abs().max() + b.abs().max() * lam.abs().max()) * X.abs().max() * n)
    orth = (X.t() @ b @ X - torch.eye(n, dtype=torch.float64, device="cuda")).abs().max()
    print(f"\n[sygst] eigenpairs n={n}: |A X - B X L| / (|A| |X| n) = {res.item():.1e}, |X^T B X - I| = {orth.item():.1e}")
    assert res <= 1e-13 and orth <= 1e-12


@pytest.mark.parametrize("ci", [0, 1])
@pytest.mark.parametrize("k", [1, 37])
def test_halves_make_the_solve(topo, ci, k):
    n = 3000
    B = cb.matrix(n, n, 1, 1).distribute_symmetric(topo)
    args = cb.cholinv.info(ci, 1, -3, "U")
    cb.cholinv.factor(B, args, topo)
    rhs = torch.randn(n, k, dtype=torch.float64, device="cuda", generator=torch.Generator("cuda").manual_seed(k))
    Y = cb.cholinv.apply_RinvT(args, rhs, topo)
    X = cb.cholinv.apply_Rinv(args, Y, topo)
    assert torch.equal(X, cb.cholinv.solve(args, rhs, topo))
    R = cb.cholinv.construct_R(args)
    assert ((Y - torch.linalg.solve_triangular(R.t(), rhs, upper=False)).abs().max() <= 1e-13 * Y.abs().max()).item()
    assert ((X - torch.linalg.solve_triangular(R, Y, upper=True)).abs().max() <= 1e-13 * X.abs().max()).item()
    # in place (X = B) through the C ABI, and host pointers: the same bits
    ctx = topo.context()
    ca = args._c()
    for trans, want in ((1, Y), (0, X)):
        buf = (rhs if trans else Y).t().clone(memory_format=torch.contiguous_format)  # a copy: for k = 1 .t() is already contiguous
        ctx.check(_lib.lib().capital_cholinv_apply_rinv_f64(ctx.handle, n, C.byref(ca), _lib.UPPERTRI_PACKED, args.R.data_ptr(),
                                                            args.Rinv.data_ptr(), trans, k, buf.data_ptr(), n, buf.data_ptr(), n))
        assert torch.equal(buf.t(), want)
    h = cb.cholinv.info(ci, 1, -3, "U")
    h.R, h.Rinv, h.local_dim, h.global_dim = args.R.cpu(), args.Rinv.cpu(), n, n
    assert torch.equal(cb.cholinv.apply_RinvT(h, rhs.cpu(), topo), Y.cpu())
    assert torch.equal(cb.cholinv.apply_Rinv(h, Y.cpu(), topo), X.cpu())


def test_c_abi_rejects_overlaps_and_a_missing_R(topo):
    n = 512
    B = cb.matrix(n, n, 1, 1).distribute_symmetric(topo)
    A = _random_symmetric(n, 1)
    args = cb.cholinv.info(0, 1, -2, "U")
    cb.cholinv.factor(B, args, topo)
    out = torch.empty_like(args.Rinv)
    ctx = topo.context()
    ca = args._c()
    L = _lib.lib()
    P = _lib.UPPERTRI_PACKED
    # the top node splits and Rinv12 was skipped: R is needed
    assert L.capital_cholinv_sygst_f64(ctx.handle, n, C.byref(ca), P, None, args.Rinv.data_ptr(), A.data.data_ptr(), out.data_ptr()) \
        == _lib.ERR_INVALID
    for bad_out in (args.Rinv.data_ptr() + 8, args.R.data_ptr(), A.data.data_ptr() + 8 * n):
        assert L.capital_cholinv_sygst_f64(ctx.handle, n, C.byref(ca), P, args.R.data_ptr(), args.Rinv.data_ptr(), A.data.data_ptr(),
                                           bad_out) == _lib.ERR_INVALID
    bad = _lib.CholinvArgs(0, 0, -2, b"U")
    assert L.capital_cholinv_sygst_f64(ctx.handle, n, C.byref(bad), P, args.R.data_ptr(), args.Rinv.data_ptr(), A.data.data_ptr(),
                                       out.data_ptr()) == _lib.ERR_INVALID
    assert L.capital_cholinv_sygst_f64(ctx.handle, n, C.byref(ca), 7, args.R.data_ptr(), args.Rinv.data_ptr(), A.data.data_ptr(),
                                       out.data_ptr()) == _lib.ERR_INVALID
    x = torch.zeros(n, dtype=torch.float64, device="cuda")
    assert L.capital_cholinv_apply_rinv_f64(ctx.handle, n, C.byref(ca), P, args.R.data_ptr(), args.Rinv.data_ptr(), 2, 1, x.data_ptr(),
                                            n, x.data_ptr(), n) == _lib.ERR_INVALID


def _run_grid(nproc, same_device, timeout=1500):
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={nproc}", "--master-addr", "127.0.0.1",
           "--master-port", str(29761 + nproc), os.path.join(ROOT, "tests", "mp_worker_sygst.py")]
    env = dict(os.environ)
    if same_device:
        env["CAPITAL_MP_SAME_DEVICE"] = "1"
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=timeout, env=env)
    assert r.returncode == 0 and "MP_OK" in r.stdout, r.stdout[-3000:] + r.stderr[-3000:]
    print("\n" + r.stdout.strip()[-2000:])


@pytest.mark.parametrize("nproc", [2, 4, 8])
def test_grid_sygst_with_ranks_sharing_one_gpu(nproc):
    """2x1x1, 1x2x2 and 2x2x2 with every rank on cuda:0 (mp_worker_sygst.py)."""
    _run_grid(nproc, True)


@pytest.mark.parametrize("nproc", [2, 4, 8])
def test_grid_sygst_on_separate_gpus(nproc):
    if torch.cuda.device_count() < nproc:
        pytest.skip(f"needs {nproc} GPUs")
    _run_grid(nproc, False)
