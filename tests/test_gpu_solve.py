"""cholinv::solve on the GPU: A X = B from the CholInv factors (capital_cholinv_solve_f64), one GPU and the square grids."""
import ctypes as C
import os, subprocess, sys
import numpy as np
import pytest
import torch
import capital_b200 as cb
from capital_b200 import _lib
from oracle import capital_oracle as co
from solve_reference import cholesky_solve

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
W = 32  # panel width of the kernel (SOLVE_W)


@pytest.fixture(scope="module")
def topo():
    return cb.topo.square(1, 0, 1)


def _rhs(n, k, seed):
    return torch.from_numpy(np.random.default_rng(seed).standard_normal((n, k))).cuda()


def _rel(x, ref):
    return float(np.abs(np.asarray(x) - ref).max() / np.abs(ref).max())


@pytest.mark.parametrize("n", [64, 777, 2048, 4096])
@pytest.mark.parametrize("ci", [0, 1])
@pytest.mark.parametrize("serialize", [True, False])
@pytest.mark.parametrize("split", [1, 2])
def test_solve_matches_numpy(topo, n, ci, serialize, split):
    A = cb.matrix(n, n, 1, 1).distribute_symmetric(topo)
    args = cb.cholinv.info(ci, split, -2, "U", serialize=serialize)
    cb.cholinv.factor(A, args, topo)
    a = co.spd_global(n)
    for k in (1, 7, W, W + 1, 100):
        B = _rhs(n, k, n + k)
        X = cb.cholinv.solve(args, B, topo)
        assert X.shape == B.shape and X.is_cuda
        ref = np.linalg.solve(a, B.cpu().numpy())
        assert _rel(X.cpu().numpy(), ref) <= 1e-12, (k, _rel(X.cpu().numpy(), ref))
    b1 = B[:, 0].contiguous()
    x1 = cb.cholinv.solve(args, b1, topo)
    assert x1.shape == (n,) and _rel(x1.cpu().numpy(), np.linalg.solve(a, b1.cpu().numpy())) <= 1e-12


@pytest.mark.parametrize("n,split", [(1000, 1), (2048, 2)])
def test_device_solve_equals_the_block_formula(topo, n, split):
    """complete_inv = 0: the library's block solve against the numpy restatement of the same formula on the oracle's factors."""
    A = cb.matrix(n, n, 1, 1).distribute_symmetric(topo)
    args = cb.cholinv.info(0, split, -3, "U")
    cb.cholinv.factor(A, args, topo)
    B = _rhs(n, 9, 3)
    X = cb.cholinv.solve(args, B, topo).cpu().numpy()
    r, ri = co.cholinv(co.spd_global(n), False, split, co.bc_dimension(n, 1, 1, -3))
    assert _rel(X, cholesky_solve(r, ri, B.cpu().numpy(), False, split, co.bc_dimension(n, 1, 1, -3))) <= 1e-13


@pytest.mark.parametrize("n", [512, 1500])
def test_top_level_base_case_needs_no_R(topo, n):
    """bc_mult_dim >= 0: the top node is the base case and Rinv is complete even with complete_inv = 0, so R may be NULL."""
    A = cb.matrix(n, n, 1, 1).distribute_symmetric(topo)
    args = cb.cholinv.info(0, 1, 0, "U")
    cb.cholinv.factor(A, args, topo)
    B = _rhs(n, 3, 11)
    X = cb.cholinv.solve(args, B, topo)
    assert _rel(X.cpu().numpy(), np.linalg.solve(co.spd_global(n), B.cpu().numpy())) <= 1e-12
    Bc, Xc = B.t().contiguous(), torch.empty(3, n, dtype=torch.float64, device="cuda")
    ctx = topo.context()
    ca = args._c()
    ctx.check(_lib.lib().capital_cholinv_solve_f64(ctx.handle, n, C.byref(ca), _lib.UPPERTRI_PACKED, None, args.Rinv.data_ptr(), 3,
                                                   Bc.data_ptr(), n, Xc.data_ptr(), n))
    assert torch.equal(Xc.t(), X)
    # a split top node with the skipped block does need R
    a2 = cb.cholinv.info(0, 1, -2, "U")
    cb.cholinv.factor(A, a2, topo)
    ca2 = a2._c()
    assert _lib.lib().capital_cholinv_solve_f64(ctx.handle, n, C.byref(ca2), _lib.UPPERTRI_PACKED, None, a2.Rinv.data_ptr(), 3,
                                                Bc.data_ptr(), n, Xc.data_ptr(), n) == _lib.ERR_INVALID


def test_complete_and_block_solutions_agree(topo):
    n = 3000
    A = cb.matrix(n, n, 1, 1).distribute_symmetric(topo)
    B = _rhs(n, 40, 5)
    xs = []
    for ci in (0, 1):
        args = cb.cholinv.info(ci, 1, -3, "U")
        cb.cholinv.factor(A, args, topo)
        xs.append(cb.cholinv.solve(args, B, topo))
    assert ((xs[0] - xs[1]).abs().max() / xs[1].abs().max()).item() <= 1e-13


def test_ill_conditioned_forward_error(topo):
    """SPD with cond ~ 1e6 given as data: forward error of the Rinv-based solve <= 1e-9."""
    n = 1024
    rng = np.random.default_rng(17)
    q, _ = np.linalg.qr(rng.standard_normal((n, n)))
    a = (q * np.logspace(0, 6, n)) @ q.T
    a = 0.5 * (a + a.T)
    A = cb.matrix(n, n, 1, 1, data=torch.from_numpy(np.asfortranarray(a).ravel(order="F").copy()).cuda())
    xt = rng.standard_normal((n, 4))
    B = torch.from_numpy(a @ xt).cuda()
    for ci in (0, 1):
        args = cb.cholinv.info(ci, 1, -2, "U")
        cb.cholinv.factor(A, args, topo)
        X = cb.cholinv.solve(args, B, topo).cpu().numpy()
        assert np.abs(X - xt).max() / np.abs(xt).max() <= 1e-9


@pytest.mark.parametrize("k", [1, 32])
def test_large_matches_torch_cholesky_solve(topo, k):
    n = 16384
    A = cb.matrix(n, n, 1, 1).distribute_symmetric(topo)
    args = cb.cholinv.info(0, 1, -5, "U")
    cb.cholinv.factor(A, args, topo)
    B = _rhs(n, k, 21)
    X = cb.cholinv.solve(args, B, topo)
    V = A.view2d()
    Lc = torch.linalg.cholesky(torch.triu(V) + torch.triu(V, 1).t())  # the factor reads the upper triangle only
    ref = torch.cholesky_solve(B, Lc)
    del Lc
    assert ((X - ref).abs().max() / ref.abs().max()).item() <= 1e-12


@pytest.mark.parametrize("ci", [0, 1])
def test_bit_identical_calls_paths_and_in_place(topo, ci):
    n, k = 2500, 45
    A = cb.matrix(n, n, 1, 1).distribute_symmetric(topo)
    args = cb.cholinv.info(ci, 1, -3, "U")
    cb.cholinv.factor(A, args, topo)
    B = _rhs(n, k, 8)
    X1 = cb.cholinv.solve(args, B, topo)
    X2 = cb.cholinv.solve(args, B, topo)
    assert torch.equal(X1, X2)
    # host pointers: factors, B and X on the host
    h = cb.cholinv.info(ci, 1, -3, "U")
    h.R, h.Rinv, h.local_dim, h.global_dim = args.R.cpu(), args.Rinv.cpu(), n, n
    Xh = cb.cholinv.solve(h, B.cpu(), topo)
    assert not Xh.is_cuda and torch.equal(Xh, X1.cpu())
    # in place (X = B), column-major with ld > n
    ld = n + 3
    buf = torch.full((k, ld), float("nan"), dtype=torch.float64, device="cuda")
    buf[:, :n] = B.t()
    ctx = topo.context()
    ca = args._c()
    ctx.check(_lib.lib().capital_cholinv_solve_f64(ctx.handle, n, C.byref(ca), _lib.UPPERTRI_PACKED, args.R.data_ptr(), args.Rinv.data_ptr(),
                                                   k, buf.data_ptr(), ld, buf.data_ptr(), ld))
    assert torch.equal(buf[:, :n].t(), X1)
    assert torch.isnan(buf[:, n:]).all()  # rows n .. ld of every column are not touched
    # host in place
    hb = buf.cpu()
    hb[:, :n] = B.t().cpu()
    ctx.check(_lib.lib().capital_cholinv_solve_f64(ctx.handle, n, C.byref(ca), _lib.UPPERTRI_PACKED, h.R.data_ptr(), h.Rinv.data_ptr(),
                                                   k, hb.data_ptr(), ld, hb.data_ptr(), ld))
    assert torch.equal(hb[:, :n].t(), X1.cpu()) and torch.isnan(hb[:, n:]).all()


def test_factor_solve_factor_is_bit_identical(topo):
    n = 4096
    A = cb.matrix(n, n, 1, 1).distribute_symmetric(topo)
    args = cb.cholinv.info(0, 1, -3, "U")
    cb.cholinv.factor(A, args, topo)
    R0, Ri0 = args.R.clone(), args.Rinv.clone()
    cb.cholinv.solve(args, _rhs(n, 33, 2), topo)
    cb.cholinv.factor(A, args, topo)
    assert torch.equal(R0, args.R) and torch.equal(Ri0, args.Rinv)


def _run_grid(nproc, same_device, timeout=1200):
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={nproc}", "--master-addr", "127.0.0.1",
           "--master-port", str(29701 + nproc), os.path.join(ROOT, "tests", "mp_worker_solve.py")]
    env = dict(os.environ)
    if same_device:
        env["CAPITAL_MP_SAME_DEVICE"] = "1"
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=timeout, env=env)
    assert r.returncode == 0 and "MP_OK" in r.stdout, r.stdout[-3000:] + r.stderr[-3000:]


@pytest.mark.parametrize("nproc", [2, 4, 8])
def test_grid_solve_with_ranks_sharing_one_gpu(nproc):
    """2x1x1, 1x2x2 and 2x2x2 with every rank on cuda:0: X against numpy, bit-identical on every rank, host path == device path."""
    _run_grid(nproc, True)


@pytest.mark.parametrize("nproc", [2, 4, 8])
def test_grid_solve_on_separate_gpus(nproc):
    if torch.cuda.device_count() < nproc:
        pytest.skip(f"needs {nproc} GPUs")
    _run_grid(nproc, False)
