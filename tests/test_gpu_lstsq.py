"""cacqr::apply_QT / apply_Q / lstsq on the GPU (capital_cacqr_apply_qt_f64, capital_cacqr_apply_q_f64, capital_cacqr_lstsq_f64):
one GPU against numpy on the library's own Q and R, and the 1D row grid through tests/mp_worker_lstsq.py."""
import ctypes as C
import os, subprocess, sys
import numpy as np
import pytest
import scipy.linalg as sla
import torch
import capital_b200 as cb
from capital_b200 import _lib

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
W = 32  # panel width of the kernels (SOLVE_W)
NRHS = (1, 7, W, W + 1, 100)


@pytest.fixture(scope="module")
def topo():
    return cb.topo.rect(1, 0, 1)


def _factored(topo, m, n, num_iter=2, serialize=True, key=3):
    A = cb.matrix(n, m, 1, 1).distribute_random(topo, key)
    args = cb.cacqr.info(num_iter, cb.cholinv.info(0, 1, 0, "U"), serialize=serialize)
    cb.cacqr.factor(A, args, topo)
    return A, args


def _rel(x, ref):
    return float(np.abs(np.asarray(x) - ref).max() / np.abs(ref).max())


_LSTSQ = {}


def _numpy_lstsq(a, b, key):
    """np.linalg.lstsq of the widest right-hand side, once per matrix: narrower panels are its leading columns"""
    if key not in _LSTSQ:
        _LSTSQ[key] = np.linalg.lstsq(a, b, rcond=None)[0]
    return _LSTSQ[key]


@pytest.mark.parametrize("m", [4096, (1 << 17) + 3])
@pytest.mark.parametrize("n", [17, 64, 256, 1000])
@pytest.mark.parametrize("num_iter", [1, 2])
@pytest.mark.parametrize("serialize", [True, False])
def test_matches_numpy_on_the_library_factors(topo, m, n, num_iter, serialize):
    A, args = _factored(topo, m, n, num_iter, serialize)
    a = A.view2d().cpu().numpy()
    q = cb.cacqr.construct_Q(args).cpu().numpy()
    r = cb.cacqr.construct_R(args).cpu().numpy()
    cond = float(np.linalg.cond(r))
    rng = np.random.default_rng(m + n)
    b_all = rng.standard_normal((m, max(NRHS)))
    z_all = rng.standard_normal((n, max(NRHS)))
    qtb_all = q.T @ b_all
    qz_all = q @ z_all
    x_np_all = _numpy_lstsq(a, b_all, (m, n))
    for k in NRHS:
        B = torch.from_numpy(b_all[:, :k].copy()).cuda()
        Y = cb.cacqr.apply_QT(B, args, topo)
        assert Y.shape == (n, k) and Y.is_cuda
        assert _rel(Y.cpu().numpy(), qtb_all[:, :k]) <= 1e-13 * np.sqrt(m), (k, _rel(Y.cpu().numpy(), qtb_all[:, :k]))
        X = cb.cacqr.lstsq(args, B, topo)
        assert X.shape == (n, k) and X.is_cuda
        x = X.cpu().numpy()
        ref = sla.solve_triangular(r, qtb_all[:, :k])
        assert _rel(x, ref) <= 1e-14 * np.sqrt(m) * cond, (k, _rel(x, ref), cond)
        assert _rel(x, x_np_all[:, :k]) <= 1e-13 * np.sqrt(m) * cond ** 2, (k, _rel(x, x_np_all[:, :k]), cond)
        res = b_all[:, :k] - a @ x  # normal equations: A^T (B - A X) = 0
        assert np.linalg.norm(a.T @ res) <= 1e-13 * np.sqrt(m) * cond * np.linalg.norm(a) * np.linalg.norm(res)
        Cq = cb.cacqr.apply_Q(torch.from_numpy(z_all[:, :k].copy()).cuda(), args, topo)
        assert Cq.shape == (m, k) and Cq.is_cuda
        assert _rel(Cq.cpu().numpy(), qz_all[:, :k]) <= 1e-13
    # 1-D right-hand sides keep their rank
    b1 = torch.from_numpy(b_all[:, 0].copy()).cuda()
    assert cb.cacqr.apply_QT(b1, args, topo).shape == (n,)
    x1 = cb.cacqr.lstsq(args, b1, topo)
    assert x1.shape == (n,) and torch.equal(x1, cb.cacqr.lstsq(args, b1[:, None], topo)[:, 0])
    assert cb.cacqr.apply_Q(torch.from_numpy(z_all[:, 0].copy()).cuda(), args, topo).shape == (m,)


def test_ill_conditioned_consistent_system(topo):
    """kappa(A) = 1e6 from a chosen SVD, B = A X_true: forward error <= 1e-8."""
    m, n = 8192, 96
    rng = np.random.default_rng(5)
    u, _ = np.linalg.qr(rng.standard_normal((m, n)))
    v, _ = np.linalg.qr(rng.standard_normal((n, n)))
    a = (u * np.logspace(0, -6, n)) @ v.T
    A = cb.matrix(n, m, 1, 1, data=torch.from_numpy(a.ravel(order="F").copy()).cuda())
    args = cb.cacqr.info(2, cb.cholinv.info(0, 1, 0, "U"))
    cb.cacqr.factor(A, args, topo)
    xt = rng.standard_normal((n, 5))
    X = cb.cacqr.lstsq(args, torch.from_numpy(a @ xt).cuda(), topo).cpu().numpy()
    assert np.abs(X - xt).max() / np.abs(xt).max() <= 1e-8


@pytest.mark.parametrize("k", [1, 32])
def test_large_matches_torch_on_the_device(topo, k):
    m, n = 1 << 20, 256
    A, args = _factored(topo, m, n)
    B = torch.rand(m, k, dtype=torch.float64, device="cuda", generator=torch.Generator(device="cuda").manual_seed(k)) - 0.5
    X = cb.cacqr.lstsq(args, B, topo)
    Q, R = cb.cacqr.construct_Q(args), cb.cacqr.construct_R(args)
    ref = torch.linalg.solve_triangular(R, Q.t() @ B, upper=True)
    assert ((X - ref).abs().max() / ref.abs().max()).item() <= 1e-11
    del A, Q


def test_more_row_blocks_than_one_launch_takes(topo):
    """apply_Q owns 64-row blocks of Q; past 65535 of them the rows go in several launches"""
    m, n = 64 * 65535 + 100, 17
    A, args = _factored(topo, m, n)
    g = torch.Generator(device="cuda").manual_seed(4)
    Z = torch.rand(n, 3, dtype=torch.float64, device="cuda", generator=g) - 0.5
    B = torch.rand(m, 3, dtype=torch.float64, device="cuda", generator=g) - 0.5
    Q, R = cb.cacqr.construct_Q(args), cb.cacqr.construct_R(args)
    ref = Q @ Z
    assert ((cb.cacqr.apply_Q(Z, args, topo) - ref).abs().max() / ref.abs().max()).item() <= 1e-13
    ref = torch.linalg.solve_triangular(R, Q.t() @ B, upper=True)
    assert ((cb.cacqr.lstsq(args, B, topo) - ref).abs().max() / ref.abs().max()).item() <= 1e-11


def test_bit_identical_calls_host_path_and_slack(topo):
    m, n, k = 20001, 300, 45
    A, args = _factored(topo, m, n)
    g = torch.Generator(device="cuda").manual_seed(9)
    B = torch.rand(m, k, dtype=torch.float64, device="cuda", generator=g) - 0.5
    Z = torch.rand(n, k, dtype=torch.float64, device="cuda", generator=g) - 0.5
    Y1, X1, C1 = cb.cacqr.apply_QT(B, args, topo), cb.cacqr.lstsq(args, B, topo), cb.cacqr.apply_Q(Z, args, topo)
    assert torch.equal(Y1, cb.cacqr.apply_QT(B, args, topo))
    assert torch.equal(X1, cb.cacqr.lstsq(args, B, topo))
    assert torch.equal(C1, cb.cacqr.apply_Q(Z, args, topo))
    # host pointers: factors, right-hand sides and outputs on the host
    h = cb.cacqr.info(2, cb.cholinv.info(0, 1, 0, "U"))
    h.Q, h.R, h.n, h.rows_local, h.m_global, h.n_global = args.Q.cpu(), args.R.cpu(), n, m, m, n
    Yh, Xh, Ch = cb.cacqr.apply_QT(B.cpu(), h, topo), cb.cacqr.lstsq(h, B.cpu(), topo), cb.cacqr.apply_Q(Z.cpu(), h, topo)
    assert not Xh.is_cuda and torch.equal(Yh, Y1.cpu()) and torch.equal(Xh, X1.cpu()) and torch.equal(Ch, C1.cpu())
    # NaN slack past ldx / ldc is not touched, on the device and on the host
    ctx, L = topo.context(), _lib.lib()
    Bc, Zc = B.t().contiguous(), Z.t().contiguous()
    for dev in ("cuda", "cpu"):
        q, r = (args.Q, args.R) if dev == "cuda" else (h.Q, h.R)
        bc, zc = Bc.to(dev), Zc.to(dev)
        xb = torch.full((k, n + 5), float("nan"), dtype=torch.float64, device=dev)
        ctx.check(L.capital_cacqr_lstsq_f64(ctx.handle, m, n, q.data_ptr(), _lib.UPPERTRI_PACKED, r.data_ptr(), k, bc.data_ptr(), m,
                                            xb.data_ptr(), n + 5))
        assert torch.equal(xb[:, :n].t().cpu(), X1.cpu()) and torch.isnan(xb[:, n:]).all()
        yb = torch.full((k, n + 3), float("nan"), dtype=torch.float64, device=dev)
        ctx.check(L.capital_cacqr_apply_qt_f64(ctx.handle, m, n, q.data_ptr(), k, bc.data_ptr(), m, yb.data_ptr(), n + 3))
        assert torch.equal(yb[:, :n].t().cpu(), Y1.cpu()) and torch.isnan(yb[:, n:]).all()
        cb_ = torch.full((k, m + 7), float("nan"), dtype=torch.float64, device=dev)
        ctx.check(L.capital_cacqr_apply_q_f64(ctx.handle, m, n, q.data_ptr(), k, zc.data_ptr(), n, cb_.data_ptr(), m + 7))
        assert torch.equal(cb_[:, :m].t().cpu(), C1.cpu()) and torch.isnan(cb_[:, m:]).all()


def test_factor_lstsq_factor_is_bit_identical(topo):
    m, n = 65536, 256
    A, args = _factored(topo, m, n)
    Q0, R0 = args.Q.clone(), args.R.clone()
    cb.cacqr.lstsq(args, torch.ones(m, 33, dtype=torch.float64, device="cuda"), topo)
    cb.cacqr.factor(A, args, topo)
    assert torch.equal(Q0, args.Q) and torch.equal(R0, args.R)


def test_bad_arguments_are_invalid(topo):
    m, n, k = 4096, 64, 3
    A, args = _factored(topo, m, n)
    ctx, L = topo.context(), _lib.lib()
    q, r = args.Q.data_ptr(), args.R.data_ptr()
    buf = torch.zeros(k * m, dtype=torch.float64, device="cuda").data_ptr()
    P = _lib.UPPERTRI_PACKED
    assert L.capital_cacqr_lstsq_f64(ctx.handle, m, n, q, P, r, k, buf, m - 1, buf, n) == _lib.ERR_INVALID   # ldb < lr
    assert L.capital_cacqr_lstsq_f64(ctx.handle, m, n, q, P, r, k, buf, m, buf, n - 1) == _lib.ERR_INVALID   # ldx < n
    assert L.capital_cacqr_lstsq_f64(ctx.handle, n - 1, n, q, P, r, k, buf, m, buf, n) == _lib.ERR_INVALID   # m < n
    assert L.capital_cacqr_lstsq_f64(ctx.handle, m, n, q, 7, r, k, buf, m, buf, n) == _lib.ERR_INVALID       # structure
    assert L.capital_cacqr_lstsq_f64(ctx.handle, m, n, q, P, None, k, buf, m, buf, n) == _lib.ERR_INVALID    # NULL R
    assert L.capital_cacqr_lstsq_f64(ctx.handle, m, n, q, P, r, 0, buf, m, buf, n) == _lib.ERR_INVALID       # nrhs < 1
    assert L.capital_cacqr_apply_qt_f64(ctx.handle, m, n, q, k, buf, m - 1, buf, n) == _lib.ERR_INVALID
    assert L.capital_cacqr_apply_qt_f64(ctx.handle, m, n, q, k, buf, m, buf, n - 1) == _lib.ERR_INVALID
    assert L.capital_cacqr_apply_qt_f64(ctx.handle, n - 1, n, q, k, buf, m, buf, n) == _lib.ERR_INVALID
    assert L.capital_cacqr_apply_q_f64(ctx.handle, m, n, q, k, buf, n - 1, buf, m) == _lib.ERR_INVALID
    assert L.capital_cacqr_apply_q_f64(ctx.handle, m, n, q, k, buf, n, buf, m - 1) == _lib.ERR_INVALID
    assert L.capital_cacqr_apply_q_f64(ctx.handle, n - 1, n, q, k, buf, n, buf, m) == _lib.ERR_INVALID


def _run_grid(nproc, same_device, timeout=1200):
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={nproc}", "--master-addr", "127.0.0.1",
           "--master-port", str(29741 + nproc), os.path.join(ROOT, "tests", "mp_worker_lstsq.py")]
    env = dict(os.environ)
    if same_device:
        env["CAPITAL_MP_SAME_DEVICE"] = "1"
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=timeout, env=env)
    assert r.returncode == 0 and "MP_OK" in r.stdout, r.stdout[-3000:] + r.stderr[-3000:]


@pytest.mark.parametrize("nproc", [2, 4, 8])
def test_grid_lstsq_with_ranks_sharing_one_gpu(nproc):
    """the 1D row grid with every rank on cuda:0: X against numpy, bit-identical on every rank, host path == device path"""
    _run_grid(nproc, True)


@pytest.mark.parametrize("nproc", [2, 4, 8])
def test_grid_lstsq_on_separate_gpus(nproc):
    if torch.cuda.device_count() < nproc:
        pytest.skip(f"needs {nproc} GPUs")
    _run_grid(nproc, False)
