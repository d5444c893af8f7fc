"""Shifted CholeskyQR3 (cacqr num_iter = 3) on the GPU: one H100 against the numpy restatement (tests/scqr3_reference.py) up to
kappa = 1e12, and the 1D, 3D and tunable grids through tests/mp_worker_scqr3.py."""
import os, subprocess, sys
import numpy as np
import pytest
import torch
import capital_b200 as cb
from capital_b200 import _lib
from oracle import capital_oracle as co
from scqr3_reference import ill_conditioned, scqr3

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_A = {}


@pytest.fixture(scope="module")
def topo():
    return cb.topo.rect(1, 0, 1)


def _ill(m, n, kappa):
    if (m, n, kappa) not in _A:
        _A[(m, n, kappa)] = ill_conditioned(m, n, kappa, m + n)
    return _A[(m, n, kappa)]


def _mat(a):
    m, n = a.shape
    return cb.matrix(n, m, 1, 1, data=torch.from_numpy(a.ravel(order="F").copy()).cuda())


def _factor(topo, A, num_iter=3):
    args = cb.cacqr.info(num_iter, cb.cholinv.info(0, 1, 0, "U"))
    cb.cacqr.factor(A, args, topo)
    return args


@pytest.mark.parametrize("m,n", [(8192, 256), (2048, 512), (65539, 96)])
@pytest.mark.parametrize("kappa", [1e6, 1e10, 1e12])
def test_accuracy_up_to_kappa_1e12(topo, m, n, kappa):
    a = _ill(m, n, kappa)
    A = _mat(a)
    args = _factor(topo, A)
    res, orth = cb.cacqr.validate(A, args, topo)
    r = cb.cacqr.construct_R(args).cpu().numpy()
    assert res <= 1e-14 and orth <= 1e-15, (res, orth)
    assert (np.diag(r) > 0).all()
    if kappa == 1e6:  # above it Q's trailing columns move by about kappa u under rounding: only the metrics are compared
        q_o, r_o = scqr3(a)
        q = cb.cacqr.construct_Q(args).cpu().numpy()
        assert np.abs(q - q_o).max() <= 1e-10  # Q has orthonormal columns: absolute is relative to ||Q||_2 = 1
        assert np.abs(r - r_o).max() <= 1e-10 * np.abs(r_o).max()


def test_well_conditioned_q_matches_cholesky_qr2(topo):
    m, n = 65536, 256
    A = cb.matrix(n, m, 1, 1).distribute_random(topo, 7)
    q2 = _factor(topo, A, 2).Q.clone()
    q3 = _factor(topo, A, 3).Q
    assert (q3 - q2).abs().max().item() <= 1e-12


def test_cholesky_qr2_fails_where_scqr3_does_not(topo):
    """kappa = 1e10: CholeskyQR2 breaks down (NOT_SPD) or loses orthogonality; the shifted variant does neither"""
    a = _ill(8192, 256, 1e10)
    A = _mat(a)
    try:
        args = _factor(topo, A, 2)
        _, orth2 = cb.cacqr.validate(A, args, topo)
        assert orth2 > 1e-6, orth2
    except _lib.CapitalError as ex:
        assert ex.status == _lib.ERR_NOT_SPD
    _, orth3 = cb.cacqr.validate(A, _factor(topo, A, 3), topo)
    assert orth3 <= 1e-15


def test_lstsq_from_scqr3_factors(topo):
    """consistent system at kappa = 1e10: forward error <= 1e-6 (the CPU model gives 2.1e-8)"""
    m, n = 16384, 96
    a = ill_conditioned(m, n, 1e10, 11)
    args = _factor(topo, _mat(a))
    xt = np.random.default_rng(12).standard_normal((n, 5))
    X = cb.cacqr.lstsq(args, torch.from_numpy(a @ xt).cuda(), topo).cpu().numpy()
    err = np.abs(X - xt).max() / np.abs(xt).max()
    assert err <= 1e-6, err


def test_repeat_and_host_path_are_bit_identical(topo):
    a = _ill(8192, 256, 1e10)
    A = _mat(a)
    args = _factor(topo, A)
    Q0, R0 = args.Q.clone(), args.R.clone()
    args2 = _factor(topo, A)
    assert torch.equal(Q0, args2.Q) and torch.equal(R0, args2.R)
    hostA = cb.matrix(256, 8192, 1, 1, data=A.data.cpu().pin_memory())
    h = _factor(topo, hostA)
    assert not h.Q.is_cuda and torch.equal(h.Q, Q0.cpu()) and torch.equal(h.R, R0.cpu())


def test_zero_column_is_not_spd_then_recovers(topo):
    """an exactly zero column: the shifted sweep succeeds, the next sweep's Gram matrix has an exact zero pivot -- a status return"""
    m, n = 4096, 64
    a = ill_conditioned(m, n, 1e3, 13)
    a[:, 20] = 0.0
    with pytest.raises(_lib.CapitalError) as ei:
        _factor(topo, _mat(a))
    assert ei.value.status == _lib.ERR_NOT_SPD and "rank deficient" in str(ei.value)
    good = _ill(8192, 256, 1e6)
    A = _mat(good)
    res, orth = cb.cacqr.validate(A, _factor(topo, A), topo)
    assert res <= 1e-14 and orth <= 1e-15


def _run_grid(nproc, grid, same_device, timeout=1500):
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={nproc}", "--master-addr", "127.0.0.1",
           "--master-port", str(29851 + nproc + (100 if grid != "1d" else 0)), os.path.join(ROOT, "tests", "mp_worker_scqr3.py")]
    env = dict(os.environ, CAPITAL_SCQR3_GRID=grid)
    if same_device:
        env["CAPITAL_MP_SAME_DEVICE"] = "1"
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=timeout, env=env)
    assert r.returncode == 0 and "MP_OK" in r.stdout, r.stdout[-3000:] + r.stderr[-3000:]
    print("\n" + [l for l in r.stdout.splitlines() if l.startswith("MP_OK")][0])


GRIDS = [(2, "1d"), (4, "1d"), (8, "1d"), (8, "3d"), (16, "tune")]


@pytest.mark.parametrize("nproc,grid", GRIDS)
def test_grid_with_ranks_sharing_one_gpu(nproc, grid):
    _run_grid(nproc, grid, True)


@pytest.mark.parametrize("nproc,grid", GRIDS)
def test_grid_on_separate_gpus(nproc, grid):
    if torch.cuda.device_count() < nproc:
        pytest.skip(f"needs {nproc} GPUs")
    _run_grid(nproc, grid, False)
