"""cholinv::inverse on the GPU: A^-1 = Rinv Rinv^T from the CholInv factors (capital_cholinv_inverse_f64), one GPU and the square
grids, and its validator (capital_cholinv_inverse_residual_f64)."""
import ctypes as C
import os, subprocess, sys
import numpy as np
import pytest
import torch
import capital_b200 as cb
from capital_b200 import _lib
from oracle import capital_oracle as co

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
U = 2.0 ** -53  # unit roundoff of FP64


@pytest.fixture(scope="module")
def topo():
    return cb.topo.square(1, 0, 1)


def _full(Ainv, n, serialize):
    """n x n view of the output: the upper triangle (zeros below) when packed, the full block when rect"""
    if not serialize:
        return Ainv.view(n, n).t()
    out = torch.zeros(n, n, dtype=torch.float64, device=Ainv.device)
    iu = torch.triu_indices(n, n, device=Ainv.device)
    out[iu[0], iu[1]] = Ainv[(iu[1] * (iu[1] + 1)) // 2 + iu[0]]
    return out


def _rel(x, ref):
    return float(np.abs(np.asarray(x) - ref).max() / np.abs(ref).max())


@pytest.mark.parametrize("n", [64, 777, 2048, 4096])
@pytest.mark.parametrize("ci", [0, 1])
@pytest.mark.parametrize("serialize", [True, False])
@pytest.mark.parametrize("split", [1, 2])
def test_inverse_matches_numpy(topo, n, ci, serialize, split):
    A = cb.matrix(n, n, 1, 1).distribute_symmetric(topo)
    args = cb.cholinv.info(ci, split, -2, "U", serialize=serialize)
    cb.cholinv.factor(A, args, topo)
    Ainv = cb.cholinv.inverse(args, topo)
    assert Ainv.is_cuda and Ainv.shape == args.Rinv.shape
    M = _full(Ainv, n, serialize)
    ref = np.linalg.inv(co.spd_global(n))
    if serialize:
        assert _rel(M.cpu().numpy(), np.triu(ref)) <= 1e-12
    else:
        assert torch.equal(M, M.t())  # exactly symmetric
        assert _rel(M.cpu().numpy(), ref) <= 1e-12
    assert cb.cholinv.inverse_residual(A, Ainv, args, topo) <= 1e-14


@pytest.mark.parametrize("n", [512, 1500])
def test_top_level_base_case_needs_no_R(topo, n):
    """bc_mult_dim >= 0: the top node is the base case and Rinv is complete even with complete_inv = 0, so R may be NULL."""
    A = cb.matrix(n, n, 1, 1).distribute_symmetric(topo)
    args = cb.cholinv.info(0, 1, 0, "U")
    cb.cholinv.factor(A, args, topo)
    ref = cb.cholinv.inverse(args, topo)
    out = torch.empty_like(ref)
    ctx = topo.context()
    ca = args._c()
    ctx.check(_lib.lib().capital_cholinv_inverse_f64(ctx.handle, n, C.byref(ca), _lib.UPPERTRI_PACKED, None, args.Rinv.data_ptr(),
                                                     out.data_ptr()))
    assert torch.equal(out, ref)
    assert _rel(_full(out, n, True).cpu().numpy(), np.triu(np.linalg.inv(co.spd_global(n)))) <= 1e-12
    # a split top node with the skipped block does need R
    a2 = cb.cholinv.info(0, 1, -2, "U")
    cb.cholinv.factor(A, a2, topo)
    ca2 = a2._c()
    assert _lib.lib().capital_cholinv_inverse_f64(ctx.handle, n, C.byref(ca2), _lib.UPPERTRI_PACKED, None, a2.Rinv.data_ptr(),
                                                  out.data_ptr()) == _lib.ERR_INVALID
    # the output may not overlap an input
    assert _lib.lib().capital_cholinv_inverse_f64(ctx.handle, n, C.byref(ca), _lib.UPPERTRI_PACKED, None, args.Rinv.data_ptr(),
                                                  args.Rinv.data_ptr() + 8) == _lib.ERR_INVALID


@pytest.mark.parametrize("split", [1, 2])
def test_complete_and_rebuilt_inverses_agree(topo, split):
    """complete_inv = 0 rebuilds the skipped Rinv12 with the factor's own two products (same kernel, flags and shapes)."""
    n = 3000
    A = cb.matrix(n, n, 1, 1).distribute_symmetric(topo)
    outs = []
    for ci in (0, 1):
        args = cb.cholinv.info(ci, split, -3, "U")
        cb.cholinv.factor(A, args, topo)
        outs.append(cb.cholinv.inverse(args, topo))
    rel = ((outs[0] - outs[1]).abs().max() / outs[1].abs().max()).item()
    print(f"\n[inverse] n={n} split={split}: complete_inv 0 vs 1 bit-identical={torch.equal(outs[0], outs[1])} max rel diff={rel:.1e}")
    assert rel <= 1e-14


def test_ill_conditioned_residual(topo):
    """SPD with cond ~ 1e6 given as data: the residual stays within a few kappa u."""
    n, kappa = 1024, 1e6
    rng = np.random.default_rng(17)
    q, _ = np.linalg.qr(rng.standard_normal((n, n)))
    a = (q * np.logspace(0, 6, n)) @ q.T
    a = 0.5 * (a + a.T)
    A = cb.matrix(n, n, 1, 1, data=torch.from_numpy(np.asfortranarray(a).ravel(order="F").copy()).cuda())
    for ci in (0, 1):
        for serialize in (True, False):
            args = cb.cholinv.info(ci, 1, -2, "U", serialize=serialize)
            cb.cholinv.factor(A, args, topo)
            res = cb.cholinv.inverse_residual(A, cb.cholinv.inverse(args, topo), args, topo)
            print(f"\n[inverse] kappa=1e6 ci={ci} serialize={serialize}: residual {res:.2e} (kappa u = {kappa * U:.1e})")
            assert res <= 4 * kappa * U


@pytest.mark.parametrize("ci", [0, 1])
def test_large_matches_torch_cholesky_inverse(topo, ci):
    n = 16384
    A = cb.matrix(n, n, 1, 1).distribute_symmetric(topo)
    args = cb.cholinv.info(ci, 1, -5, "U")
    cb.cholinv.factor(A, args, topo)
    ctx = topo.context()
    ctx.reset_counters()
    Ainv = cb.cholinv.inverse(args, topo)
    torch.cuda.synchronize()
    flops = ctx.counters().gemm_flops
    # the inverse product is n^3 / 3; a rebuilt Rinv12 adds its two products, (n / 2)^3 each
    expect = n ** 3 / 3 + (0 if ci else 2 * (n // 2) ** 3)
    assert abs(flops / expect - 1) <= 0.03, (flops, expect)
    R = cb.cholinv.construct_R(args)
    ref = torch.cholesky_inverse(R, upper=True)
    del R
    M = _full(Ainv, n, True)
    rel = ((M - torch.triu(ref)).abs().max() / ref.abs().max()).item()
    assert rel <= 1e-12, rel


@pytest.mark.parametrize("ci", [0, 1])
@pytest.mark.parametrize("serialize", [True, False])
def test_bit_identical_repeats_and_host_path(topo, ci, serialize):
    n = 2500
    A = cb.matrix(n, n, 1, 1).distribute_symmetric(topo)
    args = cb.cholinv.info(ci, 1, -3, "U", serialize=serialize)
    cb.cholinv.factor(A, args, topo)
    X1 = cb.cholinv.inverse(args, topo)
    X2 = cb.cholinv.inverse(args, topo)
    assert torch.equal(X1, X2)
    h = cb.cholinv.info(ci, 1, -3, "U", serialize=serialize)
    h.R, h.Rinv, h.local_dim, h.global_dim = args.R.cpu(), args.Rinv.cpu(), n, n
    Xh = cb.cholinv.inverse(h, topo)
    assert not Xh.is_cuda and Xh.is_pinned() and torch.equal(Xh, X1.cpu())
    # the validator takes host operands too (its sum of squares is accumulated atomically: equal up to the order of the additions)
    Ah = cb.matrix(n, n, 1, 1, data=A.data.cpu())
    assert cb.cholinv.inverse_residual(Ah, Xh, h, topo) == pytest.approx(cb.cholinv.inverse_residual(A, X1, args, topo), rel=1e-9)


def test_factor_inverse_factor_is_bit_identical(topo):
    n = 4096
    A = cb.matrix(n, n, 1, 1).distribute_symmetric(topo)
    args = cb.cholinv.info(0, 1, -3, "U")
    cb.cholinv.factor(A, args, topo)
    R0, Ri0 = args.R.clone(), args.Rinv.clone()
    cb.cholinv.inverse(args, topo)
    cb.cholinv.factor(A, args, topo)
    assert torch.equal(R0, args.R) and torch.equal(Ri0, args.Rinv)


def _run_grid(nproc, same_device, timeout=1200):
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={nproc}", "--master-addr", "127.0.0.1",
           "--master-port", str(29731 + nproc), os.path.join(ROOT, "tests", "mp_worker_inverse.py")]
    env = dict(os.environ)
    if same_device:
        env["CAPITAL_MP_SAME_DEVICE"] = "1"
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=timeout, env=env)
    assert r.returncode == 0 and "MP_OK" in r.stdout, r.stdout[-3000:] + r.stderr[-3000:]
    print("\n" + r.stdout.strip()[-1500:])


@pytest.mark.parametrize("nproc", [2, 4, 8])
def test_grid_inverse_with_ranks_sharing_one_gpu(nproc):
    """2x1x1, 1x2x2 and 2x2x2 with every rank on cuda:0: the assembled A^-1 against numpy, identical layer replicas, an exactly
    symmetric rect output, the residual, host path == device path."""
    _run_grid(nproc, True)


@pytest.mark.parametrize("nproc", [2, 4, 8])
def test_grid_inverse_on_separate_gpus(nproc):
    if torch.cuda.device_count() < nproc:
        pytest.skip(f"needs {nproc} GPUs")
    _run_grid(nproc, False)
