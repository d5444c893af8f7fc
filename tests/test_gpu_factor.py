"""GPU parity of the factorization entry points (single GPU) against the reference's own dumps (tests/golden),
the oracle restatement, and size-independent properties at larger n."""
import json, os
import numpy as np
import pytest
import torch
import capital_b200 as cb
from capital_b200 import _lib
from oracle import capital_oracle as co

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), "golden")


def load(name):
    z = np.load(os.path.join(GOLD, name + ".npz"))
    return json.loads(str(z["meta"])), z


@pytest.fixture(scope="module")
def topo():
    return cb.topo.square(1, 0, 1)


@pytest.mark.parametrize("name", ["cholinv_p1_n96_ci1", "cholinv_p1_n128_ci0"])
def test_cholinv_matches_reference_dump(topo, name):
    meta, z = load(name)
    n = meta["n"]
    A = cb.matrix(n, n, 1, 1).distribute_symmetric(topo)
    assert np.array_equal(A.data.cpu().numpy(), z["A_0"])
    args = cb.cholinv.info(meta["complete_inv"], meta["split"], meta["bc_mult_dim"], "U")
    cb.cholinv.factor(A, args, topo)
    r, ri = args.R.cpu().numpy(), args.Rinv.cpu().numpy()
    assert np.abs(r - z["R_0"]).max() <= 1e-13 * np.abs(z["R_0"]).max()
    assert np.abs(ri - z["Rinv_0"]).max() <= 1e-13 * np.abs(z["Rinv_0"]).max()
    if not meta["complete_inv"]:
        assert np.array_equal(ri == 0, z["Rinv_0"] == 0)  # same zero block (cholinv.hpp:147)
    assert cb.cholinv.residual(A, args, topo) < 1e-14


@pytest.mark.parametrize("n,ci,bcm", [(64, 1, 0), (200, 1, -1), (512, 0, -2), (777, 1, -2), (1000, 0, -3), (2048, 0, -2), (2048, 1, -2)])
@pytest.mark.parametrize("serialize", [True, False])
def test_cholinv_matches_oracle(topo, n, ci, bcm, serialize):
    A = cb.matrix(n, n, 1, 1).distribute_symmetric(topo)
    args = cb.cholinv.info(ci, 1, bcm, "U", serialize=serialize)
    cb.cholinv.factor(A, args, topo)
    a = co.spd_global(n)
    r_o, ri_o = co.cholinv(a, bool(ci), 1, co.bc_dimension(n, 1, 1, bcm))
    R = cb.cholinv.construct_R(args, topo).cpu().numpy()
    Ri = cb.cholinv.construct_Rinv(args, topo).cpu().numpy()
    assert np.abs(R - r_o).max() <= 2e-13 * np.abs(r_o).max()
    assert np.abs(Ri - ri_o).max() <= 2e-13 * np.abs(ri_o).max()
    assert np.array_equal(np.tril(R, -1), np.zeros_like(R)) and np.array_equal(np.tril(Ri, -1), np.zeros_like(Ri))
    res = cb.cholinv.residual(A, args, topo)
    assert res <= 1e-12 and abs(res - co.cholesky_residual(a, R)) < 1e-15


@pytest.mark.parametrize("n", [512, 2000])
@pytest.mark.parametrize("serialize", [True, False])
def test_cholinv_whole_matrix_is_the_reference_base_case(topo, n, serialize):
    """bc_mult_dim >= 0 on one rank: n <= bcDimension, so the reference's invoke goes straight to its base case (potrf + trtri of the
    whole block, cholinv.hpp:93-104) and returns the FULL inverse even when complete_inv == 0 -- nothing is skipped, nothing stale."""
    A = cb.matrix(n, n, 1, 1).distribute_symmetric(topo)
    junk = cb.cholinv.info(1, 1, -3, "U", serialize=serialize)  # fills the work buffers with the values of another schedule first
    cb.cholinv.factor(A, junk, topo)
    args = cb.cholinv.info(0, 1, 0, "U", serialize=serialize)
    args.R = torch.full_like(junk.R, float("nan"))
    args.Rinv = torch.full_like(junk.Rinv, float("nan"))
    cb.cholinv.factor(A, args, topo)
    a = co.spd_global(n)
    r_o, ri_o = co.cholinv(a, False, 1, co.bc_dimension(n, 1, 1, 0))
    assert np.count_nonzero(np.triu(ri_o, 1)) > n * (n - 1) // 2 - 8  # the oracle (= reference) inverse is full
    R = cb.cholinv.construct_R(args, topo).cpu().numpy()
    Ri = cb.cholinv.construct_Rinv(args, topo).cpu().numpy()
    assert np.abs(R - r_o).max() <= 2e-13 * np.abs(r_o).max()
    assert np.abs(Ri - ri_o).max() <= 2e-13 * np.abs(ri_o).max()


def test_release_workspace_then_factor_again(topo):
    """FlushIntermediates semantics (cholinv/policy.h:85-156): every work buffer can be dropped between calls."""
    n = 1024
    A = cb.matrix(n, n, 1, 1).distribute_symmetric(topo)
    args = cb.cholinv.info(1, 1, -2, "U")
    cb.cholinv.factor(A, args, topo)
    keep = args.R.clone()
    free0 = torch.cuda.mem_get_info()[0]
    topo.context().release_workspace()
    assert torch.cuda.mem_get_info()[0] > free0
    cb.cholinv.factor(A, args, topo)
    assert torch.equal(keep, args.R)


def test_context_follows_the_current_torch_stream(topo):
    n = 768
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        A = cb.matrix(n, n, 1, 1).distribute_symmetric(topo)
        args = cb.cholinv.info(1, 1, -2, "U")
        cb.cholinv.factor(A, args, topo)
        assert cb.cholinv.residual(A, args, topo) < 1e-14
    A2 = cb.matrix(n, n, 1, 1).distribute_symmetric(topo)  # back on the default stream
    a2 = cb.cholinv.info(1, 1, -2, "U")
    cb.cholinv.factor(A2, a2, topo)
    assert torch.equal(a2.R, args.R)


def test_cholinv_host_pointers_and_reuse(topo):
    """reference-facing call: pinned host buffers in, pinned host buffers out; repeated calls reuse the workspaces."""
    n = 640
    a = torch.from_numpy(np.asfortranarray(co.spd_global(n)).ravel(order="F").copy()).pin_memory()
    A = cb.matrix(n, n, 1, 1, data=a)
    args = cb.cholinv.info(1, 1, -2, "U")
    ctx = topo.context()
    for _ in range(2):
        ctx.reset_counters()
        cb.cholinv.factor(A, args, topo)
        cnt = ctx.counters()
        # only the upper triangle of A travels (column chunks, rows 0..chunk end)
        assert n * (n + 1) // 2 * 8 <= cnt.h2d_bytes <= n * n * 8 * 0.6 and cnt.d2h_bytes == 2 * (n * (n + 1) // 2) * 8 and cnt.kernel_launches > 0
    assert not args.R.is_cuda
    r_o, ri_o = co.cholinv(co.spd_global(n), True, 1, co.bc_dimension(n, 1, 1, -2))
    assert np.abs(co.unpack_upper(args.R.numpy(), n) - r_o).max() < 1e-12
    assert np.abs(co.unpack_upper(args.Rinv.numpy(), n) - ri_o).max() < 1e-13


@pytest.mark.parametrize("n,ci", [(8192, 1), (8192, 0), (9088, 1), (16384, 0)])
def test_cholinv_streamed_host_path_equals_resident_path(topo, n, ci):
    """host buffers at a size where A12 is multiplied while it is still arriving and the top-level inverse block leaves in column
    chunks: every tile computes what it computes in the resident schedule, so the outputs are identical bit for bit."""
    A = cb.matrix(n, n, 1, 1).distribute_symmetric(topo)
    dev = cb.cholinv.info(ci, 1, -4, "U")
    cb.cholinv.factor(A, dev, topo)
    hostA = cb.matrix(n, n, 1, 1, data=A.data.cpu().pin_memory())
    hst = cb.cholinv.info(ci, 1, -4, "U")
    ctx = topo.context()
    for _ in range(2):
        ctx.reset_counters()
        cb.cholinv.factor(hostA, hst, topo)
        assert ctx.counters().d2h_bytes == 2 * (n * (n + 1) // 2) * 8
    assert not hst.R.is_cuda and not hst.Rinv.is_cuda
    assert torch.equal(hst.R, dev.R.cpu()) and torch.equal(hst.Rinv, dev.Rinv.cpu())
    assert cb.cholinv.residual(A, dev, topo) <= 1e-12


def test_cholinv_rejects_non_spd(topo):
    n = 256
    A = cb.matrix(n, n, 1, 1).distribute_symmetric(topo)
    A.view2d()[100, 100] = -1.0
    with pytest.raises(_lib.CapitalError) as e:
        cb.cholinv.factor(A, cb.cholinv.info(1, 1, -1, "U"), topo)
    assert e.value.status == _lib.ERR_NOT_SPD


@pytest.mark.parametrize("n", [4096, 8192])
def test_cholinv_large_properties(topo, n):
    """size-independent properties: residual, R Rinv = I on the diagonal blocks, idempotent re-factorization."""
    A = cb.matrix(n, n, 1, 1).distribute_symmetric(topo)
    args = cb.cholinv.info(0, 1, -3, "U", serialize=False)
    cb.cholinv.factor(A, args, topo)
    assert cb.cholinv.residual(A, args, topo) <= 1e-12
    R, Ri = cb.cholinv.construct_R(args), cb.cholinv.construct_Rinv(args)
    h = n // 2
    eye = torch.eye(h, dtype=torch.float64, device="cuda")
    assert (Ri[:h, :h] @ R[:h, :h] - eye).abs().max().item() < 1e-12
    assert (Ri[h:, h:] @ R[h:, h:] - eye).abs().max().item() < 1e-12
    assert torch.count_nonzero(Ri[:h, h:]).item() == 0
    keep = args.R.clone()
    cb.cholinv.factor(A, args, topo)
    assert torch.equal(keep, args.R)  # deterministic


@pytest.mark.parametrize("name", ["cacqr_p1_m512_n32"])
def test_cacqr_matches_reference_dump(name):
    meta, z = load(name)
    m, n = meta["m"], meta["n"]
    topo = cb.topo.rect(1, 0, 1)
    A = cb.matrix(n, m, 1, 1).distribute_random(topo, 0)
    assert np.array_equal(A.data.cpu().numpy(), z["A_0"])
    args = cb.cacqr.info(2, cb.cholinv.info(0, 1, 0, "U"))
    cb.cacqr.factor(A, args, topo)
    assert np.abs(args.R.cpu().numpy() - z["R_0"]).max() < 1e-12 * np.abs(z["R_0"]).max()
    assert np.abs(args.Q.cpu().numpy() - z["Q_0"]).max() < 1e-12
    res, orth = cb.cacqr.validate(A, args, topo)
    assert res < 1e-14 and orth < 1e-15


@pytest.mark.parametrize("m,n,it", [(4096, 64, 2), (10000, 100, 2), (65536, 256, 2), (3000, 48, 1)])
def test_cacqr_matches_oracle(m, n, it):
    topo = cb.topo.rect(1, 0, 1)
    A = cb.matrix(n, m, 1, 1).distribute_random(topo, 3)
    args = cb.cacqr.info(it, cb.cholinv.info(0, 1, 0, "U"))
    cb.cacqr.factor(A, args, topo)
    a = co.random_local(m, n, 1, 1, 0, 0, 3)
    qs, r = co.cacqr_1d([a], it)
    Q, R = cb.cacqr.construct_Q(args).cpu().numpy(), cb.cacqr.construct_R(args).cpu().numpy()
    assert np.abs(R - r).max() < 1e-11 * np.abs(r).max()
    assert np.abs(Q - qs[0]).max() < 1e-11
    res, orth = cb.cacqr.validate(A, args, topo)
    assert res < 1e-13
    assert orth < (1e-14 if it == 2 else 1e-12)
    assert abs(res - co.qr_residual(a, Q, R)) < 1e-15


@pytest.mark.parametrize("m,n,k", [(256, 192, 320), (1000, 520, 777), (2048, 2048, 1024)])
def test_summa_gemm_entry_point(topo, m, n, k):
    """matmult::summa::invoke (T*N form) on the 1x1x1 grid against an FP64 torch reference."""
    A = cb.matrix(m, k, 1, 1); B = cb.matrix(n, k, 1, 1); C = cb.matrix(n, m, 1, 1)
    g = torch.Generator(device="cuda").manual_seed(7)
    for M in (A, B, C):
        M.data.copy_(torch.rand(M.data.numel(), dtype=torch.float64, device="cuda", generator=g) - 0.5)
    ref = 0.5 * (A.view2d().t() @ B.view2d()) - 2.0 * C.view2d()
    cb.summa.invoke(A, B, C, topo, alpha=0.5, beta=-2.0)
    assert (C.view2d() - ref).abs().max().item() < 1e-12


@pytest.mark.parametrize("m,n,it", [(2048, 128, 2), (4096, 320, 2), (1024, 64, 1)])
def test_cacqr_3d_code_path_on_degenerate_grid(m, n, it, monkeypatch):
    """qr::cacqr::invoke_3d (cacqr.hpp:195-215) -- the SUMMA-based Gram / cholinv / trmm composition -- forced onto the 1x1x1 grid
    (where the reference itself would take the 1D path) and compared with the 1D oracle: the factors are unique."""
    monkeypatch.setenv("CAPITAL_FORCE_QR3D", "1")
    topo = cb.topo.rect(1, 0, 1)
    A = cb.matrix(n, m, 1, 1).distribute_random(topo, 11)
    args = cb.cacqr.info(it, cb.cholinv.info(1, 1, -1, "U"))
    cb.cacqr.factor(A, args, topo)
    a = co.random_local(m, n, 1, 1, 0, 0, 11)
    qs, r = co.cacqr_1d([a], it)
    Q, R = cb.cacqr.construct_Q(args).cpu().numpy(), cb.cacqr.construct_R(args).cpu().numpy()
    assert np.abs(R - r).max() < 1e-11 * np.abs(r).max()
    assert np.abs(Q - qs[0]).max() < 1e-11
    res, orth = cb.cacqr.validate(A, args, topo)
    assert res < 1e-13 and orth < (1e-14 if it == 2 else 1e-12)


def test_plain_c_caller_runs():
    """the plain-C driver (reference bench protocol, host buffers) factors and validates on the GPU"""
    import subprocess, tempfile
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    exe = os.path.join(tempfile.mkdtemp(), "cholinv_driver")
    libdir = os.path.join(root, "capital_b200")
    subprocess.run(["gcc", "-O2", "-I" + os.path.join(root, "include"), os.path.join(root, "examples", "cholinv_driver.c"), "-L" + libdir,
                    "-lcapital_b200", "-Wl,-rpath," + libdir, "-lm", "-o", exe], check=True)
    r = subprocess.run([exe, "2048", "1", "0", "1", "-2", "0", "0", "2"], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0, r.stdout + r.stderr
    lines = r.stdout.strip().splitlines()
    assert sum(l.startswith("total time - ") for l in lines) == 2 and float(lines[-1]) < 1e-14
