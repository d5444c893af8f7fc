"""Batched CholeskyQR on the GPU (capital_cacqr_factor_batched_f64 / capital_cacqr_lstsq_batched_f64): the same bits as the
single-matrix factor and lstsq where the single path's base case is one kernel, accuracy where n is padded, chunking, local
failures and rejections."""
import ctypes as C
import numpy as np
import pytest
import torch
import capital_b200 as cb
from capital_b200 import _lib
from scqr3_reference import ill_conditioned

pytestmark = pytest.mark.gpu
U = np.finfo(np.float64).eps / 2


@pytest.fixture(scope="module")
def topo():
    return cb.topo.rect(1, 0, 1)


def _batch(b, m, n, seed):
    """b distinct, well-conditioned m x n matrices on the GPU, column-major (A.mT contiguous)"""
    g = torch.Generator(device="cpu").manual_seed(seed)
    return torch.randn(b, n, m, dtype=torch.float64, generator=g).cuda().mT


def _single(topo, a, num_iter):
    """Q (m x n) and R (n x n, rect) of cacqr.factor on the one matrix a"""
    m, n = a.shape
    M = cb.matrix(n, m, 1, 1, data=a.mT.contiguous().reshape(-1).clone())
    args = cb.cacqr.info(num_iter, cb.cholinv.info(0, 1, 0, "U"), serialize=False)
    cb.cacqr.factor(M, args, topo)
    return cb.cacqr.construct_Q(args), cb.cacqr.construct_R(args), args


def _same(x, y):
    return torch.equal(x.contiguous().view(torch.int64), y.contiguous().view(torch.int64))


@pytest.mark.parametrize("n", [8, 32, 64, 128, 256, 512])
@pytest.mark.parametrize("num_iter", [1, 2, 3])
@pytest.mark.parametrize("mm", ["n", 1000, 1023, 4096])
def test_bits_match_the_single_matrix_factor(topo, n, num_iter, mm):
    m = n if mm == "n" else mm
    if m < n:
        pytest.skip("m < n")
    A = _batch(3, m, n, 17 * n + m + num_iter)
    Q, R, info = cb.cacqr.factor_batched(A, topo, num_iter)
    assert Q.shape == (3, m, n) and R.shape == (3, n, n) and info.dtype == torch.int32 and info.shape == (3,)
    assert info.tolist() == [0, 0, 0]
    for b in range(3):
        q1, r1, _ = _single(topo, A[b], num_iter)
        assert _same(Q[b], q1), b
        assert _same(R[b], r1), b


def test_row_major_input_is_copied_and_gives_the_same_bits(topo):
    A = _batch(4, 1000, 64, 5)
    Q, R, info = cb.cacqr.factor_batched(A, topo)
    Q2, R2, info2 = cb.cacqr.factor_batched(A.contiguous(), topo)  # row-major: one copy to column-major
    assert _same(Q, Q2) and _same(R, R2) and info2.tolist() == [0] * 4
    # a 16-byte misaligned column-major A (offset by one double) is read through the padded copy
    buf = torch.empty(4 * 1000 * 64 + 1, dtype=torch.float64, device="cuda")
    Am = buf[1:].view(4, 64, 1000)
    Am.copy_(A.mT)
    Q3, R3, _ = cb.cacqr.factor_batched(Am.mT, topo)
    assert _same(Q, Q3) and _same(R, R3)


def _validate(topo, a, q, r):
    """(residual, orthogonality) of the library's validator (cacqr.validate) on one matrix and its batched factors"""
    m, n = a.shape
    M = cb.matrix(n, m, 1, 1, data=a.mT.contiguous().reshape(-1).clone())
    args = cb.cacqr.info(2, cb.cholinv.info(0, 1, 0, "U"), serialize=False)
    args.Q, args.R = q.mT.contiguous().reshape(-1), r.mT.contiguous().reshape(-1)
    return cb.cacqr.validate(M, args, topo)


@pytest.mark.parametrize("n", [65, 100, 200, 511])
@pytest.mark.parametrize("num_iter", [2, 3])
def test_padded_n(topo, n, num_iter):
    m = 1500
    A = _batch(3, m, n, 1000 + n)
    Q, R, info = cb.cacqr.factor_batched(A, topo, num_iter)
    assert info.tolist() == [0, 0, 0]
    for b in range(3):
        res, orth = _validate(topo, A[b], Q[b], R[b])
        assert res <= 100 * U and orth <= 10 * U, (res, orth)
        r_ref = np.linalg.qr(A[b].cpu().numpy(), mode="r")
        r_ref = r_ref * np.sign(np.diag(r_ref))[:, None]
        kappa = np.linalg.cond(r_ref)
        assert np.linalg.norm(R[b].cpu().numpy() - r_ref) <= n * U * kappa * np.linalg.norm(r_ref)
    lower = torch.ones(n, n, dtype=torch.bool, device="cuda").tril(-1)
    assert not R[:, lower].any() and not torch.signbit(R[:, lower]).any()


def test_batch_above_the_workspace_cap_equals_separate_calls(topo):
    """n = 512, m = 4096: 300 matrices need about 15 GiB of intermediates, several chunks of the 2 GiB cap"""
    m, n, b = 4096, 512, 300
    g = torch.Generator(device="cuda").manual_seed(3)
    A = torch.randn(b, n, m, dtype=torch.float64, device="cuda", generator=g).mT
    Q, R, info = cb.cacqr.factor_batched(A, topo)
    assert int(info.abs().sum()) == 0
    for b0, b1 in ((0, 1), (1, 150), (150, 300)):
        q, r, inf = cb.cacqr.factor_batched(A[b0:b1], topo)
        assert _same(q, Q[b0:b1]) and _same(r, R[b0:b1]) and int(inf.abs().sum()) == 0
    del A, Q, R
    torch.cuda.empty_cache()


def test_many_small_matrices_equal_separate_calls(topo):
    """n = 8, m = 16: 70 000 matrices, more than one chunk of 65 535"""
    A = _batch(70000, 16, 8, 9)
    Q, R, info = cb.cacqr.factor_batched(A, topo)
    assert int(info.abs().sum()) == 0
    q, r, _ = cb.cacqr.factor_batched(A[65000:], topo)
    assert _same(q, Q[65000:]) and _same(r, R[65000:])


@pytest.mark.parametrize("n", [32, 256])
@pytest.mark.parametrize("num_iter", [1, 2, 3])
def test_failures_stay_local(topo, n, num_iter):
    A = _batch(5, 1000, n, 7 + n)
    Q, R, info = cb.cacqr.factor_batched(A, topo, num_iter)
    assert info.tolist() == [0] * 5
    bad = A.mT.contiguous().mT
    j = n // 2
    bad[2, :, j] = 0.0  # a zero column: the first Gram matrix has an exactly zero pivot at j
    Q2, R2, info2 = cb.cacqr.factor_batched(bad, topo, num_iter)
    if num_iter < 3:
        assert int(info2[2]) == j + 1
    for b in (0, 1, 3, 4):
        assert info2[b] == 0 and _same(Q2[b], Q[b]) and _same(R2[b], R[b]), b


def test_ill_conditioned_cholesky_qr2_fails_and_shifted_qr3_succeeds(topo):
    m, n, kappa = 4096, 128, 1e10
    a = torch.from_numpy(np.stack([ill_conditioned(m, n, kappa, s) for s in (1, 2, 3)])).cuda()
    _, _, info2 = cb.cacqr.factor_batched(a, topo, 2)
    assert (info2 != 0).all()
    Q, R, info3 = cb.cacqr.factor_batched(a, topo, 3)
    assert info3.tolist() == [0, 0, 0]
    for b in range(3):
        q1, r1, args = _single(topo, a[b], 3)
        assert _same(Q[b], q1) and _same(R[b], r1)
        M = cb.matrix(n, m, 1, 1, data=a[b].mT.contiguous().reshape(-1).clone())
        res, orth = cb.cacqr.validate(M, args, topo)
        assert res <= 1e-14 and orth <= 1e-15, (res, orth)  # the single path's bounds at kappa = 1e10 (test_gpu_scqr3.py)


@pytest.mark.parametrize("m,n", [(1000, 8), (1023, 100), (4096, 256), (2048, 512)])
@pytest.mark.parametrize("k", [1, 32, 33])
def test_lstsq_bits_match_the_single_lstsq(topo, m, n, k):
    A = _batch(4, m, n, m + n + k)
    Q, R, info = cb.cacqr.factor_batched(A, topo)
    g = torch.Generator(device="cpu").manual_seed(k)
    B = torch.randn(4, m, k, dtype=torch.float64, generator=g).cuda()
    X = cb.cacqr.lstsq_batched(Q, R, B, topo)
    assert X.shape == (4, n, k)
    ctx = topo.context()
    for b in range(4):
        Qc, Rc, Bc = Q[b].mT.contiguous(), R[b].mT.contiguous(), B[b].mT.contiguous()
        Xc = torch.empty(k, n, dtype=torch.float64, device="cuda")
        ctx.check(_lib.lib().capital_cacqr_lstsq_f64(ctx.handle, m, n, Qc.data_ptr(), _lib.RECT, Rc.data_ptr(), k, Bc.data_ptr(), m,
                                                     Xc.data_ptr(), n))
        assert _same(X[b], Xc.mT), b
    ref = torch.linalg.lstsq(A, B).solution
    # X is a backward-stable solution of a well-conditioned problem (kappa(A) of a few): compare normwise at 1e3 n u
    assert float(torch.linalg.norm(X - ref) / torch.linalg.norm(ref)) <= 1e3 * n * U
    x1 = cb.cacqr.lstsq_batched(Q, R, B[:, :, 0], topo)
    assert x1.shape == (4, n) and _same(x1, cb.cacqr.lstsq_batched(Q, R, B[:, :, :1], topo)[:, :, 0])


def test_c_entry_points_reject(topo):
    ctx = topo.context()
    L = _lib.lib()
    dev = torch.zeros(2 * 64 * 64, dtype=torch.float64, device="cuda")
    out = torch.zeros(2 * 64 * 64, dtype=torch.float64, device="cuda")
    host = torch.zeros(2 * 64 * 64, dtype=torch.float64)
    info = torch.zeros(2, dtype=torch.int32, device="cuda")
    p, o, i = dev.data_ptr(), out.data_ptr(), info.data_ptr()
    assert L.capital_cacqr_factor_batched_f64(ctx.handle, 600, 513, 1, 2, p, o, o, i) == _lib.ERR_UNSUPPORTED
    assert L.capital_cacqr_lstsq_batched_f64(ctx.handle, 600, 513, 1, p, p, 1, p, o) == _lib.ERR_UNSUPPORTED
    assert L.capital_cacqr_factor_batched_f64(ctx.handle, 7, 8, 2, 2, p, o, o, i) == _lib.ERR_INVALID
    assert L.capital_cacqr_lstsq_batched_f64(ctx.handle, 7, 8, 2, p, p, 1, p, o) == _lib.ERR_INVALID
    for it in (0, 4):
        assert L.capital_cacqr_factor_batched_f64(ctx.handle, 16, 8, 2, it, p, o, o, i) == _lib.ERR_INVALID
    assert L.capital_cacqr_factor_batched_f64(ctx.handle, 16, 8, 2, 2, host.data_ptr(), o, o, i) == _lib.ERR_INVALID
    assert "device pointers" in L.capital_last_error(ctx.handle).decode()
    assert L.capital_cacqr_lstsq_batched_f64(ctx.handle, 16, 8, 2, p, p, 1, host.data_ptr(), o) == _lib.ERR_INVALID
    assert L.capital_cacqr_factor_batched_f64(ctx.handle, 16, 8, 2, 2, p, p, o, i) == _lib.ERR_INVALID
    assert "overlap" in L.capital_last_error(ctx.handle).decode()
    assert L.capital_cacqr_lstsq_batched_f64(ctx.handle, 16, 8, 2, p, p, 1, o, o) == _lib.ERR_INVALID
    assert L.capital_cacqr_factor_batched_f64(ctx.handle, 16, 8, 0, 2, p, o, o, i) == _lib.ERR_INVALID
    assert L.capital_cacqr_lstsq_batched_f64(ctx.handle, 16, 8, 2, p, p, 0, p, o) == _lib.ERR_INVALID
