"""Batched CholInv on the GPU (capital_cholinv_factor_batched_f64 / capital_cholinv_solve_batched_f64): the same bits as the
single-matrix factor, padding, local failures, scaling, chunking and the solve."""
import ctypes as C
import re
import numpy as np
import pytest
import torch
import capital_b200 as cb
from capital_b200 import _lib

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def topo():
    return cb.topo.square(1, 0, 1)


def _spd(b, n, seed):
    """b distinct, exactly symmetric SPD matrices (condition number in the tens)"""
    g = torch.Generator(device="cpu").manual_seed(seed)
    G = torch.randn(b, n, n, dtype=torch.float64, generator=g)
    A = G @ G.mT / n + torch.eye(n, dtype=torch.float64)
    return ((A + A.mT) / 2).cuda()


def _single(topo, a):
    """R, Rinv of one matrix from cholinv.factor on a base case that covers n: a single leaf or width-8 cluster launch"""
    n = a.shape[0]
    M = cb.matrix(n, n, 1, 1, data=a.contiguous().reshape(-1).clone())
    args = cb.cholinv.info(1, 1, 0, "U", serialize=False)
    cb.cholinv.factor(M, args, topo)
    return args.R.view(n, n).t(), args.Rinv.view(n, n).t()


def _same(x, y):
    return torch.equal(x.contiguous().view(torch.int64), y.contiguous().view(torch.int64))


@pytest.mark.parametrize("n", [8, 64, 128, 192, 256, 512])
def test_bits_match_the_single_matrix_factor(topo, n):
    A = _spd(5, n, n)
    R, Ri, info = cb.cholinv.factor_batched(A, topo)
    assert R.shape == (5, n, n) and Ri.shape == (5, n, n) and info.dtype == torch.int32 and info.shape == (5,)
    assert int(info.abs().sum()) == 0
    for b in range(5):
        r1, ri1 = _single(topo, A[b])
        assert _same(R[b], r1) and _same(Ri[b], ri1), b
    assert torch.allclose(R.mT @ R, A, rtol=0, atol=1e-12 * float(A.abs().max()))


@pytest.mark.parametrize("n", [1, 65, 100, 200, 511])
def test_padding(topo, n):
    A = _spd(3, n, 1000 + n)
    R, Ri, info = cb.cholinv.factor_batched(A, topo)
    assert int(info.abs().sum()) == 0
    a = A.cpu().numpy()
    u = np.finfo(np.float64).eps
    for b in range(3):
        r_ref = np.linalg.cholesky(a[b]).T
        ri_ref = np.linalg.inv(r_ref)
        cond = np.linalg.cond(r_ref)
        r, ri = R[b].cpu().numpy(), Ri[b].cpu().numpy()
        assert np.linalg.norm(r - r_ref) <= 10 * n * u * cond * np.linalg.norm(r_ref)
        assert np.linalg.norm(ri - ri_ref) <= 10 * n * u * cond * np.linalg.norm(ri_ref)
    lower = torch.ones(n, n, dtype=torch.bool, device="cuda").tril(-1)
    assert not R[:, lower].any() and not Ri[:, lower].any()
    assert not torch.signbit(R[:, lower]).any() and not torch.signbit(Ri[:, lower]).any()
    # the triangle that is not read (the strict upper one in torch indexing) may hold anything
    An = A.clone()
    An[:, ~lower & ~torch.eye(n, dtype=torch.bool, device="cuda")] = float("nan")
    R2, Ri2, info2 = cb.cholinv.factor_batched(An, topo)
    assert _same(R2, R) and _same(Ri2, Ri) and torch.equal(info2, info)


@pytest.mark.parametrize("n", [32, 256])
def test_failures_stay_local(topo, n):
    A = _spd(5, n, 7 + n)
    R, Ri, info = cb.cholinv.factor_batched(A, topo)
    assert int(info.abs().sum()) == 0
    bad = A.clone()
    k = n // 2 + 3
    bad[2, k, k] = -1.0
    R2, Ri2, info2 = cb.cholinv.factor_batched(bad, topo)  # no exception: info only
    with pytest.raises(_lib.CapitalError, match="non-positive pivot") as e:
        _single(topo, bad[2])
    pivot = int(re.search(r"non-positive pivot (\d+)", str(e.value)).group(1))
    assert pivot == k + 1
    assert info2.tolist() == [0, 0, pivot, 0, 0]
    for b in (0, 1, 3, 4):
        assert _same(R2[b], R[b]) and _same(Ri2[b], Ri[b]), b


@pytest.mark.parametrize("n", [8, 256])
def test_scaled_matrices_match_the_single_matrix_factor(topo, n):
    A = _spd(4, n, 3 * n)
    A = A * torch.tensor([2.0 ** 600, 2.0 ** -600, 1.0, 2.0 ** 600], dtype=torch.float64, device="cuda").view(4, 1, 1)
    R, Ri, info = cb.cholinv.factor_batched(A, topo)
    assert int(info.abs().sum()) == 0
    for b in range(4):
        r1, ri1 = _single(topo, A[b])
        assert _same(R[b], r1) and _same(Ri[b], ri1), b
        assert torch.isfinite(R[b]).all() and torch.isfinite(Ri[b]).all()


@pytest.mark.parametrize("n,batch,parts", [(512, 600, 2), (8, 70000, 2), (200, 301, 3)])
def test_chunked_batches_equal_separate_calls(topo, n, batch, parts):
    """n = 512: 600 matrices need 2.4 GiB of intermediates, above the 2 GiB cap; n = 8: a leaf grid of 70000 CTAs"""
    g = torch.Generator(device="cuda").manual_seed(n)
    A = torch.randn(batch, n, n, dtype=torch.float64, device="cuda", generator=g) * 0.1 / n ** 0.5
    A = A + A.mT + torch.eye(n, dtype=torch.float64, device="cuda")
    R, Ri, info = cb.cholinv.factor_batched(A, topo)
    assert int(info.abs().sum()) == 0
    edges = np.linspace(0, batch, parts + 1).astype(int)
    for b0, b1 in zip(edges[:-1], edges[1:]):
        r, ri, inf = cb.cholinv.factor_batched(A[b0:b1], topo)
        assert _same(r, R[b0:b1]) and _same(ri, Ri[b0:b1]) and int(inf.abs().sum()) == 0
    del A, R, Ri
    torch.cuda.empty_cache()


@pytest.mark.parametrize("n", [8, 100, 512])
@pytest.mark.parametrize("k", [1, 32, 33])
def test_solve_matches_cholesky_solve(topo, n, k):
    A = _spd(6, n, 11 * n + k)
    R, Ri, info = cb.cholinv.factor_batched(A, topo)
    g = torch.Generator(device="cpu").manual_seed(k)
    B = torch.randn(6, n, k, dtype=torch.float64, generator=g).cuda()
    ref = torch.cholesky_solve(B, torch.linalg.cholesky(A))
    X = cb.cholinv.solve_batched(Ri, B, topo)
    assert X.shape == B.shape
    assert float((X - ref).abs().max() / ref.abs().max()) <= 1e-12
    # the C entry point in place: X aliases B (column-major n x k per matrix)
    XB = B.mT.contiguous()
    ctx = topo.context()
    ctx.check(_lib.lib().capital_cholinv_solve_batched_f64(ctx.handle, n, 6, Ri.mT.contiguous().data_ptr(), k, XB.data_ptr(),
                                                           XB.data_ptr()))
    assert _same(XB.mT, X)
    x1 = cb.cholinv.solve_batched(Ri, B[:, :, 0], topo)
    assert x1.shape == (6, n) and _same(x1, cb.cholinv.solve_batched(Ri, B[:, :, :1], topo)[:, :, 0])


def test_c_entry_points_reject_host_pointers_and_large_n(topo):
    ctx = topo.context()
    L = _lib.lib()
    dev = torch.zeros(2 * 16 * 16, dtype=torch.float64, device="cuda")
    host = torch.zeros(2 * 16 * 16, dtype=torch.float64)
    info = torch.zeros(2, dtype=torch.int32, device="cuda")
    p = dev.data_ptr()
    assert L.capital_cholinv_factor_batched_f64(ctx.handle, 16, 2, host.data_ptr(), p, p, info.data_ptr()) == _lib.ERR_INVALID
    assert "device pointers" in L.capital_last_error(ctx.handle).decode()
    assert L.capital_cholinv_solve_batched_f64(ctx.handle, 16, 2, p, 1, host.data_ptr(), p) == _lib.ERR_INVALID
    assert L.capital_cholinv_factor_batched_f64(ctx.handle, 513, 1, p, p, p, info.data_ptr()) == _lib.ERR_UNSUPPORTED
    assert L.capital_cholinv_solve_batched_f64(ctx.handle, 513, 1, p, 1, p, p) == _lib.ERR_UNSUPPORTED
    assert L.capital_cholinv_factor_batched_f64(ctx.handle, 16, 0, p, p, p, info.data_ptr()) == _lib.ERR_INVALID
    assert L.capital_cholinv_solve_batched_f64(ctx.handle, 16, 2, p, 0, p, p) == _lib.ERR_INVALID
