"""The split-k Gram product G = A^T A (gemm_tn_splitk) behind every CholeskyQR sweep and the orthogonality validator, checked against
FP64 torch on the device at the row counts where its k-chunking changes, and every single-GPU entry point run on a context whose
workspaces start as NaN (CAPITAL_POISON_WORKSPACE=1), so that a read of a value nobody wrote cannot go unnoticed.

Gram bound.  With num_iter = 1, R = chol(G).  The product and Cholesky are backward stable elementwise, so
    |R^T R - A^T A| <= 2 (gamma_k |A|^T |A| + gamma_{n+1} |R|^T |R|),   gamma_j = j u / (1 - j u)
(the 2 covers the rounding of the reference's own products).  The bound does not depend on the condition number, and losing a
single row of A moves G by about 1/k relative, far above gamma_k."""
import functools
import math
import os, subprocess, sys
import pytest
import torch
import capital_b200 as cb
from capital_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
U = 2.0 ** -53
NS = (17, 64, 96, 128, 129, 192, 256)


def _cdiv(a, b):
    return -(-a // b)


# ---- chunk arithmetic of gemm_tn_splitk (capital_b200/csrc/gemm_tn.cu): change it together with that function ----------------------
def splitk_chunks(n, k, c_upper, sms):
    """(ks, empty) for the n x n product over k rows on `sms` SMs: ks chunks are launched, chunk z takes the k tiles
    [z per, min(nk, (z + 1) per)) with per = ceil(nk / ks), and `empty` of them get no tile"""
    big = n >= 128
    t = 128 if big else 64
    g = _cdiv(n, t)
    tiles = g * (g + 1) // 2 if c_upper else g * g  # C_UPPER: the tiles below the diagonal are not launched work
    ks_sms = _cdiv(sms * (1 if big else 2), tiles)
    ks = max(1, min(ks_sms, _cdiv(k, 16 * 32)))  # at least 32 k tiles per chunk
    nk = _cdiv(k, 16)
    per = _cdiv(nk, ks)
    return ks, ks - _cdiv(nk, per)


def splitk_ks_sms(n, c_upper, sms):
    """ks when it is capped by the SM count, not by k"""
    return splitk_chunks(n, 1 << 40, c_upper, sms)[0]


@functools.lru_cache(maxsize=None)
def first_empty_k(n, c_upper, sms, limit=1 << 21):
    """the smallest k <= limit with an empty chunk, or None.  ks and the chunking depend on k only through nk = ceil(k / 16)
    (512 = 32 x 16), so the first k of each nk is enough"""
    for nk in range(1, limit // 16 + 1):
        k = 16 * (nk - 1) + 1
        if splitk_chunks(n, k, c_upper, sms)[1] > 0:
            return k
    return None


def gram_k_cases(n, c_upper, sms):
    """row counts that cover the chunk edges of one n: k < 512 (one chunk), ks capped by k, ks capped by the SM count (neither a
    multiple of 16), and the first k with an empty chunk with the k just below it (every chunk used)"""
    ks_sms = splitk_ks_sms(n, c_upper, sms)
    few = 512 * max(2, ks_sms // 2) - 5
    many = 512 * ks_sms + 16 * 5 + 3
    ks = [300, few, many]
    assert splitk_chunks(n, 300, c_upper, sms)[0] == 1
    assert 1 < splitk_chunks(n, few, c_upper, sms)[0] == _cdiv(few, 512) < ks_sms
    assert splitk_chunks(n, many, c_upper, sms)[0] == ks_sms < _cdiv(many, 512)
    ke = first_empty_k(n, c_upper, sms)
    if ke is not None:
        assert splitk_chunks(n, ke - 1, c_upper, sms) == (splitk_chunks(n, ke, c_upper, sms)[0], 0)
        ks += [ke - 1, ke]
    return ks


def test_chunk_helper_on_132_sms():
    """the helper restates the H100 SXM (132 SMs) shapes where a chunk is empty: n <= 64 from 135169 rows (7 of 264 chunks empty),
    n = 128 from 67585 (3 of 132), n = 129 ... 256 from 22529 (1 of 44) in the factor's C_UPPER product, n = 65 ... 127 from 33793
    (1 of 66) in the validator's full product; none at n = 320, nor in the validator's product at n = 256, up to 2^21 rows"""
    assert [(first_empty_k(n, True, 132), splitk_chunks(n, first_empty_k(n, True, 132), True, 132)) for n in (17, 64, 128, 256)] == [
        (135169, (264, 7)), (135169, (264, 7)), (67585, (132, 3)), (22529, (44, 1))]
    assert first_empty_k(96, False, 132) == 33793 and splitk_chunks(96, 33793, False, 132) == (66, 1)
    assert first_empty_k(320, True, 132) is None and first_empty_k(256, False, 132) is None
    for n in NS:
        for k in gram_k_cases(n, True, 132):
            assert splitk_chunks(n, k, True, 132)[0] >= 1


# ---- GPU ----------------------------------------------------------------------------------------------------------------------------
def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


@pytest.fixture(scope="module")
def topo():
    return cb.topo.rect(1, 0, 1)


def _gamma(j):
    return j * U / (1 - j * U)


def gram_bound_ratio(a, r):
    """max over the entries of |R^T R - A^T A| / (2 (gamma_k |A|^T |A| + gamma_{n+1} |R|^T |R|)) for a: (k, n), r: (n, n) upper,
    FP64 torch tensors on the device; <= 1 passes"""
    k, n = a.shape
    aa, rr = a.abs(), r.abs()
    bound = 2.0 * (_gamma(k) * (aa.T @ aa) + _gamma(n + 1) * (rr.T @ rr))
    return ((r.T @ r - a.T @ a).abs() / bound).max().item()


def orth_torch(q):
    """||Q^T Q - I||_F / n (test/qr/validate.hpp)"""
    n = q.shape[1]
    return (torch.linalg.matrix_norm(q.T @ q - torch.eye(n, dtype=q.dtype, device=q.device)) / n).item()


def _random(topo, m, n, key):
    return cb.matrix(n, m, 1, 1).distribute_random(topo, key)


def _user(m, n, seed):
    """Gaussian columns scaled over two decades, handed over as user data"""
    g = torch.Generator(device="cuda").manual_seed(seed)
    a = torch.randn(m, n, dtype=torch.float64, device="cuda", generator=g) * torch.logspace(0, 2, n, dtype=torch.float64, device="cuda")
    return cb.matrix(n, m, 1, 1, data=a.t().contiguous().view(-1))


def _factor(topo, A, num_iter=1, serialize=True):
    args = cb.cacqr.info(num_iter, cb.cholinv.info(0, 1, 0, "U"), serialize=serialize)
    cb.cacqr.factor(A, args, topo)
    return args


def _check_gram(topo, A, serialize=True, what=""):
    args = _factor(topo, A, 1, serialize)
    ratio = gram_bound_ratio(A.view2d(), cb.cacqr.construct_R(args))
    assert ratio <= 1.0, f"{what}: |R^T R - A^T A| is {ratio:.3g} x the backward-error bound"
    return args


def _check_orth(topo, A, args, what=""):
    m = A.num_rows_global
    _, orth = cb.cacqr.validate(A, args, topo)
    ref = orth_torch(cb.cacqr.construct_Q(args))
    assert math.isfinite(orth) and abs(orth - ref) <= 2 * m * U, f"{what}: validate orthogonality {orth:.6g}, torch {ref:.6g}"


@pytest.mark.gpu
@pytest.mark.parametrize("source", ["random", "user"])
@pytest.mark.parametrize("serialize", [True, False])
@pytest.mark.parametrize("n", NS)
def test_gram_through_r_at_the_chunk_edges(topo, n, serialize, source):
    sms = _sms()
    for i, k in enumerate(gram_k_cases(n, True, sms)):
        A = _random(topo, k, n, 5 + i) if source == "random" else _user(k, n, 5 + i)
        _check_gram(topo, A, serialize, f"k={k} n={n} chunks={splitk_chunks(n, k, True, sms)}")


def _sequence(n, c_upper):
    """(P, Q) row counts with the same ks: every chunk of P is used, Q has an empty one"""
    kq = first_empty_k(n, c_upper, _sms())
    assert kq is not None, f"no empty-chunk shape for n = {n}"
    ks, empty = splitk_chunks(n, kq, c_upper, _sms())
    assert empty > 0 and splitk_chunks(n, kq - 1, c_upper, _sms()) == (ks, 0)
    return kq - 1, kq


@pytest.mark.gpu
def test_helper_finds_empty_chunks_on_this_device():
    for n in (64, 128, 256):
        assert first_empty_k(n, True, _sms()) is not None, n


@pytest.mark.gpu
@pytest.mark.parametrize("n", [256, 128, 64])
def test_no_stale_partials_after_a_product_with_the_same_chunking(topo, n):
    """factor P (every chunk used), then Q (same ks and n, an empty chunk): Q's Gram matrix must not pick up P's partial sums"""
    kp, kq = _sequence(n, True)
    for k, key in ((kp, 11), (kq, 12)):
        A = _random(topo, k, n, key)
        args = _check_gram(topo, A, True, f"k={k} n={n}")
        _check_orth(topo, A, args, f"k={k} n={n}")


@pytest.mark.gpu
def test_no_stale_partials_in_the_validator(topo):
    """the validator's full (flags 0) product has other chunk edges: at n = 96 its first empty chunk comes before the factor's"""
    kp, kq = _sequence(96, False)
    for k, key in ((kp, 13), (kq, 14)):
        A = _random(topo, k, 96, key)
        args = _check_gram(topo, A, True, f"k={k} n=96")
        _check_orth(topo, A, args, f"k={k} n=96")


@pytest.mark.gpu
@pytest.mark.parametrize("num_iter", [2, 3])
def test_cholesky_qr2_and_qr3_at_an_empty_chunk_shape(topo, num_iter):
    """every sweep's Gram product has empty chunks: Q and R against torch (Householder R with a positive diagonal)"""
    n = 128
    m = first_empty_k(n, True, _sms())
    A = _user(m, n, 15)
    args = _factor(topo, A, num_iter)
    a = A.view2d()
    q, r = cb.cacqr.construct_Q(args), cb.cacqr.construct_R(args)
    r_ref = torch.linalg.qr(a, mode="r")[1]
    r_ref = r_ref * torch.sign(torch.diagonal(r_ref)).unsqueeze(1)
    assert (r - r_ref).abs().max().item() <= 1e-12 * r_ref.abs().max().item()
    assert orth_torch(q) <= 1e-14
    assert (torch.linalg.matrix_norm(q @ r - a) / torch.linalg.matrix_norm(a)).item() <= 1e-14
    _check_orth(topo, A, args, f"num_iter={num_iter}")


@pytest.mark.gpu
def test_row_grid_with_two_ranks_sharing_one_gpu():
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1",
           "--master-port", "29803", os.path.join(ROOT, "tests", "mp_worker_gram.py")]
    env = dict(os.environ, CAPITAL_MP_SAME_DEVICE="1")
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=900, env=env)
    assert r.returncode == 0 and "MP_OK" in r.stdout, r.stdout[-3000:] + r.stderr[-3000:]
    print("\n" + [l for l in r.stdout.splitlines() if l.startswith("MP_OK")][0])


# ---- poisoned workspaces --------------------------------------------------------------------------------------------------------------
class _Poisoned:
    """topo stand-in with its own context made under CAPITAL_POISON_WORKSPACE=1: every workspace it (re)allocates starts as NaN.
    context() frees the workspaces first, so that every call of an entry point (each asks for the context once) runs on fresh,
    poisoned buffers.  The forced 3D QR path is left out: its degenerate-grid buffer holds the peer exchange layout."""

    def __init__(self, topo):
        self.grid = topo.grid
        old = os.environ.get("CAPITAL_POISON_WORKSPACE")
        os.environ["CAPITAL_POISON_WORKSPACE"] = "1"
        try:
            self.ctx = _lib.Context(topo.grid, torch.cuda.current_device(), torch.cuda.current_stream().cuda_stream or 0x1)
        finally:
            if old is None:
                del os.environ["CAPITAL_POISON_WORKSPACE"]
            else:
                os.environ["CAPITAL_POISON_WORKSPACE"] = old

    def context(self):
        self.ctx.release_workspace()
        return self.ctx


@pytest.fixture(scope="module")
def poisoned(topo):
    p = _Poisoned(topo)
    yield p
    p.ctx.close()


def _host(A):
    return cb.matrix(A.num_columns_global, A.num_rows_global, 1, 1, data=A.data.cpu().pin_memory())


def _cholinv_outputs(t, A, ci, serialize):
    n = A.num_rows_global
    args = cb.cholinv.info(ci, 1, 0, "U", serialize=serialize)
    cb.cholinv.factor(A, args, t)
    dev = A.data.device
    b = torch.linspace(-1.0, 1.0, n * 3, dtype=torch.float64).view(n, 3).to(dev)
    X = cb.cholinv.solve(args, b, t)
    x1 = cb.cholinv.solve(args, b[:, 0].contiguous(), t)
    Ainv = cb.cholinv.inverse(args, t)
    out = {"R": args.R.clone(), "Rinv": args.Rinv.clone(), "X": X, "x1": x1, "Ainv": Ainv}
    scal = {"residual": cb.cholinv.residual(A, args, t), "inverse_residual": cb.cholinv.inverse_residual(A, Ainv, args, t)}
    return out, scal


def _cacqr_outputs(t, A, num_iter, serialize=True):
    args = cb.cacqr.info(num_iter, cb.cholinv.info(0, 1, 0, "U"), serialize=serialize)
    cb.cacqr.factor(A, args, t)
    m, n = A.num_rows_global, A.num_columns_global
    dev = A.data.device
    b = torch.linspace(-1.0, 1.0, m * 3, dtype=torch.float64).view(m, 3).to(dev)
    z = torch.linspace(-1.0, 1.0, n * 2, dtype=torch.float64).view(n, 2).to(dev)
    out = {"Q": args.Q.clone(), "R": args.R.clone(), "QTb": cb.cacqr.apply_QT(b, args, t), "Qz": cb.cacqr.apply_Q(z, args, t),
           "X": cb.cacqr.lstsq(args, b, t), "x1": cb.cacqr.lstsq(args, b[:, 1].contiguous(), t)}
    res, orth = cb.cacqr.validate(A, args, t)
    return out, {"residual": res, "orthogonality": orth}


def _same(plain, poisoned, what):
    (out0, scal0), (out1, scal1) = plain, poisoned
    for k in out0:
        assert bool(torch.isfinite(out1[k]).all()), f"{what}: {k} is not finite on poisoned workspaces"
        assert torch.equal(out0[k], out1[k]), f"{what}: {k} differs on poisoned workspaces"
    # the validators' sums of squares are added with atomics: the last bits may differ between runs
    for k in scal0:
        assert math.isfinite(scal1[k]) and abs(scal1[k] - scal0[k]) <= 1e-10 * abs(scal0[k]), (what, k, scal0[k], scal1[k])


@pytest.mark.gpu
@pytest.mark.parametrize("n,ci,serialize,host", [(9000, 1, True, False), (9000, 0, True, False), (3001, 0, True, True),
                                                 (3001, 1, False, True), (1000, 0, False, False)])
def test_cholinv_entry_points_on_poisoned_workspaces(topo, poisoned, n, ci, serialize, host):
    A = cb.matrix(n, n, 1, 1).distribute_symmetric(topo)
    if host:
        A = _host(A)
    _same(_cholinv_outputs(topo, A, ci, serialize), _cholinv_outputs(poisoned, A, ci, serialize), f"cholinv n={n} ci={ci}")


@pytest.mark.gpu
@pytest.mark.parametrize("num_iter", [1, 2, 3])
@pytest.mark.parametrize("shape,host,serialize", [("empty-chunk", False, True), ((65539, 96), False, False), ((65539, 96), True, True),
                                                  ((4096, 1000), False, True)])
def test_cacqr_entry_points_on_poisoned_workspaces(topo, poisoned, num_iter, shape, host, serialize):
    """the empty-chunk shape is the first k where the factor's and the validator's n = 128 products (same chunking) leave chunks
    empty; (65539, 96) has an odd row count (the panel is copied to an aligned buffer)"""
    m, n = (first_empty_k(128, True, _sms()), 128) if shape == "empty-chunk" else shape
    A = _user(m, n, 17)
    if host:
        A = _host(A)
    _same(_cacqr_outputs(topo, A, num_iter, serialize), _cacqr_outputs(poisoned, A, num_iter, serialize),
          f"cacqr m={m} n={n} num_iter={num_iter}")
