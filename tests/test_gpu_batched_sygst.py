"""Batched inverse, sygst (itypes 1, 2, 3), products with the factors and eigh_batched on the GPU: the single-matrix calls' bits on the
same factors, long-double references, scipy's generalized eigh, the contract (unread triangles, symmetry, aliasing, no copies), local
failures, chunking and the flop counters."""
import ctypes as C
import math
import numpy as np
import pytest
import scipy.linalg as sl
import torch
import capital_b200 as cb
from capital_b200 import _lib
import batched_sygst_reference as bs

pytestmark = pytest.mark.gpu

F64 = torch.float64


@pytest.fixture(scope="module")
def topo():
    return cb.topo.square(1, 0, 1)


def _sym(b, n, seed, device="cuda"):
    g = torch.Generator(device="cpu").manual_seed(seed)
    G = torch.randn(b, n, n, dtype=F64, generator=g)
    return (G + G.mT).to(device)


def _spd(b, n, seed):
    g = torch.Generator(device="cpu").manual_seed(seed)
    G = torch.randn(b, n, n, dtype=F64, generator=g)
    A = G @ G.mT / n + torch.eye(n, dtype=F64)
    return ((A + A.mT) / 2).cuda()


def _same(x, y):
    return torch.equal(x.contiguous().view(torch.int64), y.contiguous().view(torch.int64))


def _single_args(R, Ri):
    """a serialize=False cholinv.info holding one matrix's batched factors (column-major buffers)"""
    n = R.shape[0]
    args = cb.cholinv.info(1, 1, 0, "U", serialize=False)
    args.R, args.Rinv = R.mT.contiguous().reshape(-1), Ri.mT.contiguous().reshape(-1)
    args.local_dim = args.global_dim = n
    return args


def _mat(a):
    n = a.shape[0]
    return cb.matrix(n, n, 1, 1, data=a.mT.contiguous().reshape(-1).clone())


BITS_N = [1, 2, 7, 8, 17, 63, 64, 65, 100, 127, 128, 129, 192, 255, 256, 257, 383, 511, 512]


@pytest.mark.parametrize("n", BITS_N)
def test_bits_match_the_single_matrix_calls(topo, n):
    b = 3
    Bm = _spd(b, n, 5 * n)
    A = _sym(b, n, 5 * n + 1)
    R, Ri, info = cb.cholinv.factor_batched(Bm, topo)
    assert int(info.abs().sum()) == 0
    Ainv = cb.cholinv.inverse_batched(Ri, topo)
    C = {1: cb.cholinv.sygst_batched(A, None, Ri, topo, itype=1), 2: cb.cholinv.sygst_batched(A, R, None, topo, itype=2),
         3: cb.cholinv.sygst_batched(A, R, Ri, topo, itype=3)}
    assert _same(C[2], C[3])
    rhs = {k: torch.randn(b, n, k, dtype=F64, device="cuda", generator=torch.Generator("cuda").manual_seed(k)) for k in (1, 32, 33, 65)}
    X = {(name, k): fn(F, rhs[k], topo) for k in rhs for name, fn, F in (
        ("Rinv", cb.cholinv.apply_Rinv_batched, Ri), ("RinvT", cb.cholinv.apply_RinvT_batched, Ri),
        ("R", cb.cholinv.apply_R_batched, R), ("RT", cb.cholinv.apply_RT_batched, R))}
    for i in range(b):
        args = _single_args(R[i], Ri[i])
        assert _same(Ainv[i], cb.cholinv.inverse(args, topo).view(n, n)), i
        for it in (1, 2, 3):
            assert _same(C[it][i], cb.cholinv.sygst(_mat(A[i]), args, topo, itype=it).view(n, n)), (i, it)
        for k, B in rhs.items():
            single = {"Rinv": cb.cholinv.apply_Rinv, "RinvT": cb.cholinv.apply_RinvT, "R": cb.cholinv.apply_R, "RT": cb.cholinv.apply_RT}
            for name, fn in single.items():
                assert _same(X[(name, k)][i], fn(args, B[i], topo)), (i, name, k)


# ---- long-double references ---------------------------------------------------------------------------------------------------------
REF_N = [1, 17, 65, 200, 512]


def _ref_inputs(n):
    """(name, B, kappa) of the batch: kappa 10, kappa 1e8 and a graded D B D of the kappa = 10 matrix"""
    b10 = bs.spd_spectrum(n, 10.0, 3 * n + 2)
    b8 = bs.spd_spectrum(n, 1e8, 3 * n + 5)
    e = bs.ramp_exponents(n, 60)
    d = torch.from_numpy(np.ldexp(1.0, e.numpy()))
    bg = b10 * d[:, None] * d[None, :]
    return [("kappa10", b10), ("kappa1e8", b8), ("graded", bg)]


@pytest.mark.parametrize("n", REF_N)
def test_against_long_double_products(topo, n):
    inputs = _ref_inputs(n)
    Bm = torch.stack([t for _, t in inputs]).cuda()
    A = _sym(len(inputs), n, 77 * n)
    R, Ri, info = cb.cholinv.factor_batched(Bm, topo)
    assert int(info.abs().sum()) == 0
    Ainv = cb.cholinv.inverse_batched(Ri, topo).cpu().numpy()
    C1 = cb.cholinv.sygst_batched(A, R, Ri, topo, itype=1).cpu().numpy()
    C2 = cb.cholinv.sygst_batched(A, R, Ri, topo, itype=2).cpu().numpy()
    r, ri, a, bm = R.cpu().numpy(), Ri.cpu().numpy(), A.cpu().numpy(), Bm.cpu().numpy()
    for i, (name, _) in enumerate(inputs):
        for c, f, it in ((C1[i], ri[i], 1), (C2[i], r[i], 2)):
            ref = bs.sygst_ld(a[i], f, it)
            bound = bs.product_bound(a[i], f)
            err = float(np.linalg.norm((c - ref).astype(np.float64)))
            assert err <= bound, (name, it, err / bound)
            half = bs.sygst_half(a[i], f, it)
            for wrong in (half, np.zeros_like(c), -ref):  # the bound has teeth at this matrix
                assert float(np.linalg.norm((wrong - ref).astype(np.float64))) > bound, (name, it)
        ref = bs.inverse_ld(ri[i])
        pb = bs.inverse_product_bound(ri[i])
        assert float(np.linalg.norm((Ainv[i] - ref).astype(np.float64))) <= pb, name
        res = float(np.linalg.norm(bm[i] @ Ainv[i] - np.eye(n))) / math.sqrt(n)
        if name == "graded":  # kappa(B) ~ 2^240: reported only, and without a bound
            print(f"n={n} {name}: ||A Ainv - I||_F / sqrt(n) = {res:.3e}")
            continue
        rb = bs.inverse_residual_bound(bm[i])
        print(f"n={n} {name}: ||A Ainv - I||_F / sqrt(n) = {res:.3e}, a-priori bound {rb:.3e}")
        if name == "kappa10":
            assert res <= rb, (res, rb)


# ---- eigh_batched against scipy -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("itype", [1, 2, 3])
@pytest.mark.parametrize("n", [1, 17, 64, 129, 512])
def test_eigh_batched_against_scipy(topo, n, itype):
    Bm = torch.stack([bs.spd_spectrum(n, k, 11 * n + j) for j, k in enumerate((10.0, 1e4))]).cuda()
    A = _sym(2, n, 13 * n)
    w, X, info = cb.cholinv.eigh_batched(A, Bm, topo, itype=itype)
    assert w.shape == (2, n) and X.shape == (2, n, n) and info.tolist() == [0, 0]
    a, bm, wn, xn = A.cpu().numpy(), Bm.cpu().numpy(), w.cpu().numpy(), X.cpu().numpy()
    for i in range(2):
        wr = sl.eigh(a[i], bm[i], type=itype, eigvals_only=True)
        eb = bs.EighBounds(a[i], bm[i], itype)
        assert (np.abs(wn[i] - wr) <= eb.eigenvalues(wr)).all(), (i, float(np.abs(wn[i] - wr).max()))
        assert bs.eigh_residual(a[i], bm[i], wn[i], xn[i], itype) <= eb.residual(wn[i], xn[i]), i
        assert bs.eigh_orthonormality(bm[i], xn[i], itype) <= eb.orthonormality(), i


# ---- contract -----------------------------------------------------------------------------------------------------------------------
def test_unread_triangles_symmetry_and_aliasing(topo):
    n, b = 100, 4
    Bm = _spd(b, n, 3)
    A = _sym(b, n, 4)
    R, Ri, _ = cb.cholinv.factor_batched(Bm, topo)
    Ainv = cb.cholinv.inverse_batched(Ri, topo)
    C = {it: cb.cholinv.sygst_batched(A, R, Ri, topo, itype=it) for it in (1, 2)}
    assert Ainv.equal(Ainv.mT) and C[1].equal(C[1].mT) and C[2].equal(C[2].mT)
    upper = torch.ones(n, n, dtype=torch.bool, device="cuda").triu(1)
    An = A.clone()
    An[:, upper] = float("nan")  # A's unread triangle: the strict upper one in torch indexing
    Rn, Rin = R.clone(), Ri.clone()
    Rn[:, upper.mT] = float("nan")  # below the diagonal of the factors (torch indexing)
    Rin[:, upper.mT] = float("nan")
    assert _same(cb.cholinv.inverse_batched(Rin, topo), Ainv)
    for it in (1, 2):
        assert _same(cb.cholinv.sygst_batched(An, R, Ri, topo, itype=it), C[it])
        assert _same(cb.cholinv.sygst_batched(A, Rn, Rin, topo, itype=it), C[it])
    B = torch.randn(b, n, 40, dtype=F64, device="cuda", generator=torch.Generator("cuda").manual_seed(1))
    ctx = topo.context()
    L = _lib.lib()
    for F, Fn, fn, cfn in ((Ri, Rin, cb.cholinv.apply_Rinv_batched, L.capital_cholinv_apply_rinv_batched_f64),
                           (R, Rn, cb.cholinv.apply_R_batched, L.capital_cholinv_apply_r_batched_f64)):
        for trans in (0, 1):
            Bc = B.mT.contiguous()
            Xc = torch.empty_like(Bc)
            ctx.check(cfn(ctx.handle, n, b, F.mT.contiguous().data_ptr(), trans, 40, Bc.data_ptr(), Xc.data_ptr()))
            Xn = torch.empty_like(Bc)
            ctx.check(cfn(ctx.handle, n, b, Fn.mT.contiguous().data_ptr(), trans, 40, Bc.data_ptr(), Xn.data_ptr()))
            assert _same(Xn, Xc)
            XB = Bc.clone()  # X aliases B
            ctx.check(cfn(ctx.handle, n, b, F.mT.contiguous().data_ptr(), trans, 40, XB.data_ptr(), XB.data_ptr()))
            assert _same(XB, Xc)
            if trans == 0:
                assert _same(fn(F, B, topo), Xc.mT)
    # overlapping outputs are refused
    buf = torch.zeros(2 * b * n * n, dtype=F64, device="cuda")
    p = buf.data_ptr()
    assert L.capital_cholinv_inverse_batched_f64(ctx.handle, n, b, p, p + 8 * (b * n * n - 1)) == _lib.ERR_INVALID
    assert L.capital_cholinv_sygst_batched_f64(ctx.handle, n, b, p, p + 8 * b * n * n, p + 8) == _lib.ERR_INVALID
    assert L.capital_cholinv_sygst_ab_batched_f64(ctx.handle, n, b, p, p + 8 * b * n * n, p + 8 * b * n * n) == _lib.ERR_INVALID


def test_c_entry_points_reject_bad_arguments(topo):
    ctx = topo.context()
    L = _lib.lib()
    dev = torch.zeros(3 * 2 * 16 * 16, dtype=F64, device="cuda")
    host = torch.zeros(2 * 16 * 16, dtype=F64)
    p, q, r, h = dev.data_ptr(), dev.data_ptr() + 8 * 512, dev.data_ptr() + 16 * 512, host.data_ptr()
    assert L.capital_cholinv_inverse_batched_f64(ctx.handle, 16, 2, h, q) == _lib.ERR_INVALID
    assert "device pointers" in L.capital_last_error(ctx.handle).decode()
    assert L.capital_cholinv_sygst_batched_f64(ctx.handle, 16, 2, p, h, r) == _lib.ERR_INVALID
    assert L.capital_cholinv_sygst_ab_batched_f64(ctx.handle, 16, 2, p, q, None) == _lib.ERR_INVALID
    assert L.capital_cholinv_apply_rinv_batched_f64(ctx.handle, 16, 2, p, 2, 1, q, q) == _lib.ERR_INVALID
    assert "trans" in L.capital_last_error(ctx.handle).decode()
    assert L.capital_cholinv_apply_r_batched_f64(ctx.handle, 16, 2, p, 0, 0, q, q) == _lib.ERR_INVALID
    assert L.capital_cholinv_apply_r_batched_f64(ctx.handle, 16, 0, p, 0, 1, q, q) == _lib.ERR_INVALID
    assert L.capital_cholinv_apply_r_batched_f64(ctx.handle, 0, 2, p, 0, 1, q, q) == _lib.ERR_INVALID
    for fn, extra in ((L.capital_cholinv_inverse_batched_f64, ()), (L.capital_cholinv_sygst_batched_f64, (r,)),
                      (L.capital_cholinv_sygst_ab_batched_f64, (r,))):
        assert fn(ctx.handle, 513, 1, p, q, *extra) == _lib.ERR_UNSUPPORTED
    assert L.capital_cholinv_apply_rinv_batched_f64(ctx.handle, 513, 1, p, 0, 1, q, q) == _lib.ERR_UNSUPPORTED
    assert L.capital_cholinv_apply_r_batched_f64(ctx.handle, 513, 1, p, 1, 1, q, q) == _lib.ERR_UNSUPPORTED


def test_wrappers_take_factor_batched_outputs_without_a_copy(topo):
    """the only tensor the wrappers allocate is the result: R, Rinv (.mT views of column-major buffers) go in as they are"""
    n, b = 256, 64
    R, Ri, _ = cb.cholinv.factor_batched(_spd(b, n, 9), topo)
    A = _sym(b, n, 10)
    out_bytes = b * n * n * 8
    for call in (lambda: cb.cholinv.inverse_batched(Ri, topo), lambda: cb.cholinv.sygst_batched(A, None, Ri, topo, itype=1),
                 lambda: cb.cholinv.sygst_batched(A, R, None, topo, itype=3)):
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        out = call()
        torch.cuda.synchronize()
        assert torch.cuda.max_memory_allocated() - base <= out_bytes, torch.cuda.max_memory_allocated() - base
        del out
    B = torch.randn(b, n, 1, dtype=F64, device="cuda")
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    x = cb.cholinv.apply_RT_batched(R, B, topo)
    torch.cuda.synchronize()
    assert torch.cuda.max_memory_allocated() - base <= 4 * b * n * 8  # B's column-major copy, X and its layout: no factor-sized buffer
    del x


# ---- failures -----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("itype", [1, 2, 3])
@pytest.mark.parametrize("n", [64, 129])
def test_eigh_failures_stay_local(topo, n, itype):
    b = 7
    Bm = _spd(b, n, 21 * n)
    A = _sym(b, n, 22 * n)
    w, X, info = cb.cholinv.eigh_batched(A, Bm, topo, itype=itype)
    assert int(info.abs().sum()) == 0
    bad = Bm.clone()
    k = n // 2 + 1
    for i in (0, b // 2, b - 1):
        bad[i, k, k] = -1.0
    w2, X2, info2 = cb.cholinv.eigh_batched(A, bad, topo, itype=itype)  # no exception
    _, _, ref_info = cb.cholinv.factor_batched(bad, topo)
    assert torch.equal(info2, ref_info) and info2.tolist() == [k + 1 if i in (0, b // 2, b - 1) else 0 for i in range(b)]
    for i in range(b):
        if i in (0, b // 2, b - 1):
            assert torch.isnan(w2[i]).all() and torch.isnan(X2[i]).all(), i
        else:
            assert _same(w2[i], w[i]) and _same(X2[i], X[i]), i


# ---- chunking and counters ------------------------------------------------------------------------------------------------------------
def _launches(topo, fn):
    ctx = topo.context()
    torch.cuda.synchronize()
    ctx.reset_counters()
    fn()
    torch.cuda.synchronize()
    c = ctx.counters()
    return c.kernel_launches, c.gemm_launches


def test_chunk_size_at_n512(topo):
    n = 512
    ctx = topo.context()
    L = _lib.lib()
    for call in ("inverse", "sygst", "sygst_ab", "apply_rinv", "apply_r"):
        ch = bs.chunk(call, n, 10 ** 9)
        F = torch.eye(n, dtype=F64, device="cuda").expand(ch + 1, n, n).contiguous()
        big = call.startswith("apply")
        A = None if big else torch.eye(n, dtype=F64, device="cuda").expand(ch + 1, n, n).contiguous()
        B = torch.ones(ch + 1, n, dtype=F64, device="cuda") if big else None
        out = torch.empty((ch + 1, n) if big else (ch + 1, n, n), dtype=F64, device="cuda")

        def run(cnt):
            if call == "inverse":
                ctx.check(L.capital_cholinv_inverse_batched_f64(ctx.handle, n, cnt, F.data_ptr(), out.data_ptr()))
            elif call in ("sygst", "sygst_ab"):
                fn = getattr(L, f"capital_cholinv_{call}_batched_f64")
                ctx.check(fn(ctx.handle, n, cnt, F.data_ptr(), A.data_ptr(), out.data_ptr()))
            else:
                fn = getattr(L, f"capital_cholinv_{call}_batched_f64")
                ctx.check(fn(ctx.handle, n, cnt, F.data_ptr(), 0, 1, B.data_ptr(), out.data_ptr()))

        one = _launches(topo, lambda: run(1))
        assert _launches(topo, lambda: run(ch)) == one, call
        assert _launches(topo, lambda: run(ch + 1)) == (2 * one[0], 2 * one[1]), call
        if not big:
            assert torch.equal(out[:ch + 1], torch.eye(n, dtype=F64, device="cuda").expand(ch + 1, n, n)), call
        del F, A, B, out
        torch.cuda.empty_cache()


def test_tail_of_70000_matrices_matches_a_separate_call(topo):
    n, b = 8, 70000
    Bm = _spd(b, n, 1)
    A = _sym(b, n, 2)
    R, Ri, info = cb.cholinv.factor_batched(Bm, topo)
    assert int(info.abs().sum()) == 0
    rhs = torch.randn(b, n, 3, dtype=F64, device="cuda", generator=torch.Generator("cuda").manual_seed(3))
    calls = {"inverse": lambda r, ri, a, x: cb.cholinv.inverse_batched(ri, topo),
             "sygst1": lambda r, ri, a, x: cb.cholinv.sygst_batched(a, r, ri, topo, itype=1),
             "sygst3": lambda r, ri, a, x: cb.cholinv.sygst_batched(a, r, ri, topo, itype=3),
             "apply_Rinv": lambda r, ri, a, x: cb.cholinv.apply_Rinv_batched(ri, x, topo),
             "apply_RinvT": lambda r, ri, a, x: cb.cholinv.apply_RinvT_batched(ri, x, topo),
             "apply_R": lambda r, ri, a, x: cb.cholinv.apply_R_batched(r, x, topo),
             "apply_RT": lambda r, ri, a, x: cb.cholinv.apply_RT_batched(r, x, topo)}
    t0 = 65535 - 5
    for name, fn in calls.items():
        whole = fn(R, Ri, A, rhs)
        tail = fn(R[t0:], Ri[t0:], A[t0:], rhs[t0:])
        assert _same(whole[t0:], tail), name


@pytest.mark.parametrize("n", [96, 192])
def test_gemm_flops_are_batch_times_the_single_call(topo, n):
    """n divisible by 3: every count is an integer, so the sums are exact"""
    b = 5
    ctx = topo.context()
    R, Ri, _ = cb.cholinv.factor_batched(_spd(b, n, 31), topo)
    A = _sym(b, n, 32)
    args = _single_args(R[0], Ri[0])

    def flops(fn):
        torch.cuda.synchronize()
        ctx.reset_counters()
        fn()
        torch.cuda.synchronize()
        return ctx.counters().gemm_flops

    assert flops(lambda: cb.cholinv.inverse_batched(Ri, topo)) == b * flops(lambda: cb.cholinv.inverse(args, topo)) == b * n ** 3 / 3
    for it in (1, 2, 3):
        single = flops(lambda: cb.cholinv.sygst(_mat(A[0]), args, topo, itype=it))
        assert single == n ** 3
        assert flops(lambda: cb.cholinv.sygst_batched(A, R, Ri, topo, itype=it)) == b * single, it
