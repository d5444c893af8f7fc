"""Batched CholInv and CholeskyQR against long-double references (batched_reference.py): odd n on the leaf path, the padded sizes and
the cluster widths 2 / 4 / 8, ill-conditioned, graded and mixed-scale batches, local failures in LAPACK's numbering, and failures
and healthy matrices on both sides of every chunk edge of the four entry points.

Each test prints the worst ratio of each bound it gates ("[batched-ref] ..."), so the margins are in the log."""
import math
import re
import numpy as np
import pytest
import torch
import capital_b200 as cb
from capital_b200 import _lib
import batched_reference as br
from scqr3_reference import ill_conditioned

pytestmark = pytest.mark.gpu
LD = np.longdouble


@pytest.fixture(scope="module")
def sq():
    return cb.topo.square(1, 0, 1)


@pytest.fixture(scope="module")
def rect():
    return cb.topo.rect(1, 0, 1)


def _same(x, y):
    return x.shape == y.shape and torch.equal(x.contiguous().view(torch.int64), y.contiguous().view(torch.int64))


def _report(group, **ratios):
    print(f"\n[batched-ref] {group}: " + " ".join(f"{k}={v:.2e}" for k, v in ratios.items()))


def _lower_is_plus_zero(T):
    n = T.shape[-1]
    lower = torch.ones(n, n, dtype=torch.bool, device=T.device).tril(-1)
    return not T[..., lower].any() and not torch.signbit(T[..., lower]).any()


def _num_sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


# ---- single-matrix paths ------------------------------------------------------------------------------------------------------------
def _single_chol(topo, a):
    """R, Rinv of cholinv.factor on one matrix (a base case covering n: the leaf or the width-8 cluster kernel)"""
    n = a.shape[0]
    M = cb.matrix(n, n, 1, 1, data=a.contiguous().reshape(-1).clone())
    args = cb.cholinv.info(1, 1, 0, "U", serialize=False)
    cb.cholinv.factor(M, args, topo)
    return args.R.view(n, n).t(), args.Rinv.view(n, n).t()


def _single_pivot(topo, a):
    """the pivot of the single path's NOT_SPD message"""
    with pytest.raises(_lib.CapitalError, match="non-positive pivot") as e:
        _single_chol(topo, a)
    return int(re.search(r"non-positive pivot (\d+)", str(e.value)).group(1))


def _single_qr(topo, a, num_iter):
    m, n = a.shape
    M = cb.matrix(n, m, 1, 1, data=a.mT.contiguous().reshape(-1).clone())
    args = cb.cacqr.info(num_iter, cb.cholinv.info(0, 1, 0, "U"), serialize=False)
    cb.cacqr.factor(M, args, topo)
    return cb.cacqr.construct_Q(args), cb.cacqr.construct_R(args)


def _colmajor(a):
    """(b, m, n) with A[b] column-major, as factor_batched reads it without a copy"""
    return a.mT.contiguous().mT


# ---- cached references ---------------------------------------------------------------------------------------------------------------
_CHOL = {}


def _chol_ref(key, a):
    if key not in _CHOL:
        _CHOL[key] = br.chol_ld(a)[:2]
    return _CHOL[key]


def _fro(x):
    return float(np.linalg.norm(np.asarray(x, dtype=np.float64)))


# ==== cholinv.factor_batched against chol_ld ==========================================================================================
@pytest.mark.parametrize("n", br.FACTOR_N)
def test_factor_against_long_double(sq, n):
    inputs = br.factor_inputs(n)
    A = torch.stack([a for _, a, _ in inputs]).cuda()
    R, Ri, info = cb.cholinv.factor_batched(A, sq)
    assert info.tolist() == [0] * len(inputs)
    assert _lower_is_plus_zero(R) and _lower_is_plus_zero(Ri)
    worst = {"chol": 0.0, "inv": 0.0, "fwdR": 0.0, "fwdRinv": 0.0}
    for b, (name, a, grading) in enumerate(inputs):
        # position independence: the same bits in a batch of one
        r1, ri1, inf1 = cb.cholinv.factor_batched(A[b:b + 1], sq)
        assert int(inf1[0]) == 0 and _same(r1[0], R[b]) and _same(ri1[0], Ri[b]), name
        ac = A[b]
        c, i = br.chol_ratio(ac, R[b]), br.inv_ratio(R[b], Ri[b])
        assert c <= 1.0 and i <= 1.0, (name, c, i)
        r, ri = R[b].cpu().numpy(), Ri[b].cpu().numpy()
        if grading is None:
            ref = a.numpy()
        else:
            # R(D A D) = R(A) D and Rinv(D A D) = D^-1 Rinv(A); the componentwise backward error that Bounds starts from is
            # invariant under this grading, so the ungraded factors are gated with the ungraded matrix's bounds
            ref, d = grading[0].numpy(), np.ldexp(1.0, grading[1].numpy())
            r, ri = r / d[None, :], ri * d[:, None]
        r_ld, ri_ld = _chol_ref(("chol", n, name), ref)
        bd = br.Bounds(ref)
        fr = _fro(np.asarray(r, dtype=LD) - r_ld) / bd.forward_r
        fi = _fro(np.asarray(ri, dtype=LD) - ri_ld) / bd.forward_rinv
        assert fr <= 1.0 and fi <= 1.0, (name, fr, fi)
        for k, v in (("chol", c), ("inv", i), ("fwdR", fr), ("fwdRinv", fi)):
            worst[k] = max(worst[k], v)
    _report(f"factor n={n}", **worst)


# ==== cluster widths ==================================================================================================================
SCALES = [-412, -270, 270, 412]  # test_gpu_conditioning.SCALES beyond the two-pivot step's range


def _width_inputs(n):
    base = br.spd_spectrum(n, 10.0, 7 * n)
    out = [br.graded(base, br.ramp_exponents(n, 300))]
    out += [br.scaled(base, k) for k in SCALES]
    return torch.stack(out).cuda()


@pytest.mark.parametrize("n", [128, 192, 256, 512])
def test_cluster_widths_match_the_single_factor(sq, n, monkeypatch):
    """width 2 (n = 128), 4 (192, 256) and 8 (512) against the single factor's width 8, on graded and 4^k-scaled inputs"""
    A = _width_inputs(n)
    R, Ri, info = cb.cholinv.factor_batched(A, sq)
    assert info.tolist() == [0] * A.shape[0]
    for b in range(A.shape[0]):
        r1, ri1 = _single_chol(sq, A[b])
        assert _same(R[b], r1) and _same(Ri[b], ri1), b
    monkeypatch.setenv("CAPITAL_BATCHED_CW", "8")
    R8, Ri8, info8 = cb.cholinv.factor_batched(A, sq)
    assert _same(R8, R) and _same(Ri8, Ri) and torch.equal(info8, info)


@pytest.mark.parametrize("n", [100, 129, 200, 255])
def test_cluster_widths_agree_at_padded_n(sq, n, monkeypatch):
    A = _width_inputs(n)
    R, Ri, info = cb.cholinv.factor_batched(A, sq)
    assert info.tolist() == [0] * A.shape[0]
    monkeypatch.setenv("CAPITAL_BATCHED_CW", "8")
    R8, Ri8, info8 = cb.cholinv.factor_batched(A, sq)
    assert _same(R8, R) and _same(Ri8, Ri) and torch.equal(info8, info)


@pytest.mark.parametrize("n", [100, 200])
@pytest.mark.parametrize("num_iter", [1, 2, 3])
def test_qr_cluster_widths_agree(rect, n, num_iter, monkeypatch):
    """the batched QR's base case at its default width (2 at n = 100, 4 at 200) and at width 8: graded columns and 2^k scales"""
    m = 1000
    g = torch.Generator().manual_seed(n + num_iter)
    a = torch.randn(m, n, dtype=torch.float64, generator=g)
    d = torch.from_numpy(np.ldexp(1.0, br.ramp_exponents(n, 100).numpy()))
    mats = [a * d[None, :]] + [a * math.ldexp(1.0, k) for k in (-300, 300)]
    A = _colmajor(torch.stack(mats).cuda())
    Q, R, info = cb.cacqr.factor_batched(A, rect, num_iter)
    monkeypatch.setenv("CAPITAL_BATCHED_CW", "8")
    Q8, R8, info8 = cb.cacqr.factor_batched(A, rect, num_iter)
    assert torch.equal(info8, info)
    assert _same(Q8, Q) and _same(R8, R)


# ==== failures ========================================================================================================================
def _failure_cases(n):
    """(name, torch-indexed A) of each failing matrix; factor_batched reads A[b]'s lower triangle in torch indexing, the library's
    upper triangle of the column-major A[b]^T"""
    base = br.spd_spectrum(n, 10.0, 11 * n)
    out = []
    for k in (0, n // 2, n - 1):
        a = base.clone(); a[k, k] = -1.0; out.append((f"negative pivot {k}", a))
    k = n // 3
    a = base.clone(); a[k, k] = float("nan"); out.append((f"NaN diagonal {k}", a))
    i, j = n // 4, (2 * n) // 3  # library (i, j), i < j: torch [j, i]
    a = base.clone(); a[j, i] = float("nan"); out.append((f"NaN upper ({i},{j})", a))
    return base, out


@pytest.mark.parametrize("n", [17, 63, 100, 128, 511])
def test_failures_in_lapack_numbering(sq, n):
    base, cases = _failure_cases(n)
    mats = [base] + [a for _, a in cases] + [base * 2.0]
    A = torch.stack(mats).cuda()
    clean = torch.stack([base] * (len(cases) + 1) + [base * 2.0]).cuda()
    R0, Ri0, info0 = cb.cholinv.factor_batched(clean, sq)
    assert int(info0.abs().sum()) == 0
    R, Ri, info = cb.cholinv.factor_batched(A, sq)
    info = info.tolist()
    lines = []
    for b, (name, a) in enumerate(cases, start=1):
        lapack = br.first_bad_pivot(a.numpy().T)
        single = _single_pivot(sq, a.cuda())
        lines.append(f"{name}: batched {info[b]} single {single} lapack {lapack}")
        # at n = 100 and 511 the single path's recursion splits n into several base-case blocks: its pivot is still the column of
        # the whole matrix
        assert info[b] == single == lapack, lines[-1]
    print(f"\n[batched-ref] failures n={n}: " + " | ".join(lines))
    for b in (0, len(mats) - 1):
        assert info[b] == 0 and _same(R[b], R0[b]) and _same(Ri[b], Ri0[b]), b


# ==== chunk edges =====================================================================================================================
def _launches(ctx, fn):
    ctx.reset_counters()
    fn()
    return ctx.counters().kernel_launches


def _diag_dominant(batch, n, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    A = torch.randn(batch, n, n, dtype=torch.float64, device="cuda", generator=g) * 0.1 / n ** 0.5
    return A + A.mT + torch.eye(n, dtype=torch.float64, device="cuda")


@pytest.mark.parametrize("n", [512, 511])
def test_factor_chunk_edges(sq, n):
    """n = 512 runs in place (W and Rinv^T per matrix: 512 per chunk), n = 511 through padded copies (256 per chunk)"""
    chunk = br.factor_chunk(n, 1 << 30)
    assert chunk == (512 if n == 512 else 256)
    ctx = sq.context()
    A = _diag_dominant(2 * chunk + 1, n, n)
    one = _launches(ctx, lambda: cb.cholinv.factor_batched(A[:1], sq))
    assert _launches(ctx, lambda: cb.cholinv.factor_batched(A[:chunk], sq)) == one
    assert _launches(ctx, lambda: cb.cholinv.factor_batched(A[:chunk + 1], sq)) == 2 * one
    batch = A.shape[0]
    R0, Ri0, info0 = cb.cholinv.factor_batched(A, sq)
    assert int(info0.abs().sum()) == 0
    bad = {0: 0, chunk - 1: n // 2, chunk: n - 1, batch - 1: 5}  # matrix -> 0-based failing pivot
    Ab = A.clone()
    for b, k in bad.items():
        Ab[b, k, k] = -1.0
    R, Ri, info = cb.cholinv.factor_batched(Ab, sq)
    expect = torch.zeros(batch, dtype=torch.int32)
    for b, k in bad.items():
        expect[b] = k + 1
    assert torch.equal(info.cpu(), expect), [(b, int(info[b])) for b in torch.nonzero(info.cpu() != expect).flatten().tolist()[:8]]
    keep = torch.ones(batch, dtype=torch.bool)
    keep[list(bad)] = False
    keep = keep.cuda()
    assert _same(R[keep], R0[keep]) and _same(Ri[keep], Ri0[keep])
    for b in (1, chunk - 2, chunk + 1, batch - 2):
        r1, ri1, i1 = cb.cholinv.factor_batched(A[b:b + 1], sq)
        assert _same(r1[0], R[b]) and _same(ri1[0], Ri[b]) and int(i1[0]) == 0, b
    del A, Ab, R, Ri, R0, Ri0
    torch.cuda.empty_cache()


def test_qr_chunk_edges(rect):
    """m = 65536, n = 64: about 20 matrices per chunk; zero columns at both sides of the chunk edges"""
    m, n, it = 65536, 64, 2
    chunk = br.qr_chunk(m, n, 1 << 30, it, _num_sms())
    assert 2 <= chunk <= 64
    batch = 2 * chunk + 1
    g = torch.Generator(device="cuda").manual_seed(17)
    A = torch.randn(batch, n, m, dtype=torch.float64, device="cuda", generator=g).mT
    ctx = rect.context()
    one = _launches(ctx, lambda: cb.cacqr.factor_batched(A[:1], rect, it))
    assert _launches(ctx, lambda: cb.cacqr.factor_batched(A[:chunk], rect, it)) == one
    assert _launches(ctx, lambda: cb.cacqr.factor_batched(A[:chunk + 1], rect, it)) == 2 * one
    Q0, R0, info0 = cb.cacqr.factor_batched(A, rect, it)
    assert int(info0.abs().sum()) == 0
    bad = {0: 3, chunk - 1: n // 2, chunk: n - 1, batch - 1: 0}  # matrix -> zero column: the first Gram pivot at it is exactly 0
    Ab = A.mT.contiguous().mT
    for b, j in bad.items():
        Ab[b, :, j] = 0.0
    Q, R, info = cb.cacqr.factor_batched(Ab, rect, it)
    expect = torch.zeros(batch, dtype=torch.int32)
    for b, j in bad.items():
        expect[b] = j + 1
    assert torch.equal(info.cpu(), expect), info.tolist()
    keep = torch.ones(batch, dtype=torch.bool)
    keep[list(bad)] = False
    keep = keep.cuda()
    assert _same(Q[keep], Q0[keep]) and _same(R[keep], R0[keep])
    for b in (1, chunk - 2, chunk + 1, batch - 2):
        q1, r1, i1 = cb.cacqr.factor_batched(A[b:b + 1], rect, it)
        assert _same(q1[0], Q[b]) and _same(r1[0], R[b]) and int(i1[0]) == 0, b
    del A, Ab, Q, R, Q0, R0
    torch.cuda.empty_cache()


# ==== cacqr.factor_batched against qr_ld =============================================================================================
_QR = {}


def _qr_case(m, n, kappa):
    key = (m, n, kappa)
    if key not in _QR:
        a = br.qr_matrix(m, n, kappa)
        _, r = br.qr_ld(a, want_q=False)
        sv = np.linalg.svd(a, compute_uv=False)
        _QR[key] = (a, r, float(sv[0]), float(sv[0] / sv[-1]))
    return _QR[key]


@pytest.mark.parametrize("m,n", br.qr_shapes())
def test_qr_against_long_double(rect, m, n):
    worst = {}
    for it, kappas in br.QR_RUNS.items():
        cases = [_qr_case(m, n, k) for k in kappas]
        A = _colmajor(torch.from_numpy(np.stack([c[0] for c in cases])).cuda())
        Q, R, info = cb.cacqr.factor_batched(A, rect, it)
        assert info.tolist() == [0] * len(cases), (it, info.tolist())
        assert _lower_is_plus_zero(R) and bool((torch.diagonal(R, dim1=1, dim2=2) > 0).all())
        for b, (a, r_ld, norm2, kappa) in enumerate(cases):
            bd = br.QRBounds(m, n, it, kappa, norm2)
            o, s, f = bd.check(a, Q[b].cpu().numpy(), R[b].cpu().numpy(), r_ld)
            assert o <= 1 and s <= 1 and f <= 1, (it, kappa, o, s, f)
            for k, v in ((f"orth{it}", o), (f"res{it}", s), (f"fwdR{it}", f)):
                worst[k] = max(worst.get(k, 0.0), v)
            if n <= 64 and n % 2 == 1:
                q1, r1 = _single_qr(rect, A[b], it)
                assert _same(Q[b], q1) and _same(R[b], r1), (it, kappa)
    _report(f"qr m={m} n={n}", **worst)


# ==== mixed scales in one batch =======================================================================================================
@pytest.mark.parametrize("m,n", [(512, 32), (1000, 100), (777, 256)])
@pytest.mark.parametrize("num_iter", [1, 2, 3])
def test_qr_mixed_scales(rect, m, n, num_iter):
    """2^k A_b, k in {-300, 0, 300}, in one call: the Gram matrices stay in range, so Q_b and 2^-k R_b match the unscaled factors,
    and each matrix gets the bits it gets alone (a shift or norm taken from another matrix of the batch would change them)"""
    ks = (-300, 0, 300)
    base = [ill_conditioned(m, n, 100.0, 5 * n + s) for s in range(3)]
    A0 = _colmajor(torch.from_numpy(np.stack(base)).cuda())
    A = _colmajor(torch.from_numpy(np.stack([np.ldexp(a, k) for a, k in zip(base, ks)])).cuda())
    Q0, R0, info0 = cb.cacqr.factor_batched(A0, rect, num_iter)
    Q, R, info = cb.cacqr.factor_batched(A, rect, num_iter)
    assert info0.tolist() == [0, 0, 0] and info.tolist() == [0, 0, 0]
    worst = 0.0
    for b, k in enumerate(ks):
        eq = float((Q[b] - Q0[b]).abs().max() / Q0[b].abs().max())
        er = float((R[b] * math.ldexp(1.0, -k) - R0[b]).abs().max() / R0[b].abs().max())
        worst = max(worst, eq, er)
        assert eq <= 1e-14 and er <= 1e-14, (k, eq, er)
        q1, r1, i1 = cb.cacqr.factor_batched(A[b:b + 1], rect, num_iter)
        assert int(i1[0]) == 0 and _same(q1[0], Q[b]) and _same(r1[0], R[b]), k
    _report(f"mixed scales m={m} n={n} it={num_iter}", rel=worst)


# ==== solve_batched against solve_ld ==================================================================================================
def _rel(x, ref):
    return _fro(np.asarray(x, dtype=LD) - ref) / _fro(ref)


@pytest.mark.parametrize("n", br.SOLVE_N)
def test_solve_against_long_double(sq, n):
    """X against Rinv (Rinv^T B) in long double with the same Rinv (solve_product_bound, linear in kappa: 5e-4 of ||X|| at n = 512,
    kappa = 1e8), and against A^-1 B from solve_ld where the end-to-end bound solve_bound is below 1 (kappa = 10)"""
    mats = br.solve_inputs(n)
    A = torch.stack(mats).cuda()
    R, Ri, info = cb.cholinv.factor_batched(A, sq)
    assert info.tolist() == [0, 0]
    g = torch.Generator().manual_seed(n)
    B = torch.randn(2, n, max(br.SOLVE_K), dtype=torch.float64, generator=g)
    rinv = [Ri[b].cpu().numpy() for b in range(2)]
    P_ld = [br.solve_product_ld(rinv[b], B[b].numpy()) for b in range(2)]
    X_ld = [br.solve_ld(mats[b].numpy(), B[b].numpy()) for b in range(2)]
    e2e = [br.solve_bound(mats[b].numpy()) for b in range(2)]
    assert e2e[0] < 1  # kappa = 10
    Bc = B.cuda()
    worst = {"op": 0.0, "fwd": 0.0, "fwd_1e8": 0.0}
    for k in br.SOLVE_K:
        X = cb.cholinv.solve_batched(Ri, Bc[:, :, :k], sq)
        for b in range(2):
            x = X[b].cpu().numpy()
            op = _fro(np.asarray(x, dtype=LD) - P_ld[b][:, :k]) / br.solve_product_bound(rinv[b], B[b, :, :k].numpy())
            worst["op"] = max(worst["op"], op)
            assert op <= 1.0, (k, b, op)
            fwd = _rel(x, X_ld[b][:, :k])
            if e2e[b] < 1:
                worst["fwd"] = max(worst["fwd"], fwd / e2e[b])
                assert fwd <= e2e[b], (k, b, fwd, e2e[b])
            else:  # kappa = 1e8: the end-to-end error is reported, the operation is gated above
                worst["fwd_1e8"] = max(worst["fwd_1e8"], fwd)
        if k == 65:  # in place through the C entry point: three panels of B overwritten by X
            XB = Bc[:, :, :k].mT.contiguous()
            ctx = sq.context()
            ctx.check(_lib.lib().capital_cholinv_solve_batched_f64(ctx.handle, n, 2, Ri.mT.contiguous().data_ptr(), k, XB.data_ptr(),
                                                                   XB.data_ptr()))
            assert _same(XB.mT, X)
    print(f"\n[batched-ref] solve n={n}: op={worst['op']:.2e} fwd={worst['fwd']:.2e} (ratios to the bounds); "
          f"kappa=1e8 relative error {worst['fwd_1e8']:.2e}")


def test_solve_two_chunks(sq):
    """70 000 matrices at n = 8: 65 535 + 4 465; the tail matches a separate call and its own references"""
    n, batch = 8, 70000
    chunk = br.solve_chunk(n, batch)
    assert chunk == 65535
    A = _diag_dominant(batch, n, 5)
    R, Ri, info = cb.cholinv.factor_batched(A, sq)
    assert int(info.abs().sum()) == 0
    g = torch.Generator(device="cuda").manual_seed(6)
    B = torch.randn(batch, n, 3, dtype=torch.float64, device="cuda", generator=g)
    X = cb.cholinv.solve_batched(Ri, B, sq)
    Xt = cb.cholinv.solve_batched(Ri[chunk - 5:], B[chunk - 5:], sq)
    assert _same(Xt, X[chunk - 5:])
    worst = {"op": 0.0, "fwd": 0.0}
    for b in list(range(chunk - 3, chunk + 3)) + [batch - 1]:
        a, rhs, x, rinv = A[b].cpu().numpy(), B[b].cpu().numpy(), X[b].cpu().numpy(), Ri[b].cpu().numpy()
        op = _fro(np.asarray(x, dtype=LD) - br.solve_product_ld(rinv, rhs)) / br.solve_product_bound(rinv, rhs)
        fwd = _rel(x, br.solve_ld(a, rhs)) / br.solve_bound(a)
        worst = {"op": max(worst["op"], op), "fwd": max(worst["fwd"], fwd)}
        assert op <= 1.0 and fwd <= 1.0, (b, op, fwd)
    _report("solve 70000 x n=8", **worst)
    del A, R, Ri, B, X
    torch.cuda.empty_cache()


# ==== lstsq_batched against lstsq_ld ==================================================================================================
def _lstsq_op(q, r, b, x):
    """ratio of ||X - R^-1 Q^T B|| (long double, the same factors) to lstsq_product_bound"""
    ref = br.lstsq_product_ld(q, r, b)
    return _fro(np.asarray(x, dtype=LD) - ref) / br.lstsq_product_bound(q, r, b, ref)


@pytest.mark.parametrize("m,n,kappa,num_iter", br.LS_CASES)
@pytest.mark.parametrize("rho", br.LS_RHO)
def test_lstsq_against_long_double(rect, m, n, kappa, num_iter, rho):
    """X against R^-1 (Q^T B) in long double with the same Q and R (lstsq_product_bound, linear in kappa), and against the
    least-squares solution from lstsq_ld where Higham's bound (ls_bound) is below 1 (kappa = 10 and 1e5)"""
    rho = br.ls_rho(kappa, rho)  # inconsistent at kappa = 1e10: ||r|| small enough that kappa^2 ||r|| stays bounded
    k = br.LS_K
    probs = [br.ls_problem(m, n, kappa, rho, k, 7 * m + n + s) for s in range(2)]
    A = _colmajor(torch.from_numpy(np.stack([p[0] for p in probs])).cuda())
    Q, R, info = cb.cacqr.factor_batched(A, rect, num_iter)
    assert info.tolist() == [0, 0]
    B = torch.from_numpy(np.stack([p[1] for p in probs])).cuda()
    X = cb.cacqr.lstsq_batched(Q, R, B, rect)
    worst = {"op": 0.0, "fwd": 0.0, "fwd_rel": 0.0}
    for b, (a, rhs, xl, res) in enumerate(probs):
        x = X[b].cpu().numpy()
        op = _lstsq_op(Q[b].cpu().numpy(), R[b].cpu().numpy(), rhs, x)
        assert op <= 1.0, (b, op)
        bound = br.ls_bound(a, xl, res, num_iter)
        fwd = _rel(x, xl)
        worst = {"op": max(worst["op"], op), "fwd": max(worst["fwd"], fwd / bound), "fwd_rel": max(worst["fwd_rel"], fwd)}
        if kappa < 1e9:
            assert bound < 1 and fwd <= bound, (b, fwd, bound)
    _report(f"lstsq m={m} n={n} kappa={kappa:.0e} rho={rho:.0e}", **worst)


def test_lstsq_long_k_range(rect):
    """m = 2^17 + 1: Q^T B runs over 129 k chunks of 1024 rows, the last one ragged; batch 4, two panels.  The long-double
    reference of the operation is evaluated on one column of each panel (m n flops per column)"""
    m, n, k = 2 ** 17 + 1, 64, 33
    rng = np.random.default_rng(3)
    A = _colmajor(torch.from_numpy(rng.standard_normal((4, m, n))).cuda())
    Q, R, info = cb.cacqr.factor_batched(A, rect, 2)
    assert info.tolist() == [0] * 4
    B = torch.from_numpy(rng.standard_normal((4, m, k))).cuda()
    X = cb.cacqr.lstsq_batched(Q, R, B, rect)
    X3 = cb.cacqr.lstsq_batched(Q[3:], R[3:], B[3:], rect)
    assert _same(X3[0], X[3])
    worst = 0.0
    cols = [0, k - 1]
    for b in range(4):
        e = _lstsq_op(Q[b].cpu().numpy(), R[b].cpu().numpy(), B[b, :, cols].cpu().numpy(), X[b, :, cols].cpu().numpy())
        worst = max(worst, e)
        assert e <= 1.0, (b, e)
    _report("lstsq m=2^17+1 n=64", op=worst)
    del A, Q, R, B, X
    torch.cuda.empty_cache()


def test_lstsq_two_chunks(rect):
    """70 000 matrices at m = 16, n = 8: 65 535 + 4 465 for the factor and for lstsq"""
    m, n, batch = 16, 8, 70000
    assert br.lstsq_chunk(m, n, batch) == 65535 and br.qr_chunk(m, n, batch, 2, _num_sms()) == 65535
    g = torch.Generator(device="cuda").manual_seed(21)
    A = torch.randn(batch, n, m, dtype=torch.float64, device="cuda", generator=g).mT
    Q, R, info = cb.cacqr.factor_batched(A, rect)
    assert int(info.abs().sum()) == 0
    B = torch.randn(batch, m, 2, dtype=torch.float64, device="cuda", generator=g)
    X = cb.cacqr.lstsq_batched(Q, R, B, rect)
    t0 = 65535 - 5
    Xt = cb.cacqr.lstsq_batched(Q[t0:], R[t0:], B[t0:], rect)
    assert _same(Xt, X[t0:])
    worst = {"op": 0.0, "fwd": 0.0}
    for b in list(range(65535 - 3, 65535 + 3)) + [batch - 1]:
        a, rhs, x = A[b].cpu().numpy(), B[b].cpu().numpy(), X[b].cpu().numpy()
        op = _lstsq_op(Q[b].cpu().numpy(), R[b].cpu().numpy(), rhs, x)
        xl, res = br.lstsq_ld(a, rhs)
        fwd = _rel(x, xl) / br.ls_bound(a, xl, res, 2)
        worst = {"op": max(worst["op"], op), "fwd": max(worst["fwd"], fwd)}
        assert op <= 1.0 and fwd <= 1.0, (b, op, fwd)
    _report("lstsq 70000 x 16x8", **worst)
    del A, Q, R, B, X
    torch.cuda.empty_cache()
