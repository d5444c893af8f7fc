"""CPU side of the batched reference tests (no GPU): the long-double references agree with scipy and with their own residuals, LAPACK's
float64 factors, solutions and least-squares solutions stay well below every a-priori bound of batched_reference at every shape and
condition number of tests/test_gpu_batched_reference.py, each bound catches a planted error, and the restated chunk rules give the
chunk sizes the GPU tests place matrices around."""
import math
import numpy as np
import pytest
import scipy.linalg as sla
import batched_reference as br

U = br.U
ULD = float(np.finfo(np.longdouble).eps) / 2
HEADROOM = 0.1  # LAPACK's ratio to each bound stays at or below this


def _headroom(n):
    """at n <= 2 the QR residual bound is a handful of ulps, and one rounding of LAPACK's is a sizeable part of it"""
    return 0.5 if n <= 2 else HEADROOM


def _fro(x):
    return float(np.linalg.norm(np.asarray(x, dtype=np.float64)))


def _lapack_qr(a):
    q, r = sla.qr(a, mode="economic")
    s = np.sign(np.diag(r))
    s[s == 0] = 1
    return q * s[None, :], r * s[:, None]


# ---- the references ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("m,n,kappa", [(50, 17, 10.0), (33, 33, 1e5), (200, 64, 1e10), (7, 1, 1.0)])
def test_qr_ld_against_scipy_and_itself(m, n, kappa):
    a = br.qr_matrix(m, n, kappa)
    q, r = br.qr_ld(a)
    assert (np.diag(r) > 0).all() and not np.tril(r, -1).any()
    _, rs = _lapack_qr(a)
    assert _fro(r - rs) / _fro(r) <= 10 * n * U * kappa
    al = np.asarray(a, dtype=np.longdouble)
    assert _fro(al - q @ r) / _fro(a) <= 10 * n * ULD
    assert _fro(q.T @ q - np.eye(n)) <= 10 * n * ULD * kappa  # Q = A R^-1 by substitution: kappa u_ld
    _, r2 = br.qr_ld(a, want_q=False)
    assert np.array_equal(r2, r)


@pytest.mark.parametrize("kappa,rho", [(10.0, 0.0), (10.0, 1e-2), (1e6, 1e-3)])
def test_lstsq_ld_against_scipy_and_itself(kappa, rho):
    m, n, k = 120, 20, 3
    a, b, x, res = br.ls_problem(m, n, kappa, rho, k, 4)
    xs = sla.lstsq(a, b)[0]
    assert _fro(x - xs) / _fro(x) <= 100 * n * U * (kappa + kappa ** 2 * rho)
    al, bl = np.asarray(a, dtype=np.longdouble), np.asarray(b, dtype=np.longdouble)
    r = bl - al @ x
    assert np.allclose(np.sqrt((r ** 2).sum(axis=0)).astype(float), res.astype(float), rtol=1e-9, atol=1e-15)
    np.testing.assert_allclose(res.astype(float), rho * np.linalg.norm(np.asarray(x, dtype=float), axis=0), rtol=1e-6, atol=1e-14)
    assert _fro(al.T @ r) <= 100 * m * ULD * _fro(b) * kappa  # normal equations in long double
    x1, _ = br.lstsq_ld(a, b[:, 0])
    assert x1.shape == (n,) and _fro(x1 - x[:, 0]) <= 10 * ULD * kappa * _fro(x)


@pytest.mark.parametrize("n,kappa", [(1, 1.0), (17, 10.0), (65, 1e8)])
def test_solve_ld_against_scipy_and_itself(n, kappa):
    a = br.spd_spectrum(n, kappa, 5).numpy()
    b = np.random.default_rng(1).standard_normal((n, 4))
    x = br.solve_ld(a, b)
    xs = sla.cho_solve(sla.cho_factor(a), b)
    assert _fro(x - xs) / _fro(x) <= 10 * n * U * kappa
    assert _fro(np.asarray(a, dtype=np.longdouble) @ x - b) <= 10 * n * ULD * _fro(a) * _fro(x)


def test_first_bad_pivot_is_lapacks_numbering():
    n = 40
    base = br.spd_spectrum(n, 10.0, 2).numpy()
    assert br.first_bad_pivot(base) == 0
    for k in (0, 7, n // 2, n - 1):
        a = base.copy(); a[k, k] = -1.0
        _, info = sla.lapack.dpotrf(a, lower=0)
        assert br.first_bad_pivot(a) == info == k + 1
    a = base.copy(); a[11, 11] = np.nan
    assert br.first_bad_pivot(a) == 12
    a = base.copy(); a[5, 30] = np.nan  # above the diagonal: pivot 30 is the first that is NaN
    assert br.first_bad_pivot(a) == 31
    a = base.copy(); a[30, 5] = np.nan  # below the diagonal: not read
    assert br.first_bad_pivot(a) == 0


# ---- LAPACK below the bounds at every case of the GPU tables ----------------------------------------------------------------------
@pytest.mark.parametrize("n", br.FACTOR_N)
def test_factor_bounds_have_headroom(n):
    worst = 0.0
    for name, a, grading in br.factor_inputs(n):
        ref = (a if grading is None else grading[0]).numpy()
        r_ld, ri_ld = br.chol_ld(ref)[:2]
        rs = sla.cholesky(ref, lower=False)
        xs = np.triu(sla.lapack.dtrtri(rs)[0])
        bd = br.Bounds(ref)
        fr = _fro(np.asarray(rs, dtype=np.longdouble) - r_ld) / bd.forward_r
        fi = _fro(np.asarray(xs, dtype=np.longdouble) - ri_ld) / bd.forward_rinv
        worst = max(worst, fr, fi)
        assert fr <= HEADROOM and fi <= HEADROOM, (name, fr, fi)
    print(f"\n[bounds] factor n={n}: LAPACK worst {worst:.2e}")


@pytest.mark.parametrize("m,n", br.qr_shapes())
def test_qr_bounds_have_headroom(m, n):
    worst = {}
    for kappa in sorted({k for ks in br.QR_RUNS.values() for k in ks}):
        a = br.qr_matrix(m, n, kappa)
        _, r_ld = br.qr_ld(a, want_q=False)
        sv = np.linalg.svd(a, compute_uv=False)
        q, r = _lapack_qr(a)
        for it, ks in br.QR_RUNS.items():
            if kappa not in ks:
                continue
            ratios = br.QRBounds(m, n, it, float(sv[0] / sv[-1]), float(sv[0])).check(a, q, r, r_ld)
            for name, v in zip(("orth", "res", "fwdR"), ratios):
                worst[f"{name}{it}"] = max(worst.get(f"{name}{it}", 0.0), v)
            assert max(ratios) <= _headroom(n), (it, kappa, ratios)
    print(f"\n[bounds] qr m={m} n={n}: " + " ".join(f"{k}={v:.1e}" for k, v in worst.items()))


@pytest.mark.parametrize("n", br.SOLVE_N)
def test_solve_bounds_have_headroom(n):
    """LAPACK's inverse (dtrtri of dpotrf's R) applied as Rinv (Rinv^T B) in float64: its product error is well inside
    solve_product_bound at every row, and the end-to-end error inside solve_bound wherever that is below 1 (kappa = 10)"""
    for kappa, a in zip(br.SOLVE_KAPPAS, br.solve_inputs(n)):
        a = a.numpy()
        b = np.random.default_rng(n).standard_normal((n, max(br.SOLVE_K)))
        rinv = np.triu(sla.lapack.dtrtri(sla.cholesky(a, lower=False))[0])
        x = rinv @ (rinv.T @ b)
        op = _fro(np.asarray(x, dtype=np.longdouble) - br.solve_product_ld(rinv, b)) / br.solve_product_bound(rinv, b)
        assert op <= HEADROOM, (kappa, op)
        assert br.solve_product_bound(rinv, b) / _fro(x) < 1e-3  # kappa-linear: meaningful at kappa = 1e8 too
        if kappa < 1e3:
            xs = sla.cho_solve(sla.cho_factor(a), b)
            e = _fro(np.asarray(xs, dtype=np.longdouble) - br.solve_ld(a, b)) / _fro(br.solve_ld(a, b))
            assert br.solve_bound(a) < 1 and e <= HEADROOM * br.solve_bound(a), e


@pytest.mark.parametrize("m,n,kappa,num_iter", br.LS_CASES)
@pytest.mark.parametrize("rho", br.LS_RHO)
def test_lstsq_bounds_have_headroom(m, n, kappa, num_iter, rho):
    """R^-1 (Q^T B) from LAPACK's Q and R in float64 stays well inside lstsq_product_bound at every row; LAPACK's lstsq inside
    Higham's bound (ls_bound) where that is below 1 (kappa = 10 and 1e5; at kappa = 1e10 only the operation is gated)"""
    a, b, x, res = br.ls_problem(m, n, kappa, br.ls_rho(kappa, rho), br.LS_K, 1)
    q, r = _lapack_qr(a)
    y = sla.solve_triangular(r, q.T @ b)
    ref = br.lstsq_product_ld(q, r, b)
    pb = br.lstsq_product_bound(q, r, b, ref)
    op = _fro(np.asarray(y, dtype=np.longdouble) - ref) / pb
    assert op <= HEADROOM and pb / _fro(ref) < 0.1, (op, pb / _fro(ref))
    bound = br.ls_bound(a, x, res, num_iter)
    xs = sla.lstsq(a, b)[0]
    e = _fro(np.asarray(xs, dtype=np.longdouble) - x) / _fro(x) / bound
    print(f"\n[bounds] lstsq m={m} n={n} kappa={kappa:.0e} rho={rho:.0e}: operation {op:.2e}; LAPACK {e:.2e} of ls_bound ({bound:.1e})")
    if kappa < 1e9:
        assert bound < 1 and e <= HEADROOM


# ---- each bound catches a planted error ---------------------------------------------------------------------------------------
PLANT_ULPS = 400


def _bump(x, i, j):
    """x with entry (i, j) moved by PLANT_ULPS ulps of row i's norm (i = None: the row of largest norm)"""
    y = x.copy()
    if i is None:
        i = int(np.argmax(np.linalg.norm(x, axis=1)))
    y[i, j] += PLANT_ULPS * 2 * U * np.linalg.norm(x[i])
    return y


def test_qr_bounds_catch_planted_errors():
    m, n = 3, 2
    a = br.qr_matrix(m, n, 3.0)
    _, r_ld = br.qr_ld(a, want_q=False)
    sv = np.linalg.svd(a, compute_uv=False)
    bd = br.QRBounds(m, n, 2, float(sv[0] / sv[-1]), float(sv[0]))
    q, r = _lapack_qr(a)
    assert max(bd.check(a, q, r, r_ld)) <= HEADROOM
    assert bd.check(a, _bump(q, None, 1), r, r_ld)[0] > 1       # orthogonality
    assert bd.check(a, q[:, ::-1], r, r_ld)[1] > 1           # two columns of Q swapped: residual
    assert bd.check(a, q, _bump(r, 0, 1), r_ld)[2] > 1       # forward error of R
    bd1 = br.QRBounds(m, n, 1, float(sv[0] / sv[-1]), float(sv[0]))
    assert bd1.check(a, _bump(q, None, 0), r, r_ld)[0] > 1      # CholeskyQR's kappa^2 orthogonality bound


def test_solve_and_lstsq_bounds_catch_planted_errors():
    a = br.spd_spectrum(2, 2.0, 3).numpy()
    b = np.random.default_rng(2).standard_normal((2, 3))
    x = br.solve_ld(a, b)
    xs = sla.cho_solve(sla.cho_factor(a), b)
    bound = br.solve_bound(a)
    assert _fro(np.asarray(xs, dtype=np.longdouble) - x) / _fro(x) <= HEADROOM * bound
    assert _fro(np.asarray(_bump(xs, None, 1), dtype=np.longdouble) - x) / _fro(x) > bound
    a, b, x, res = br.ls_problem(2, 1, 1.0, 0.0, 3, 8)  # the bound grows as m n: the smallest shape
    bound = br.ls_bound(a, x, res, 2)
    xs = sla.lstsq(a, b)[0]
    assert _fro(np.asarray(xs, dtype=np.longdouble) - x) / _fro(x) <= HEADROOM * bound
    assert _fro(np.asarray(_bump(xs, None, 1), dtype=np.longdouble) - x) / _fro(x) > bound


def _op_err(v, ref, bound):
    return _fro(np.asarray(v, dtype=np.longdouble) - ref) / bound


def test_operation_bounds_catch_planted_errors_at_the_ill_conditioned_rows():
    """solve at n = 512, kappa = 1e8 and lstsq at m = 300, n = 32, kappa = 1e10: X = 0, -X, and the product with one term of its
    sum left out (the last row of Rinv^T B, the last row of Q^T B) fail the bounds; the right product passes"""
    n = 512
    a = br.solve_inputs(n)[1].numpy()
    b = np.random.default_rng(0).standard_normal((n, 3))
    rinv = np.triu(sla.lapack.dtrtri(sla.cholesky(a, lower=False))[0])
    ref, bound = br.solve_product_ld(rinv, b), br.solve_product_bound(rinv, b)
    t = rinv.T @ b
    x = rinv @ t
    t_bad = t.copy(); t_bad[-1] = rinv[:-1, -1] @ b[:-1]  # the diagonal term of the last row left out
    assert _op_err(x, ref, bound) <= HEADROOM
    for bad in (np.zeros_like(x), -x, rinv @ t_bad):
        assert _op_err(bad, ref, bound) > 1
    m, n = 300, 32
    a, b, _, _ = br.ls_problem(m, n, 1e10, 0.0, 3, 5)
    q, r = _lapack_qr(a)
    ref = br.lstsq_product_ld(q, r, b)
    bound = br.lstsq_product_bound(q, r, b, ref)
    y = sla.solve_triangular(r, q.T @ b)
    y_bad = sla.solve_triangular(r, q[:-1].T @ b[:-1])  # Q^T B without its last k term
    assert _op_err(y, ref, bound) <= HEADROOM
    assert _op_err(np.zeros_like(y), ref, bound) > 1 and _op_err(-y, ref, bound) > 1 and _op_err(y_bad, ref, bound) > 1


# ---- chunk rules ----------------------------------------------------------------------------------------------------------------
def test_chunk_rules():
    assert br.factor_chunk(512, 10 ** 6) == 512 and br.factor_chunk(511, 10 ** 6) == 256
    assert br.factor_chunk(512, 10 ** 6, aligned=False) == 256 and br.factor_chunk(128, 10 ** 6) == 8192
    assert br.factor_chunk(8, 70000) == 70000  # the leaf path is one launch
    assert br.solve_chunk(8, 70000) == 65535 and br.solve_chunk(512, 10 ** 6) == 8192
    assert br.qr_chunk(65536, 64, 10 ** 6, 2, 132) == 20
    assert br.qr_chunk(16, 8, 70000, 2, 132) == 65535
    assert br.lstsq_chunk(16, 8, 70000) == 65535 and br.lstsq_chunk(2 ** 17 + 1, 64, 10 ** 6) == 1016


def test_batched_gram_never_needs_a_second_grid_piece():
    """launch_batched (gemm_tn.cu) cuts grid z = matrices x k chunks into pieces of 65535 / ks matrices.  Under the 2 GiB cap a chunk
    of the batched QR never reaches that: every matrix holds at least ldt m >= 16 m doubles and ks <= ceil(m / 512), so
    chunk ks <= 2^24 / m * (m / 512 + 1) < 65535 for m > 512, and ks = 1 below.  Checked at m = 2^e - 1, 2^e, 2^e + 1 up to 2^24 and
    around 512, at the table's n and their neighbours, every num_iter, for 132 SMs (an H100) and others."""
    ms = sorted({v for e in range(1, 25) for v in (2 ** e - 1, 2 ** e, 2 ** e + 1)} | {511, 512, 513, 514, 1023, 1025})
    for sms in (78, 114, 132, 148):
        for n in sorted({1, 2, 7, 8, 16, 17, 31, 63, 64, 65, 100, 127, 128, 129, 200, 255, 256, 257, 383, 448, 511, 512}):
            for m in ms:
                if m < n:
                    continue
                for it in (1, 2, 3):
                    for in_place in (True, False):
                        z = br.gram_grid_z(m, n, 10 ** 9, it, sms, in_place)
                        assert z <= 65535, (m, n, it, sms, in_place, z)
