"""CPU side of the conditioning tests (no GPU): the bounds of conditioning_reference hold with headroom for LAPACK-based factors of
every input the GPU tests use, scipy factors every one of those inputs, and the scalar restatement of the cluster base case's
two-pivot step fails outside the double range without the fix and is bit-for-bit unchanged by it for blocks of ordinary scale."""
import math
import numpy as np
import pytest
import scipy.linalg as sla
import torch
from oracle import capital_oracle as co
import conditioning_reference as cr

GATE = 1.0      # the gate of both bound ratios in test_gpu_conditioning
HEADROOM = 10.0


def _bc(n):
    return co.bc_dimension(n, 1, 1, -int(np.log2(n // 512)) if n % 512 == 0 else 0)


def _ratios(a: np.ndarray, n1=None):
    """(oracle R ratio, oracle Rinv ratio, scipy R ratio, scipy Rinv ratio)"""
    at = torch.from_numpy(a)
    r, ri = co.cholinv(a, True, 1, _bc(a.shape[0]))
    rs = sla.cholesky(a, lower=False)  # raises when the matrix does not factor
    xs, info = sla.lapack.dtrtri(rs)
    assert info == 0
    R, X, Rs, Xs = (torch.from_numpy(np.ascontiguousarray(v)) for v in (r, ri, rs, np.triu(xs)))
    return cr.chol_ratio(at, R), cr.inv_ratio(R, X, n1), cr.chol_ratio(at, Rs), cr.inv_ratio(Rs, Xs, n1)


# every (n, kappa) of the GPU spectrum tests; n = 4096 at the largest kappa only (the bound evaluation is n^3 on the host)
CASES = [(n, k) for n in (512, 777, 2048) for k in (1e2, 1e7, 1e11)] + [(4096, 1e11)]


@pytest.mark.parametrize("n,kappa", CASES)
def test_bounds_have_headroom_on_lapack_factors(n, kappa):
    a = cr.spd_spectrum(n, kappa, 1234).numpy()
    ratios = _ratios(a)
    print(f"\n[bounds] n={n} kappa={kappa:.0e}: oracle R {ratios[0]:.2e} Rinv {ratios[1]:.2e} | scipy R {ratios[2]:.2e} "
          f"Rinv {ratios[3]:.2e}")
    assert max(ratios) * HEADROOM <= GATE


@pytest.mark.parametrize("n", [512, 777])
def test_bounds_have_headroom_on_graded_and_scaled_inputs(n):
    """the graded inputs of the GPU tests (spd_global and a kappa = 1e7 core, e from -300 to 300) and the extreme uniform scales"""
    e = cr.ramp_exponents(n, 300)
    inputs = {"graded spd_global": cr.graded(torch.from_numpy(co.spd_global(n)), e),
              "graded kappa=1e7": cr.graded(cr.spd_spectrum(n, 1e7, 1234), e),
              "spd_global 4^-412": cr.scaled(torch.from_numpy(co.spd_global(n)), -412),
              "spd_global 4^412": cr.scaled(torch.from_numpy(co.spd_global(n)), 412)}
    for name, a in inputs.items():
        ratios = _ratios(a.numpy())
        print(f"\n[bounds] n={n} {name}: {', '.join(f'{v:.2e}' for v in ratios)}")
        assert max(ratios) * HEADROOM <= GATE, name


def test_graded_profile_crosses_the_double_range():
    """the ramp from -300 to 300 puts neighbouring diagonal products of D A D outside [2^-1022, 2^1024] at both ends"""
    for n in (32, 512, 777, 4096):
        lo, hi = cr.pair_product_log2(torch.from_numpy(co.spd_global(n)), cr.ramp_exponents(n, 300))
        assert lo < -1022 and hi > 1024, (n, lo, hi)


def test_bounds_see_an_error_in_a_small_entry():
    """a relative error of 1e-10 in one small off-diagonal entry of R (1e-6 of max |R|) is far outside the componentwise bound,
    though a normwise check against max |R| would pass it"""
    a = torch.from_numpy(co.spd_global(128))
    r = torch.linalg.cholesky(a, upper=True)
    x = torch.linalg.inv(r)
    assert cr.chol_ratio(a, r) < 0.1 and cr.inv_ratio(r, x) < 0.1
    i, j = 3, 90
    r_bad = r.clone(); r_bad[i, j] *= 1 + 1e-10
    x_bad = x.clone(); x_bad[i, j] *= 1 + 1e-10
    assert cr.chol_ratio(a, r_bad) > GATE and cr.inv_ratio(r, x_bad) > GATE


# ---- the two-pivot step --------------------------------------------------------------------------------------------------------
BLOCK = co.spd_global(64)[:32, :32]


def _scipy_rel(a, r):
    ref = sla.cholesky(a)
    return float(np.abs(r - ref).max() / np.abs(ref).max()) if np.isfinite(r).all() else math.inf


@pytest.mark.parametrize("e", [-600, -560, -540, 520, 540])
def test_unguarded_pair_step_fails_outside_the_range(e):
    """diagonal entries of about 32 2^e: a b underflows (e < 0) or l^2 and a b overflow (e > 0)"""
    a = np.ldexp(BLOCK, e)
    r_old, info_old = cr.warp_potrf_32(a, guarded=False)
    assert info_old != 0 or _scipy_rel(a, r_old) > 1e-6, (info_old, _scipy_rel(a, r_old))
    r_new, info_new = cr.warp_potrf_32(a, guarded=True)
    assert info_new == 0 and _scipy_rel(a, r_new) <= 1e-15


def test_unguarded_pair_step_fails_on_a_graded_block():
    e = cr.ramp_exponents(32, 300)
    a = cr.graded(torch.from_numpy(BLOCK), e).numpy()
    d = np.ldexp(1.0, e.numpy())
    ref = sla.cholesky(BLOCK)
    r_old, info_old = cr.warp_potrf_32(a, guarded=False)
    assert info_old != 0
    r_new, info_new = cr.warp_potrf_32(a, guarded=True)
    assert info_new == 0
    assert np.abs(r_new / d[None, :] - ref).max() <= 1e-15 * np.abs(ref).max() * 32


def _ordinary_blocks():
    """blocks whose diagonal lies in [2^-400, 2^400]: the fixed kernel leaves them as they are"""
    yield "spd_global", BLOCK
    yield "kappa=1e6", cr.spd_spectrum(32, 1e6, 7).numpy()
    for e in (-380, -100, 100, 380):
        yield f"2^{e}", np.ldexp(BLOCK, e)
    yield "graded +-150", cr.graded(torch.from_numpy(BLOCK), cr.ramp_exponents(32, 150)).numpy()
    yield "diagonal", np.diag(np.arange(1.0, 33.0))


@pytest.mark.parametrize("name,a", list(_ordinary_blocks()), ids=lambda v: v if isinstance(v, str) else "")
def test_fix_keeps_the_bits_of_ordinary_blocks(name, a):
    d = np.diag(a)
    assert (d >= cr.BLOCK_SAFE[0]).all() and (d <= cr.BLOCK_SAFE[1]).all()
    r_old, info_old = cr.warp_potrf_32(a, guarded=False)
    r_new, info_new = cr.warp_potrf_32(a, guarded=True)
    assert info_old == info_new == 0
    assert np.array_equal(r_old, r_new)
    assert cr.chol_ratio(torch.from_numpy(a), torch.from_numpy(r_new)) <= GATE  # n = 32: one rounding is a sizeable part of gamma_33


@pytest.mark.parametrize("e", [-420, 410])
def test_equilibrated_blocks_match_lapack(e):
    """diagonal entries just outside [2^-400, 2^400], where the pairs are still in range: both routes agree with dpotrf"""
    a = np.ldexp(BLOCK, e)
    for guarded in (False, True):
        r, info = cr.warp_potrf_32(a, guarded)
        assert info == 0 and _scipy_rel(a, r) <= 1e-15


@pytest.mark.parametrize("e", [-600, 0, 540])
@pytest.mark.parametrize("pivot", [6, 7])
def test_guarded_pair_step_still_reports_non_spd(e, pivot):
    """a negative diagonal entry, and a zero row and column, at an even and an odd pivot (the first and second of a pair)"""
    neg = BLOCK.copy(); neg[pivot, pivot] = -5.0
    zero = BLOCK.copy(); zero[pivot, :] = 0.0; zero[:, pivot] = 0.0
    for a in (neg, zero):
        _, info = cr.warp_potrf_32(np.ldexp(a, e), guarded=True)
        assert info == pivot + 1
