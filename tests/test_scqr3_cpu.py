"""Shifted CholeskyQR3 (cacqr num_iter = 3) without a GPU.

  * the CholeskyQR / CholeskyQR2 schedules of the 3D and tunable grids enqueue exactly what they did before num_iter = 3 existed
    (sha256 of the capital_dist_trace_cacqr records of every rank);
  * the numpy restatement (tests/scqr3_reference.py) against an independent scipy formulation, and its accuracy up to kappa = 1e12;
  * the flag protocol of num_iter = 3 on the 2 x 2 x 2 and 2 x 4 x 2 grids (the replay checker of tests/test_dist_protocol.py),
    and that the waits of the Gram shift's scalar sum are load-bearing;
  * argument checks.
"""
import ctypes as C
import hashlib

import numpy as np
import pytest
import scipy.linalg as sla

import capital_b200 as cb
from capital_b200 import _lib
from oracle import capital_oracle as co
from scqr3_reference import ill_conditioned, scqr3, shift_coef
from test_cacqr_tune_cpu import cacqr_trace
from test_dist_protocol import Replay, T_WAIT

CTRL_SAR_LO, CTRL_SAR_HI = 288, 304  # control words of the Gram shift's flags (peer.cuh)

# sha256 over all ranks' capital_dist_trace_cacqr records (m, n = 512, 64, bc_mult_dim -1), recorded before num_iter = 3 existed.
# (size, num_iter, complete_inv); the 3D schedule always forms the complete inverse, so complete_inv does not change the records.
CACQR_TRACE_SHA256 = {
    (8, 1, 0): "23b5be187299cf1d87d43c791fca446abf9d9879f5c74c59848f7756fdcebbf4",
    (8, 1, 1): "23b5be187299cf1d87d43c791fca446abf9d9879f5c74c59848f7756fdcebbf4",
    (8, 2, 0): "03123753a8362ccd423704a2db0d5ebed946434a95aa8cfbfe68c66cbe87d89f",
    (8, 2, 1): "03123753a8362ccd423704a2db0d5ebed946434a95aa8cfbfe68c66cbe87d89f",
    (16, 1, 0): "0dd2ab68f79abd19931a4a4e07a90e9f9bbf2d25bd23916be7c776f20523a45a",
    (16, 1, 1): "0dd2ab68f79abd19931a4a4e07a90e9f9bbf2d25bd23916be7c776f20523a45a",
    (16, 2, 0): "afd9aba679ffcac0c1f12e53be2af8f2915f9e5cf56b3cf465ea6e4bebaef442",
    (16, 2, 1): "afd9aba679ffcac0c1f12e53be2af8f2915f9e5cf56b3cf465ea6e4bebaef442",
}


@pytest.mark.parametrize("size,num_iter,ci", sorted(CACQR_TRACE_SHA256))
def test_cqr_and_cqr2_schedules_unchanged(size, num_iter, ci):
    h = hashlib.sha256()
    for r in range(size):
        h.update(cacqr_trace(size, r, 2, 512, 64, num_iter, ci, -1).tobytes())
    assert h.hexdigest() == CACQR_TRACE_SHA256[(size, num_iter, ci)]


def test_restatement_matches_independent_scipy_formulation():
    m, n = 4096, 128
    a = ill_conditioned(m, n, 1e6, 1)
    # independent: shifted Cholesky, then two plain sweeps, Q by triangular solves instead of explicit inverses
    q, rs = a.copy(), []
    for it in range(3):
        g = q.T @ q
        if it == 0:
            g += shift_coef(m, n) * np.trace(g) * np.eye(n)
        r = sla.cholesky(g, lower=False)
        q = sla.solve_triangular(r, q.T, trans="T", lower=False).T
        rs.append(r)
    r_ind = rs[2] @ rs[1] @ rs[0]
    # R agrees to 1e-13 relative; Q's trailing columns move by about kappa u = 1.1e-10 under rounding (observed 5.7e-12)
    for bc in (None, 64):
        q_o, r_o = scqr3(a, bc)
        assert np.abs(r_o - r_ind).max() <= 1e-13 * np.abs(r_ind).max(), bc
        assert np.abs(q_o - q).max() <= 1e6 * 2.0 ** -53, bc


@pytest.mark.parametrize("m,n,kappa", [(8192, 256, 1e10), (8192, 256, 1e12), (2048, 512, 1e10), (2048, 512, 1e12)])
def test_restatement_accuracy_at_high_condition_numbers(m, n, kappa):
    a = ill_conditioned(m, n, kappa, 2)
    q, r = scqr3(a, 64)
    assert co.qr_residual(a, q, r) <= 1e-14
    assert co.qr_orthogonality(q) <= 1e-15
    assert (np.diag(r) > 0).all()
    with pytest.raises((np.linalg.LinAlgError, sla.LinAlgError, AssertionError)):
        co.cacqr_1d([a], 2)  # CholeskyQR2 breaks down on the same matrix


def test_restatement_3d_cholinv_agrees():
    """the 3D grids factor each Gram matrix with the distributed CholInv (process-face edge c): the same Q to rounding"""
    m, n = 2048, 128
    a = ill_conditioned(m, n, 1e10, 3)
    bc = co.bc_dimension(co.local_dim(n, 2), 2, 2, -1)
    q3, r3 = scqr3(a, bc, 2)
    assert co.qr_residual(a, q3, r3) <= 1e-14 and co.qr_orthogonality(q3) <= 1e-15


def sar_waits(tr):
    return (tr[:, 0] == T_WAIT) & (tr[:, 2] >= CTRL_SAR_LO) & (tr[:, 2] < CTRL_SAR_HI)


@pytest.mark.parametrize("size", [8, 16])
@pytest.mark.parametrize("ci", [0, 1])
def test_scqr3_protocol_is_deadlock_free_and_race_free(size, ci):
    traces = [cacqr_trace(size, r, 2, 512, 64, 3, ci, -1) for r in range(size)]
    # every diagonal rank (x = y) but the contributors of its own x waits once per call for each other contributor
    assert sum(int(sar_waits(tr).sum()) for tr in traces) > 0
    rp = Replay(traces)
    stuck = rp.run((2, 2))
    assert not stuck, f"deadlock: {len(stuck)} streams blocked, e.g. {stuck[:4]}"
    bad = rp.races()
    assert not bad, f"{len(bad)} unordered conflicting accesses, e.g. {bad[:3]}"


@pytest.mark.parametrize("size", [8, 16])
def test_shift_sum_wait_is_load_bearing(size):
    """without the waits for the contributors' flags the sum reads trace partials their copies may still be writing"""
    traces = [cacqr_trace(size, r, 2, 512, 64, 3, 1, -1) for r in range(size)]
    rp = Replay([tr[~sar_waits(tr)] for tr in traces])
    assert not rp.run((2, 2))
    assert rp.races()


@pytest.mark.parametrize("size,c", [(8, 1), (16, 1), (4, 1), (9, 3)])
def test_trace_rejects_grids_without_a_cube_schedule(size, c):
    g = cb.topo.rect(size, 0, c).grid
    args = _lib.CholinvArgs(1, 1, -1, b"U")
    cnt = C.c_int64()
    assert _lib.lib().capital_dist_trace_cacqr(C.byref(g), 512, 64, 3, C.byref(args), None, 0, C.byref(cnt)) == _lib.ERR_UNSUPPORTED


@pytest.mark.parametrize("num_iter", [0, 4])
def test_num_iter_outside_1_to_3_is_invalid(num_iter):
    g = cb.topo.rect(8, 0, 2).grid
    args = _lib.CholinvArgs(1, 1, -1, b"U")
    cnt = C.c_int64()
    assert _lib.lib().capital_dist_trace_cacqr(C.byref(g), 512, 64, num_iter, C.byref(args), None, 0, C.byref(cnt)) == _lib.ERR_INVALID
    with pytest.raises(ValueError):
        cb.cacqr.info(num_iter, cb.cholinv.info(0, 1, 0, "U"))


def test_info_accepts_three():
    assert cb.cacqr.info(3, cb.cholinv.info(0, 1, 0, "U")).num_iter == 3
