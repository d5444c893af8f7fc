"""CA-CholeskyQR2 on the tunable c x d x c grid (1 < c < d; the reference's sweep_tune, cacqr.hpp:122-170), without a GPU.

  * the reference's own 16-rank dumps (tests/golden/cacqr_p16_tune_*.npz) against the generator and the numpy restatement
    (the tunable grid computes what the 3D algorithm computes on the whole matrix);
  * the flag protocol of the schedule: `capital_dist_trace_cacqr` dry-runs what each of the 16 ranks of the 2 x 4 x 2 grid enqueues
    for two consecutive cacqr::factor calls -- two 2x2x2 cubes plus the cross-cube Gram all-reduce -- and the traces are replayed
    with the checker of tests/test_dist_protocol.py (deadlock freedom, every conflicting arena access ordered by happens-before);
  * the grids that existed before keep their schedules.
"""
import ctypes as C
import hashlib
import json
import os

import numpy as np
import pytest

import capital_b200 as cb
from capital_b200 import _lib
from oracle import capital_oracle as co
from test_dist_protocol import Replay, T_WAIT, trace as cholinv_trace

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
TUNE = ["cacqr_p16_tune_m512_n64", "cacqr_p16_tune_m512_n64_ci0", "cacqr_p16_tune_m512_n64_it1"]
P, C_, D_ = 16, 2, 4
CTRL_GAR_LO, CTRL_GAR_HI = 272, 288  # control words of the cross-cube all-reduce flags (peer.cuh)


def load(name):
    z = dict(np.load(os.path.join(GOLD, name + ".npz")))
    meta = json.loads(str(z["meta"]))
    for r, s in meta.get("replica_of", {}).items():  # layer replicas are stored once (tests/golden/make_golden_tune.py)
        for k in [k for k in z if k.endswith(f"_{s}")]:
            z[k[: -len(str(s))] + r] = z[k]
    return meta, z


def local(v, rows, cols):
    return v.reshape(cols, rows).T  # column-major local block


def expected_packed_R(R, c, x, yc):
    """the rank's packed block of R on its cube's c x c square grid: cyclic (x, y mod c), zeros on the local diagonal when y > x"""
    loc = np.triu(co.cyclic_local(R, c, c, x, yc))
    if yc > x:
        np.fill_diagonal(loc, 0.0)
    return co.pack_upper(loc)


@pytest.mark.parametrize("name", TUNE)
def test_generator_matches_reference_dump(name):
    meta, z = load(name)
    m, n = meta["m"], meta["n"]
    assert (meta["P"], meta["c"], meta["d"]) == (P, C_, D_)
    for r in range(P):
        t = co.topo_rect(P, r, C_)
        a = co.random_local(m, n, C_, D_, t["x"], t["y"], r // C_)
        assert np.array_equal(a.ravel(order="F"), z[f"A_{r}"]), r


@pytest.mark.parametrize("name", TUNE)
def test_reference_dump_matches_restatement(name):
    meta, z = load(name)
    m, n, it = meta["m"], meta["n"], meta["variant"]
    ci = 0 if name.endswith("_ci0") else 1
    lr, lc = m // D_, n // C_
    blocks_a, blocks_q = {}, {}
    for r in range(P):
        t = co.topo_rect(P, r, C_)
        blocks_a[(t["x"], t["y"])] = local(z[f"A_{r}"], lr, lc)
        blocks_q[(t["x"], t["y"])] = local(z[f"Q_{r}"], lr, lc)
    A = co.cyclic_assemble(blocks_a, m, n, C_, D_)
    Q = co.cyclic_assemble(blocks_q, m, n, C_, D_)
    q_o, r_o = co.cacqr_3d(A, C_, it, bool(ci), 1, -1)
    assert np.abs(Q - q_o).max() <= 1e-13
    for r in range(P):
        t = co.topo_rect(P, r, C_)
        exp = expected_packed_R(r_o, C_, t["x"], t["y"] % C_)
        assert np.abs(z[f"R_{r}"] - exp).max() <= 1e-13 * np.abs(r_o).max(), r
        if r < P // 2:
            assert np.array_equal(z[f"R_{r}"], z[f"R_{r + P // 2}"]), r  # R is replicated in both cubes
    assert meta["residual"] < 1e-14 and meta["orthogonality"] < 1e-15


def cacqr_trace(size, rank, c, m, n, num_iter, ci, bcm):
    g = cb.topo.rect(size, rank, c).grid
    args = _lib.CholinvArgs(ci, 1, bcm, b"U")
    cnt = C.c_int64()
    L = _lib.lib()
    st = L.capital_dist_trace_cacqr(C.byref(g), m, n, num_iter, C.byref(args), None, 0, C.byref(cnt))
    assert st == 0
    buf = np.zeros((cnt.value, 8), dtype=np.int64)
    st = L.capital_dist_trace_cacqr(C.byref(g), m, n, num_iter, C.byref(args), buf.ctypes.data_as(C.POINTER(C.c_int64)), cnt.value,
                                    C.byref(cnt))
    assert st == 0
    return buf


def gar_waits(tr):
    return (tr[:, 0] == T_WAIT) & (tr[:, 2] >= CTRL_GAR_LO) & (tr[:, 2] < CTRL_GAR_HI)


# (m, n, bc_mult): n = 128 with bc_mult -3 gives the cube's cholinv several recursion levels (local 64 -> ... -> base case 2)
@pytest.mark.parametrize("m,n,bcm", [(512, 64, -1), (256, 128, -3)])
@pytest.mark.parametrize("num_iter", [1, 2])
@pytest.mark.parametrize("ci", [0, 1])
def test_tunable_grid_protocol_is_deadlock_free_and_race_free(m, n, bcm, num_iter, ci):
    traces = [cacqr_trace(P, r, C_, m, n, num_iter, ci, bcm) for r in range(P)]
    for tr in traces:
        assert gar_waits(tr).sum() == 2 * num_iter  # one cross-cube all-reduce per sweep, two calls, one partner cube
    rp = Replay(traces)
    stuck = rp.run((C_, C_))
    assert not stuck, f"deadlock: {len(stuck)} streams blocked, e.g. {stuck[:4]}"
    bad = rp.races()
    assert not bad, f"{len(bad)} unordered conflicting accesses, e.g. {bad[:3]}"


def test_cross_cube_wait_is_load_bearing():
    """without the wait for the partner cube's flag the sum reads a Gram slot the partner's copy may still be writing"""
    traces = [cacqr_trace(P, r, C_, 512, 64, 2, 1, -1) for r in range(P)]
    rp = Replay([tr[~gar_waits(tr)] for tr in traces])
    assert not rp.run((C_, C_))
    assert rp.races()


def test_second_slot_set_is_load_bearing(monkeypatch):
    """with a single set of Gram slots the second sweep's copy overwrites a slot the partner cube has not added up yet"""
    monkeypatch.setenv("CAPITAL_DIST_GRAM_SETS", "1")
    traces = [cacqr_trace(P, r, C_, 512, 64, 2, 1, -1) for r in range(P)]
    rp = Replay(traces)
    assert not rp.run((C_, C_))
    assert rp.races()


def test_3d_grid_protocol_is_clean_too():
    traces = [cacqr_trace(8, r, 2, 256, 64, 2, 1, -1) for r in range(8)]
    assert not any(gar_waits(tr).any() for tr in traces)  # a c == d grid is one cube: no cross-cube step
    rp = Replay(traces)
    assert not rp.run((2, 2))
    assert not rp.races()


@pytest.mark.parametrize("size,c", [(8, 1), (16, 1), (4, 1), (9, 3)])
def test_trace_rejects_grids_without_a_cube_schedule(size, c):
    g = cb.topo.rect(size, 0, c).grid
    args = _lib.CholinvArgs(1, 1, -1, b"U")
    cnt = C.c_int64()
    assert _lib.lib().capital_dist_trace_cacqr(C.byref(g), 512, 64, 2, C.byref(args), None, 0, C.byref(cnt)) == _lib.ERR_UNSUPPORTED


# sha256 over the 8 ranks' capital_dist_trace_cholinv records of the 2x2x2 grid, recorded before the schedules learned to run on a
# sub-grid: the grids without cubes must enqueue exactly what they did
CHOLINV_TRACE_SHA256 = {
    (1024, 1, -2): "4ced59a4827b26d9f6a1ab28d67420195294096032ab897ee07d66187f206807",
    (2048, 0, -3): "3d62da0c24d3190836ffde8411666e45efc482af7e2784b62e11700e197c5192",
}


@pytest.mark.parametrize("n,ci,bcm", sorted(CHOLINV_TRACE_SHA256))
def test_cholinv_schedule_unchanged(n, ci, bcm, monkeypatch):
    for k in ("CAPITAL_DIST_FAR_MIN", "CAPITAL_DIST_SIDE_MIN", "CAPITAL_DIST_CHUNK_MIN", "CAPITAL_DIST_TWO_STREAM", "CAPITAL_DIST_CHUNKS",
              "CAPITAL_DIST_BULK", "CAPITAL_DIST_PIPELINE", "CAPITAL_DIST_FLUSH_READS"):
        monkeypatch.delenv(k, raising=False)
    h = hashlib.sha256()
    for r in range(8):
        h.update(cholinv_trace(8, r, 2, n, ci, bcm).tobytes())
    assert h.hexdigest() == CHOLINV_TRACE_SHA256[(n, ci, bcm)]
