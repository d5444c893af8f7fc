"""CPU half of the grid edge tests (tests/mp_worker_grid_edges.py is the GPU half, tests/grid_edges_reference.py holds what they share).

  * the extended-precision reference against the oracle and scipy at every table size;
  * the protocol replay of tests/test_dist_protocol.py over the GPU worker's table: ragged local sizes (L = 501, 513, 648, 695, 777,
    1001) move every window offset, and CAPITAL_DIST_CHUNKS=3 at n = 1390 changes the chunk widths.  Every (grid, n, bc, knob set) is
    replayed on the 2- and 4-rank grids; on 2x2x2, where a replay takes tens of seconds, the two odd sizes under every knob set;
  * each knob set reaches the path it is named after, read from the trace -- this is what makes the GPU cases mean what they say."""
import numpy as np
import pytest
import scipy.linalg as sla

import grid_edges_reference as ge
from oracle import capital_oracle as co
from test_dist_protocol import Replay, trace, T_PRODUCT

DEFERRED = (2, 3, 4)  # compute streams of the deferred classes (S_FAR0 .. in dist.cu)
BULK_PUSH = 9         # push stream of the node-entry operands


@pytest.mark.parametrize("n", sorted(set(ge.SIZES[1] + ge.SIZES[2])))
def test_extended_precision_reference(n):
    a = co.spd_global(n)
    r, ri, r64, ri64 = ge.chol_ld(a)
    b = ge.Bounds(a)
    assert b.kappa < 2  # diagonally dominant generator
    # its own residuals are at the long double's rounding level, far below anything float64 can reach
    e_a, e_i = ge.residual_rows(r, ri, a, np.arange(0, n, 16))
    assert e_a <= n * 2.0 ** -63 * b.norm2 and e_i <= n * 2.0 ** -63 * b.kappa
    s = sla.cholesky(a, lower=False)
    assert np.abs(s - r64).max() <= b.forward_r and np.array_equal(np.tril(r64, -1), np.zeros_like(r64))
    assert np.abs(np.linalg.inv(s) - ri64).max() <= b.forward_rinv
    for d in (d for d in (1, 2) if n in ge.SIZES[d]):
        c = 2
        ro, rio = co.cholinv(a, True, 2, co.bc_dimension(n // d, c, d, -3), d=d)
        assert np.abs(ro - r64).max() <= 2e-13 * np.abs(r64).max()
        assert np.abs(rio - ri64).max() <= 2e-13 * np.abs(ri64).max()
        assert np.abs(ro - r64).max() <= b.forward_r and np.abs(rio - ri64).max() <= b.forward_rinv


def set_knobs(monkeypatch, knob):
    for k in ge.KNOB_NAMES:
        monkeypatch.delenv(k, raising=False)
    for k, v in ge.KNOBS[knob].items():
        monkeypatch.setenv(k, v)


def replay_table():
    out = []
    for size, (c, d) in ge.GRIDS.items():
        seen = []
        for n, ci, split, bcm, serialize, knob in ge.cases(size):
            if (n, bcm, knob) not in seen and (size != 8 or bcm == -3):
                seen.append((n, bcm, knob))
        out += [(size, n, bcm, knob) + ((0, 2), (1, 1))[i % 2] for i, (n, bcm, knob) in enumerate(seen)]
    return out


@pytest.mark.parametrize("size,n,bcm,knob,ci,split", replay_table())
def test_table_drains_race_free_and_reaches_its_path(size, n, bcm, knob, ci, split, monkeypatch):
    c, d = ge.GRIDS[size]

    def traces(name):
        set_knobs(monkeypatch, name)
        return [trace(size, r, c, n, ci, bcm, split) for r in range(size)]

    def products(trs, streams=None):
        return sum(int(((t[:, 0] == T_PRODUCT) & (np.isin(t[:, 1], streams) if streams else True)).sum()) for t in trs)

    def same(a, b):
        return all(x.shape == y.shape and np.array_equal(x, y) for x, y in zip(a, b))

    trs = traces(knob)
    rp = Replay(trs)
    stuck = rp.run((c, d))
    assert not stuck, f"deadlock: {len(stuck)} streams blocked, e.g. {stuck[:4]}"
    bad = rp.races()
    assert not bad, f"{len(bad)} unordered conflicting accesses, e.g. {bad[:3]}"
    if knob == "default":
        return
    base = traces("default")
    if knob == "one":
        assert products(trs, DEFERRED) == 0
        assert products(trs) > products(base)  # ... and its products are chunked on the chain
        return
    assert products(trs) > products(base)      # CHUNK_MIN lowered: chunked, pushed products
    assert products(trs, DEFERRED) > products(base, DEFERRED)  # SIDE_MIN / FAR_MIN lowered: deferred classes (none by default for L < 1024)
    if knob != "low":
        assert not same(trs, traces("low")), f"{knob} schedules exactly what low does at n = {n}"
    if knob == "nobulk":
        on_bulk = lambda ts: sum(int((t[:, 1] == BULK_PUSH).sum()) for t in ts)
        assert on_bulk(trs) < on_bulk(traces("low"))
