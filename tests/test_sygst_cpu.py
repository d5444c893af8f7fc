"""cholinv::sygst and apply_Rinv / apply_RinvT without a GPU: the numpy model of the n^3 formulation against LAPACK's dsygst, the flag
protocol of the grid schedule (dry-run traces replayed under CUDA's ordering rules), and the argument checks of the C ABI and of the
Python mirror (they must reject bad input before any device call)."""
import ctypes as C
import numpy as np
import pytest
import scipy.linalg as sla
import torch
import capital_b200 as cb
from capital_b200 import _lib
from oracle import capital_oracle as co
from solve_reference import top_split
from sygst_reference import bound, dsygst_full, sygst, u_transpose
from test_dist_protocol import GRIDS, T_DMA, T_PRODUCT, T_WAIT, T_WRITE, Replay


def _symmetric(n, seed):
    g = np.random.default_rng(seed).standard_normal((n, n))
    return g + g.T


@pytest.mark.parametrize("n", [96, 128, 200])
@pytest.mark.parametrize("d", [1, 2])
@pytest.mark.parametrize("split", [1, 2])
@pytest.mark.parametrize("ci", [0, 1])
def test_model_matches_dsygst(n, d, split, ci):
    b = co.spd_global(n)
    bc = co.bc_dimension(n // d, d, d, -2)
    r, ri = co.cholinv(b, bool(ci), split, bc, d=d)
    if not ci:
        n1 = top_split(n, False, split, bc, d)
        assert n1 is not None and np.count_nonzero(ri[:n1, n1:]) == 0  # the skipped block really is missing
    a = _symmetric(n, n + 7 * d + split)
    c = sygst(a, r, ri, bool(ci), split, bc, d)
    ref = dsygst_full(a, r)
    ri_full = np.linalg.inv(r)
    err = np.abs(c - ref)
    bnd = bound(a, ri_full)
    assert np.all(err <= bnd / 10), float((err / bnd).max())  # the model keeps a 10x margin inside the bound the GPU tests use
    assert np.array_equal(c, c.T)


def test_model_reads_only_the_lower_triangle_and_gives_the_eigenvalues():
    n = 200
    b = co.spd_global(n)
    r, ri = co.cholinv(b, True, 1, co.bc_dimension(n, 1, 1, -2))
    a = _symmetric(n, 3)
    poisoned = a.copy()
    poisoned[np.triu_indices(n, 1)] = np.nan
    c = sygst(poisoned, r, ri, True, 1, n)
    assert np.array_equal(c, sygst(a, r, ri, True, 1, n))
    ut = u_transpose(a)
    assert np.array_equal(ut + ut.T, a)  # the split is exact
    lam = np.linalg.eigvalsh(c)
    ref = sla.eigh(a, b, eigvals_only=True)
    assert np.abs(lam - ref).max() <= 1e-13 * np.abs(ref).max()


def _trace(size, rank, c, n, ci, bcm, split=1):
    g = cb.topo.square(size, rank, c).grid
    args = _lib.CholinvArgs(ci, split, bcm, b"U")
    cnt = C.c_int64()
    L = _lib.lib()
    assert L.capital_dist_trace_cholinv_sygst(C.byref(g), n, C.byref(args), None, 0, C.byref(cnt)) == _lib.OK
    buf = np.zeros((cnt.value, 8), dtype=np.int64)
    assert L.capital_dist_trace_cholinv_sygst(C.byref(g), n, C.byref(args), buf.ctypes.data_as(C.POINTER(C.c_int64)), cnt.value,
                                              C.byref(cnt)) == _lib.OK
    return buf


def _pushed_windows(tr):
    """(destination rank, arena offset) of every peer DMA of the trace: the write record that precedes each T_DMA"""
    out = []
    for i in range(1, len(tr)):
        if tr[i, 0] == T_DMA and tr[i - 1, 0] == T_WRITE:
            out.append((int(tr[i - 1, 2]), int(tr[i - 1, 3])))
    return out


@pytest.mark.parametrize("size", [2, 4, 8])
@pytest.mark.parametrize("ci", [0, 1])
@pytest.mark.parametrize("n,split", [(1024, 1), (2048, 2)])
def test_flag_protocol_is_deadlock_free_and_race_free(size, ci, n, split, monkeypatch):
    monkeypatch.setenv("CAPITAL_DIST_CHUNK_MIN", "256")  # a rebuilt Rinv12 is produced and pushed in chunks
    c, d = GRIDS[size]
    traces = [_trace(size, r, c, n, ci, -3, split) for r in range(size)]
    rp = Replay(traces)
    stuck = rp.run((c, d))
    assert not stuck, f"deadlock: {len(stuck)} streams blocked, e.g. {stuck[:4]}"
    kinds = np.concatenate(traces)[:, 0]
    assert (kinds == T_PRODUCT).sum() > 0
    if d > 1:
        assert (kinds == T_DMA).sum() > 0 and (kinds == T_WAIT).sum() > 0
    bad = rp.races()
    assert not bad, f"{len(bad)} unordered conflicting accesses, e.g. {bad[:3]}"
    # every window of a mirror slot is pushed at most once per call (the trace holds two calls)
    for tr in traces:
        keys, counts = np.unique(np.array(_pushed_windows(tr) or [(0, 0)]), axis=0, return_counts=True)
        assert counts.max() <= 2, keys[counts.argmax()]


def test_skipped_block_adds_the_two_products():
    """complete_inv = 0 on a splitting top node: the trace holds the T^T and Rinv12 products besides the three of sygst."""
    counts = []
    for ci in (0, 1):
        tr = _trace(8, 0, 2, 1024, ci, -3)
        counts.append(int((tr[:, 0] == T_PRODUCT).sum()))
    assert counts[0] > counts[1] > 0


def test_trace_rejects_bad_arguments():
    g = cb.topo.square(8, 0, 2).grid
    cnt = C.c_int64()
    bad = _lib.CholinvArgs(1, 0, -2, b"U")
    assert _lib.lib().capital_dist_trace_cholinv_sygst(C.byref(g), 1024, C.byref(bad), None, 0, C.byref(cnt)) == _lib.ERR_INVALID
    ok = _lib.CholinvArgs(1, 1, -2, b"U")
    assert _lib.lib().capital_dist_trace_cholinv_sygst(C.byref(g), 1025, C.byref(ok), None, 0, C.byref(cnt)) == _lib.ERR_UNSUPPORTED


def test_c_abi_rejects_a_null_context():
    args = _lib.CholinvArgs(1, 1, -1, b"U")
    x = (C.c_double * 16)()
    y = (C.c_double * 16)()
    L = _lib.lib()
    assert L.capital_cholinv_sygst_f64(None, 4, C.byref(args), _lib.UPPERTRI_PACKED, x, x, x, y) == _lib.ERR_INVALID
    for trans in (0, 1):
        assert L.capital_cholinv_apply_rinv_f64(None, 4, C.byref(args), _lib.UPPERTRI_PACKED, None, x, trans, 1, x, 4, y, 4) \
            == _lib.ERR_INVALID


def _factored_info(n, serialize=True):
    args = cb.cholinv.info(1, 1, -1, "U", serialize=serialize)
    args.R = torch.zeros(n * (n + 1) // 2 if serialize else n * n, dtype=torch.float64)
    args.Rinv = torch.zeros_like(args.R)
    args.local_dim = args.global_dim = n
    return args


def test_python_rejects_an_unfactored_info():
    topo = cb.topo.square(1, 0, 1)
    with pytest.raises(ValueError):
        cb.cholinv.sygst(cb.matrix(8, 8, 1, 1, device="cpu"), cb.cholinv.info(1, 1, -1, "U"), topo)
    for fn in (cb.cholinv.apply_Rinv, cb.cholinv.apply_RinvT):
        with pytest.raises(ValueError):
            fn(cb.cholinv.info(1, 1, -1, "U"), torch.zeros(8, dtype=torch.float64), topo)


@pytest.mark.parametrize("serialize", [True, False])
def test_python_rejects_factors_of_the_wrong_size(serialize):
    topo = cb.topo.square(1, 0, 1)
    A = cb.matrix(8, 8, 1, 1, device="cpu")
    args = _factored_info(8, serialize)
    args.Rinv = torch.zeros(args.R.numel() + 1, dtype=torch.float64)
    with pytest.raises(ValueError):
        cb.cholinv.sygst(A, args, topo)
    with pytest.raises(ValueError):
        cb.cholinv.apply_Rinv(args, torch.zeros(8, dtype=torch.float64), topo)
    args = _factored_info(8, serialize)
    args.local_dim = 9
    with pytest.raises(ValueError):
        cb.cholinv.apply_RinvT(args, torch.zeros(8, dtype=torch.float64), topo)


@pytest.mark.parametrize("bad", ["size", "dtype", "matrix", "object"])
def test_python_sygst_rejects_a_wrong_matrix(bad):
    args = _factored_info(8)
    A = cb.matrix(8, 8, 1, 1, device="cpu")
    if bad == "size":
        A = cb.matrix(9, 9, 1, 1, device="cpu")
    elif bad == "dtype":
        A.data = torch.zeros(64, dtype=torch.float32)
    elif bad == "matrix":
        A = cb.matrix(8, 16, 1, 2, device="cpu")  # 8 local rows but 16 global ones
    else:
        A = torch.zeros(64, dtype=torch.float64)
    with pytest.raises(ValueError):
        cb.cholinv.sygst(A, args, cb.topo.square(1, 0, 1))


@pytest.mark.parametrize("shape", [(7,), (9, 2), (8, 0), (8, 2, 1)])
@pytest.mark.parametrize("dtype", [torch.float64, torch.float32])
def test_python_apply_rejects_wrong_right_hand_sides(shape, dtype):
    if dtype == torch.float32:
        shape = (8, 2)
    for fn in (cb.cholinv.apply_Rinv, cb.cholinv.apply_RinvT):
        with pytest.raises(ValueError):
            fn(_factored_info(8), torch.zeros(shape, dtype=dtype), cb.topo.square(1, 0, 1))
