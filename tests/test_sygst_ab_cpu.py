"""cholinv::sygst for itype 2 and 3 (A B x = lambda x, B A x = lambda x) and apply_R / apply_RT without a GPU: the numpy model of the
n^3 formulation against LAPACK's dsygst, the flag protocol of the grid schedule (dry-run traces replayed under CUDA's ordering rules),
and the argument checks of the C ABI and of the Python mirror (they must reject bad input before any device call)."""
import ctypes as C
import numpy as np
import pytest
import scipy.linalg as sla
import torch
import capital_b200 as cb
from capital_b200 import _lib
from oracle import capital_oracle as co
from sygst_ab_reference import bound, dsygst_full, sygst_ab
from sygst_reference import u_transpose
from test_dist_protocol import GRIDS, T_DMA, T_PRODUCT, T_WAIT, T_WRITE, Replay


def _symmetric(n, seed):
    g = np.random.default_rng(seed).standard_normal((n, n))
    return g + g.T


@pytest.mark.parametrize("n", [96, 128, 200])
@pytest.mark.parametrize("d", [1, 2])
@pytest.mark.parametrize("itype", [2, 3])
def test_model_matches_dsygst(n, d, itype):
    b = co.spd_global(n)
    r, _ = co.cholinv(b, True, 1, co.bc_dimension(n // d, d, d, -2), d=d)
    a = _symmetric(n, n + 7 * d + itype)
    c = sygst_ab(a, r)
    ref = dsygst_full(a, r, itype)
    err = np.abs(c - ref)
    bnd = bound(a, r)
    assert np.all(err <= bnd / 10), float((err / bnd).max())  # the model keeps a 10x margin inside the bound the GPU tests use
    assert np.array_equal(c, c.T)
    w = r @ u_transpose(a).T
    assert np.count_nonzero(np.tril(w, -1)) == 0  # W = R U is upper triangular, exactly


@pytest.mark.parametrize("itype", [2, 3])
def test_model_reads_only_the_lower_triangle_and_gives_the_eigenvalues(itype):
    n = 200
    b = co.spd_global(n)
    r, _ = co.cholinv(b, True, 1, co.bc_dimension(n, 1, 1, -2))
    a = _symmetric(n, 3)
    poisoned = a.copy()
    poisoned[np.triu_indices(n, 1)] = np.nan
    c = sygst_ab(poisoned, r)
    assert np.array_equal(c, sygst_ab(a, r))
    lam = np.linalg.eigvalsh(c)
    ref = sla.eigh(a, b, type=itype, eigvals_only=True)
    assert np.abs(lam - ref).max() <= 1e-13 * np.abs(ref).max()


def _trace(size, rank, c, n, ci, bcm, split=1):
    g = cb.topo.square(size, rank, c).grid
    args = _lib.CholinvArgs(ci, split, bcm, b"U")
    cnt = C.c_int64()
    L = _lib.lib()
    assert L.capital_dist_trace_cholinv_sygst_ab(C.byref(g), n, C.byref(args), None, 0, C.byref(cnt)) == _lib.OK
    buf = np.zeros((cnt.value, 8), dtype=np.int64)
    assert L.capital_dist_trace_cholinv_sygst_ab(C.byref(g), n, C.byref(args), buf.ctypes.data_as(C.POINTER(C.c_int64)), cnt.value,
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
def test_flag_protocol_is_deadlock_free_and_race_free(size, ci, n, split):
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


def test_complete_inv_changes_nothing():
    """only R is read: the schedule is the same whether or not the factor skipped the top-level Rinv12"""
    assert np.array_equal(_trace(8, 0, 2, 1024, 0, -3), _trace(8, 0, 2, 1024, 1, -3))


def test_trace_rejects_bad_arguments():
    g = cb.topo.square(8, 0, 2).grid
    cnt = C.c_int64()
    bad = _lib.CholinvArgs(1, 0, -2, b"U")
    assert _lib.lib().capital_dist_trace_cholinv_sygst_ab(C.byref(g), 1024, C.byref(bad), None, 0, C.byref(cnt)) == _lib.ERR_INVALID
    ok = _lib.CholinvArgs(1, 1, -2, b"U")
    assert _lib.lib().capital_dist_trace_cholinv_sygst_ab(C.byref(g), 1025, C.byref(ok), None, 0, C.byref(cnt)) == _lib.ERR_UNSUPPORTED


def test_c_abi_rejects_a_null_context():
    args = _lib.CholinvArgs(1, 1, -1, b"U")
    x = (C.c_double * 16)()
    y = (C.c_double * 16)()
    L = _lib.lib()
    assert L.capital_cholinv_sygst_ab_f64(None, 4, C.byref(args), _lib.UPPERTRI_PACKED, x, x, y) == _lib.ERR_INVALID
    for trans in (0, 1, 2):
        assert L.capital_cholinv_apply_r_f64(None, 4, C.byref(args), _lib.UPPERTRI_PACKED, x, trans, 1, x, 4, y, 4) == _lib.ERR_INVALID


def _factored_info(n, serialize=True):
    args = cb.cholinv.info(1, 1, -1, "U", serialize=serialize)
    args.R = torch.zeros(n * (n + 1) // 2 if serialize else n * n, dtype=torch.float64)
    args.Rinv = torch.zeros_like(args.R)
    args.local_dim = args.global_dim = n
    return args


@pytest.mark.parametrize("itype", [0, 4, -1, 2.5, "2", True, None])
def test_python_sygst_rejects_a_bad_itype(itype):
    with pytest.raises(ValueError):
        cb.cholinv.sygst(cb.matrix(8, 8, 1, 1, device="cpu"), _factored_info(8), cb.topo.square(1, 0, 1), itype=itype)


def test_python_rejects_an_unfactored_info():
    topo = cb.topo.square(1, 0, 1)
    for itype in (2, 3):
        with pytest.raises(ValueError):
            cb.cholinv.sygst(cb.matrix(8, 8, 1, 1, device="cpu"), cb.cholinv.info(1, 1, -1, "U"), topo, itype=itype)
    for fn in (cb.cholinv.apply_R, cb.cholinv.apply_RT):
        with pytest.raises(ValueError):
            fn(cb.cholinv.info(1, 1, -1, "U"), torch.zeros(8, dtype=torch.float64), topo)


@pytest.mark.parametrize("serialize", [True, False])
def test_python_rejects_factors_of_the_wrong_size(serialize):
    topo = cb.topo.square(1, 0, 1)
    A = cb.matrix(8, 8, 1, 1, device="cpu")
    args = _factored_info(8, serialize)
    args.R = torch.zeros(args.R.numel() + 1, dtype=torch.float64)
    with pytest.raises(ValueError):
        cb.cholinv.sygst(A, args, topo, itype=2)
    with pytest.raises(ValueError):
        cb.cholinv.apply_R(args, torch.zeros(8, dtype=torch.float64), topo)
    args = _factored_info(8, serialize)
    args.local_dim = 9
    with pytest.raises(ValueError):
        cb.cholinv.apply_RT(args, torch.zeros(8, dtype=torch.float64), topo)


@pytest.mark.parametrize("bad", ["size", "dtype", "matrix", "object"])
@pytest.mark.parametrize("itype", [2, 3])
def test_python_sygst_rejects_a_wrong_matrix(bad, itype):
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
        cb.cholinv.sygst(A, args, cb.topo.square(1, 0, 1), itype=itype)


@pytest.mark.parametrize("shape", [(7,), (9, 2), (8, 0), (8, 2, 1)])
@pytest.mark.parametrize("dtype", [torch.float64, torch.float32])
def test_python_apply_rejects_wrong_right_hand_sides(shape, dtype):
    if dtype == torch.float32:
        shape = (8, 2)
    for fn in (cb.cholinv.apply_R, cb.cholinv.apply_RT):
        with pytest.raises(ValueError):
            fn(_factored_info(8), torch.zeros(shape, dtype=dtype), cb.topo.square(1, 0, 1))
