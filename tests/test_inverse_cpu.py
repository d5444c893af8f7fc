"""cholinv::inverse without a GPU: the rebuilt-Rinv12 formula against the complete factors, the flag protocol of the grid schedule
(dry-run traces replayed under CUDA's ordering rules), and the argument checks of the C ABI and of the Python mirror (they must reject
bad input before any device call)."""
import ctypes as C
import numpy as np
import pytest
import torch
import capital_b200 as cb
from capital_b200 import _lib
from oracle import capital_oracle as co
from inverse_reference import cholesky_inverse, rebuild_rinv
from solve_reference import top_split
from test_dist_protocol import GRIDS, T_DMA, T_PRODUCT, T_WAIT, Replay


@pytest.mark.parametrize("n", [96, 128, 200])
@pytest.mark.parametrize("d", [1, 2])
@pytest.mark.parametrize("split", [1, 2])
def test_rebuilt_rinv12_matches_the_complete_factor(n, d, split):
    a = co.spd_global(n)
    bc = co.bc_dimension(n // d, d, d, -2)
    r1, ri1 = co.cholinv(a, True, split, bc, d=d)
    r0, ri0 = co.cholinv(a, False, split, bc, d=d)
    n1 = top_split(n, False, split, bc, d)
    assert n1 is not None and np.count_nonzero(ri0[:n1, n1:]) == 0  # the skipped block really is missing
    assert np.abs(rebuild_rinv(r0, ri0, False, split, bc, d) - ri1).max() <= 1e-14 * np.abs(ri1).max()
    ainv = cholesky_inverse(r0, ri0, False, split, bc, d)
    ref = np.linalg.inv(a)
    assert np.abs(ainv - ref).max() <= 1e-13 * np.abs(ref).max()


def _trace(size, rank, c, n, ci, bcm, split=1):
    g = cb.topo.square(size, rank, c).grid
    args = _lib.CholinvArgs(ci, split, bcm, b"U")
    cnt = C.c_int64()
    L = _lib.lib()
    assert L.capital_dist_trace_cholinv_inverse(C.byref(g), n, C.byref(args), None, 0, C.byref(cnt)) == _lib.OK
    buf = np.zeros((cnt.value, 8), dtype=np.int64)
    assert L.capital_dist_trace_cholinv_inverse(C.byref(g), n, C.byref(args), buf.ctypes.data_as(C.POINTER(C.c_int64)), cnt.value,
                                                C.byref(cnt)) == _lib.OK
    return buf


@pytest.mark.parametrize("size", [2, 4, 8])
@pytest.mark.parametrize("ci", [0, 1])
@pytest.mark.parametrize("n,split", [(1024, 1), (2048, 2)])
def test_flag_protocol_is_deadlock_free_and_race_free(size, ci, n, split, monkeypatch):
    monkeypatch.setenv("CAPITAL_DIST_CHUNK_MIN", "256")  # the rebuilt Rinv12 is produced and pushed in chunks
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


def test_skipped_block_adds_the_two_products():
    """complete_inv = 0 on a splitting top node: the trace holds the T^T and Rinv12 products besides the inverse product."""
    counts = []
    for ci in (0, 1):
        tr = _trace(8, 0, 2, 1024, ci, -3)
        counts.append(int((tr[:, 0] == T_PRODUCT).sum()))
    assert counts[0] > counts[1] > 0


def test_trace_rejects_bad_arguments():
    g = cb.topo.square(8, 0, 2).grid
    cnt = C.c_int64()
    bad = _lib.CholinvArgs(1, 0, -2, b"U")
    assert _lib.lib().capital_dist_trace_cholinv_inverse(C.byref(g), 1024, C.byref(bad), None, 0, C.byref(cnt)) == _lib.ERR_INVALID
    ok = _lib.CholinvArgs(1, 1, -2, b"U")
    assert _lib.lib().capital_dist_trace_cholinv_inverse(C.byref(g), 1025, C.byref(ok), None, 0, C.byref(cnt)) == _lib.ERR_UNSUPPORTED


def test_c_abi_rejects_a_null_context():
    args = _lib.CholinvArgs(1, 1, -1, b"U")
    x = (C.c_double * 16)()
    y = (C.c_double * 16)()
    r = C.c_double()
    L = _lib.lib()
    assert L.capital_cholinv_inverse_f64(None, 4, C.byref(args), _lib.UPPERTRI_PACKED, x, x, y) == _lib.ERR_INVALID
    assert L.capital_cholinv_inverse_residual_f64(None, x, 4, _lib.RECT, y, C.byref(r)) == _lib.ERR_INVALID


def _factored_info(n, serialize=True):
    args = cb.cholinv.info(1, 1, -1, "U", serialize=serialize)
    args.R = torch.zeros(n * (n + 1) // 2 if serialize else n * n, dtype=torch.float64)
    args.Rinv = torch.zeros_like(args.R)
    args.local_dim = args.global_dim = n
    return args


def test_python_inverse_rejects_an_unfactored_info():
    topo = cb.topo.square(1, 0, 1)
    with pytest.raises(ValueError):
        cb.cholinv.inverse(cb.cholinv.info(1, 1, -1, "U"), topo)
    with pytest.raises(ValueError):
        cb.cholinv.inverse_residual(cb.matrix(8, 8, 1, 1, device="cpu"), torch.zeros(36, dtype=torch.float64),
                                    cb.cholinv.info(1, 1, -1, "U"), topo)


@pytest.mark.parametrize("serialize", [True, False])
def test_python_inverse_rejects_factors_of_the_wrong_size(serialize):
    args = _factored_info(8, serialize)
    args.Rinv = torch.zeros(args.R.numel() + 1, dtype=torch.float64)
    with pytest.raises(ValueError):
        cb.cholinv.inverse(args, cb.topo.square(1, 0, 1))
    args = _factored_info(8, serialize)
    args.local_dim = 9
    with pytest.raises(ValueError):
        cb.cholinv.inverse(args, cb.topo.square(1, 0, 1))


@pytest.mark.parametrize("bad", ["size", "dtype", "matrix"])
def test_python_inverse_residual_rejects_wrong_operands(bad):
    args = _factored_info(8)
    A = cb.matrix(8, 8, 1, 1, device="cpu")
    Ainv = torch.zeros(36, dtype=torch.float64)
    if bad == "size":
        Ainv = torch.zeros(64, dtype=torch.float64)
    elif bad == "dtype":
        Ainv = torch.zeros(36, dtype=torch.float32)
    else:
        A = cb.matrix(9, 9, 1, 1, device="cpu")
    with pytest.raises(ValueError):
        cb.cholinv.inverse_residual(A, Ainv, args, cb.topo.square(1, 0, 1))
