"""cacqr::apply_QT / apply_Q / lstsq without a GPU: the argument checks of the C ABI and of the Python mirror (they must reject bad
input before any device call)."""
import ctypes as C
import pytest
import torch
import capital_b200 as cb
from capital_b200 import _lib


def test_c_abi_rejects_a_null_context():
    x = (C.c_double * 64)()
    L = _lib.lib()
    assert L.capital_cacqr_apply_qt_f64(None, 8, 4, x, 1, x, 8, x, 4) == _lib.ERR_INVALID
    assert L.capital_cacqr_apply_q_f64(None, 8, 4, x, 1, x, 4, x, 8) == _lib.ERR_INVALID
    assert L.capital_cacqr_lstsq_f64(None, 8, 4, x, _lib.UPPERTRI_PACKED, x, 1, x, 8, x, 4) == _lib.ERR_INVALID


def _factored_info(m=10, n=4, serialize=True):
    args = cb.cacqr.info(2, cb.cholinv.info(0, 1, 0, "U"), serialize=serialize)
    args.Q = torch.zeros(m * n, dtype=torch.float64)
    args.R = torch.zeros(n * (n + 1) // 2 if serialize else n * n, dtype=torch.float64)
    args.n, args.rows_local, args.m_global, args.n_global = n, m, m, n
    return args


def _calls(args, T):
    topo = cb.topo.rect(1, 0, 1)
    return [lambda: cb.cacqr.apply_QT(T, args, topo), lambda: cb.cacqr.apply_Q(T, args, topo), lambda: cb.cacqr.lstsq(args, T, topo)]


def test_python_mirrors_reject_an_unfactored_info():
    for call in _calls(cb.cacqr.info(2, cb.cholinv.info(0, 1, 0, "U")), torch.zeros(10, 2, dtype=torch.float64)):
        with pytest.raises(ValueError):
            call()


@pytest.mark.parametrize("shape", [(7,), (11, 2), (10, 0), (4, 0), (10, 2, 1), (4, 2, 1), ()])
def test_python_mirrors_reject_wrong_shapes(shape):
    # rows_local = 10 for B (apply_QT, lstsq), n = 4 for Z (apply_Q): none of these shapes fits its call
    for call in _calls(_factored_info(), torch.zeros(shape, dtype=torch.float64)):
        with pytest.raises(ValueError):
            call()


def test_python_mirrors_reject_a_right_hand_side_of_the_other_height():
    args, topo = _factored_info(), cb.topo.rect(1, 0, 1)
    with pytest.raises(ValueError):
        cb.cacqr.apply_QT(torch.zeros(4, 2, dtype=torch.float64), args, topo)
    with pytest.raises(ValueError):
        cb.cacqr.lstsq(args, torch.zeros(4, 2, dtype=torch.float64), topo)
    with pytest.raises(ValueError):
        cb.cacqr.apply_Q(torch.zeros(10, 2, dtype=torch.float64), args, topo)


@pytest.mark.parametrize("dtype", [torch.float32, torch.int64, torch.complex128])
def test_python_mirrors_reject_non_float64(dtype):
    args = _factored_info()
    topo = cb.topo.rect(1, 0, 1)
    with pytest.raises(ValueError):
        cb.cacqr.apply_QT(torch.zeros(10, 2, dtype=dtype), args, topo)
    with pytest.raises(ValueError):
        cb.cacqr.lstsq(args, torch.zeros(10, 2, dtype=dtype), topo)
    with pytest.raises(ValueError):
        cb.cacqr.apply_Q(torch.zeros(4, 2, dtype=dtype), args, topo)


def test_python_lstsq_rejects_an_R_of_the_wrong_size():
    args = _factored_info()
    args.R = torch.zeros(3, dtype=torch.float64)
    with pytest.raises(ValueError):
        cb.cacqr.lstsq(args, torch.zeros(10, 2, dtype=torch.float64), cb.topo.rect(1, 0, 1))


def test_python_mirrors_reject_non_tensors():
    for call in _calls(_factored_info(), [[0.0] * 2] * 10):
        with pytest.raises(ValueError):
            call()
