"""cholinv::solve without a GPU: the numpy block formula against scipy, and the argument checks of the C ABI and of the Python mirror
(they must reject bad input before any device call)."""
import ctypes as C
import numpy as np
import pytest
import scipy.linalg as sla
import torch
import capital_b200 as cb
from capital_b200 import _lib
from oracle import capital_oracle as co
from solve_reference import cholesky_solve, top_split


@pytest.mark.parametrize("n", [96, 128, 200])
@pytest.mark.parametrize("d", [1, 2])
@pytest.mark.parametrize("split", [1, 2])
@pytest.mark.parametrize("ci", [0, 1])
def test_block_solve_matches_cho_solve(n, d, split, ci):
    a = co.spd_global(n)
    bc = co.bc_dimension(n // d, d, d, -2)
    r, ri = co.cholinv(a, bool(ci), split, bc, d=d)
    if not ci:
        n1 = top_split(n, False, split, bc, d)
        assert n1 is not None and np.count_nonzero(ri[:n1, n1:]) == 0  # the skipped block really is missing
    b = np.random.default_rng(n + 7 * d + split).standard_normal((n, 5))
    x = cholesky_solve(r, ri, b, bool(ci), split, bc, d)
    ref = sla.cho_solve((sla.cholesky(a), False), b)
    assert np.abs(x - ref).max() <= 1e-13 * np.abs(ref).max()


def test_top_level_base_case_has_no_skipped_block():
    n = 128
    a = co.spd_global(n)
    bc = co.bc_dimension(n, 1, 1, 0)  # bc_mult_dim >= 0: the whole matrix is the base case
    assert top_split(n, False, 1, bc) is None
    r, ri = co.cholinv(a, False, 1, bc)
    b = np.ones((n, 2))
    assert np.abs(cholesky_solve(r, ri, b, False, 1, bc) - np.linalg.solve(a, b)).max() < 1e-12


def test_c_abi_rejects_a_null_context():
    args = _lib.CholinvArgs(1, 1, -1, b"U")
    x = (C.c_double * 4)()
    assert _lib.lib().capital_cholinv_solve_f64(None, 4, C.byref(args), _lib.UPPERTRI_PACKED, None, x, 1, x, 4, x, 4) == _lib.ERR_INVALID


def _factored_info(n):
    args = cb.cholinv.info(1, 1, -1, "U")
    args.R = torch.zeros(n * (n + 1) // 2, dtype=torch.float64)
    args.Rinv = torch.zeros_like(args.R)
    args.local_dim = args.global_dim = n
    return args


def test_python_solve_rejects_an_unfactored_info():
    with pytest.raises(ValueError):
        cb.cholinv.solve(cb.cholinv.info(1, 1, -1, "U"), torch.zeros(8, dtype=torch.float64), cb.topo.square(1, 0, 1))


@pytest.mark.parametrize("shape", [(7,), (9, 2), (8, 0), (8, 2, 1)])
def test_python_solve_rejects_wrong_rows(shape):
    with pytest.raises(ValueError):
        cb.cholinv.solve(_factored_info(8), torch.zeros(shape, dtype=torch.float64), cb.topo.square(1, 0, 1))


@pytest.mark.parametrize("dtype", [torch.float32, torch.int64])
def test_python_solve_rejects_non_float64(dtype):
    with pytest.raises(ValueError):
        cb.cholinv.solve(_factored_info(8), torch.zeros(8, 2, dtype=dtype), cb.topo.square(1, 0, 1))
