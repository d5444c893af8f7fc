"""Batched CholInv without a GPU: the C entry points reject a NULL context, and the Python wrappers reject every malformed input with
ValueError before any device call (their device check comes last, so host tensors exercise all the others)."""
import pytest
import torch
import capital_b200 as cb
from capital_b200 import _lib


def test_entry_points_reject_a_null_context():
    L = _lib.lib()
    assert L.capital_cholinv_factor_batched_f64(None, 8, 2, None, None, None, None) == _lib.ERR_INVALID
    assert L.capital_cholinv_solve_batched_f64(None, 8, 2, None, 1, None, None) == _lib.ERR_INVALID


def _spd(b, n, dtype=torch.float64):
    return torch.eye(n, dtype=dtype).expand(b, n, n).clone()


@pytest.mark.parametrize("A,what", [
    (_spd(2, 8, torch.float32), "float64"),
    (_spd(2, 8).numpy(), "float64"),
    (torch.eye(8, dtype=torch.float64), "shape"),
    (torch.zeros(2, 8, 8, 1, dtype=torch.float64), "shape"),
    (torch.zeros(0, 8, 8, dtype=torch.float64), "shape"),
    (torch.zeros(2, 8, 7, dtype=torch.float64), "shape"),
    (_spd(1, 513), "513 > 512"),
    (_spd(2, 8), "CUDA"),
])
def test_factor_batched_rejects(A, what):
    with pytest.raises(ValueError, match=what):
        cb.cholinv.factor_batched(A, None)


@pytest.mark.parametrize("Rinv,B,what", [
    (_spd(2, 8, torch.float32), torch.zeros(2, 8, dtype=torch.float64), "Rinv must be a float64"),
    (_spd(2, 8), torch.zeros(2, 8, dtype=torch.float32), "B must be a float64"),
    (torch.eye(8, dtype=torch.float64), torch.zeros(2, 8, dtype=torch.float64), "Rinv has shape"),
    (_spd(2, 8), torch.zeros(16, dtype=torch.float64), "B has shape"),
    (_spd(2, 8), torch.zeros(2, 8, 1, 1, dtype=torch.float64), "B has shape"),
    (torch.zeros(2, 8, 7, dtype=torch.float64), torch.zeros(2, 8, dtype=torch.float64), "Rinv must have shape"),
    (_spd(2, 8), torch.zeros(3, 8, dtype=torch.float64), "B must have shape"),
    (_spd(2, 8), torch.zeros(2, 9, 4, dtype=torch.float64), "B must have shape"),
    (_spd(1, 513), torch.zeros(1, 513, dtype=torch.float64), "513 > 512"),
    (_spd(2, 8), torch.zeros(2, 8, 3, dtype=torch.float64), "CUDA"),
])
def test_solve_batched_rejects(Rinv, B, what):
    with pytest.raises(ValueError, match=what):
        cb.cholinv.solve_batched(Rinv, B, None)
