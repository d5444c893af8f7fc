"""Batched CholeskyQR without a GPU: the C entry points reject a NULL context, and the Python wrappers reject every malformed input
with ValueError before any device call (their device check comes last, so host tensors exercise all the others)."""
import pytest
import torch
import capital_b200 as cb
from capital_b200 import _lib


def test_entry_points_reject_a_null_context():
    L = _lib.lib()
    assert L.capital_cacqr_factor_batched_f64(None, 16, 8, 2, 2, None, None, None, None) == _lib.ERR_INVALID
    assert L.capital_cacqr_lstsq_batched_f64(None, 16, 8, 2, None, None, 1, None, None) == _lib.ERR_INVALID


def _f64(*shape):
    return torch.zeros(*shape, dtype=torch.float64)


@pytest.mark.parametrize("A,kw,what", [
    (torch.zeros(2, 16, 8, dtype=torch.float32), {}, "float64"),
    (_f64(2, 16, 8).numpy(), {}, "float64"),
    (_f64(16, 8), {}, "shape"),
    (_f64(2, 16, 8, 1), {}, "shape"),
    (_f64(0, 16, 8), {}, "shape"),
    (_f64(2, 16, 8), {"num_iter": 0}, "num_iter"),
    (_f64(2, 16, 8), {"num_iter": 4}, "num_iter"),
    (_f64(1, 600, 513), {}, "513 > 512"),
    (_f64(2, 7, 8), {}, "m = 7 < n = 8"),
    (_f64(2, 16, 8), {}, "CUDA"),
])
def test_factor_batched_rejects(A, kw, what):
    with pytest.raises(ValueError, match=what):
        cb.cacqr.factor_batched(A, None, **kw)


@pytest.mark.parametrize("Q,R,B,what", [
    (torch.zeros(2, 16, 8, dtype=torch.float32), _f64(2, 8, 8), _f64(2, 16), "Q must be a float64"),
    (_f64(2, 16, 8), torch.zeros(2, 8, 8, dtype=torch.float32), _f64(2, 16), "R must be a float64"),
    (_f64(2, 16, 8), _f64(2, 8, 8), torch.zeros(2, 16, dtype=torch.float32), "B must be a float64"),
    (_f64(16, 8), _f64(2, 8, 8), _f64(2, 16), "Q has shape"),
    (_f64(2, 16, 8), _f64(8, 8), _f64(2, 16), "R has shape"),
    (_f64(2, 16, 8), _f64(2, 8, 8), _f64(32), "B has shape"),
    (_f64(2, 16, 8), _f64(2, 8, 8), _f64(2, 16, 1, 1), "B has shape"),
    (_f64(2, 16, 8), _f64(3, 8, 8), _f64(2, 16), "R must have shape"),
    (_f64(2, 16, 8), _f64(2, 8, 7), _f64(2, 16), "R must have shape"),
    (_f64(2, 16, 8), _f64(2, 8, 8), _f64(3, 16), "B must have shape"),
    (_f64(2, 16, 8), _f64(2, 8, 8), _f64(2, 15, 4), "B must have shape"),
    (_f64(1, 600, 513), _f64(1, 513, 513), _f64(1, 600), "513 > 512"),
    (_f64(2, 7, 8), _f64(2, 8, 8), _f64(2, 7), "m = 7 < n = 8"),
    (_f64(2, 16, 8), _f64(2, 8, 8), _f64(2, 16, 3), "CUDA"),
])
def test_lstsq_batched_rejects(Q, R, B, what):
    with pytest.raises(ValueError, match=what):
        cb.cacqr.lstsq_batched(Q, R, B, None)
