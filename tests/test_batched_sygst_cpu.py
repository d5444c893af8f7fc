"""Batched inverse, sygst, products with the factors and eigh_batched without a GPU: the C entry points reject a NULL context, the Python
wrappers reject every malformed input with ValueError before any device call (their device check comes last, so host tensors exercise
all the others), the chunk rule, and the bounds of batched_sygst_reference against wrong results."""
import numpy as np
import pytest
import torch
import capital_b200 as cb
from capital_b200 import _lib
import batched_sygst_reference as bs


def test_entry_points_reject_a_null_context():
    L = _lib.lib()
    assert L.capital_cholinv_inverse_batched_f64(None, 8, 2, None, None) == _lib.ERR_INVALID
    assert L.capital_cholinv_sygst_batched_f64(None, 8, 2, None, None, None) == _lib.ERR_INVALID
    assert L.capital_cholinv_sygst_ab_batched_f64(None, 8, 2, None, None, None) == _lib.ERR_INVALID
    assert L.capital_cholinv_apply_rinv_batched_f64(None, 8, 2, None, 0, 1, None, None) == _lib.ERR_INVALID
    assert L.capital_cholinv_apply_r_batched_f64(None, 8, 2, None, 1, 1, None, None) == _lib.ERR_INVALID


def _eye(b, n, dtype=torch.float64):
    return torch.eye(n, dtype=dtype).expand(b, n, n).clone()


F64 = torch.float64


@pytest.mark.parametrize("Rinv,what", [
    (_eye(2, 8, torch.float32), "float64"),
    (_eye(2, 8).numpy(), "float64"),
    (torch.eye(8, dtype=F64), "shape"),
    (torch.zeros(0, 8, 8, dtype=F64), "shape"),
    (torch.zeros(2, 8, 7, dtype=F64), "shape"),
    (_eye(1, 513), "513 > 512"),
    (_eye(2, 8), "CUDA"),
])
def test_inverse_batched_rejects(Rinv, what):
    with pytest.raises(ValueError, match=what):
        cb.cholinv.inverse_batched(Rinv, None)


@pytest.mark.parametrize("A,R,Rinv,itype,what", [
    (_eye(2, 8, torch.float32), _eye(2, 8), _eye(2, 8), 1, "A must be a float64"),
    (_eye(2, 8), _eye(2, 8, torch.float32), _eye(2, 8), 2, "R must be a float64"),
    (_eye(2, 8), _eye(2, 8), _eye(2, 8).numpy(), 1, "Rinv must be a float64"),
    (torch.eye(8, dtype=F64), _eye(2, 8), _eye(2, 8), 1, "A has shape"),
    (_eye(2, 8), torch.zeros(2, 8, 8, 1, dtype=F64), None, 2, "R has shape"),
    (torch.zeros(2, 8, 7, dtype=F64), _eye(2, 8), _eye(2, 8), 1, "A must have shape"),
    (_eye(2, 8), _eye(3, 8), _eye(2, 8), 1, r"R must have shape \(2, 8, 8\)"),
    (_eye(2, 8), _eye(2, 8), _eye(2, 9), 1, r"Rinv must have shape \(2, 8, 8\)"),
    (_eye(1, 513), _eye(1, 513), _eye(1, 513), 1, "513 > 512"),
    (_eye(2, 8), _eye(2, 8), _eye(2, 8), 0, "itype must be 1, 2 or 3"),
    (_eye(2, 8), _eye(2, 8), _eye(2, 8), 4, "itype must be 1, 2 or 3"),
    (_eye(2, 8), _eye(2, 8), _eye(2, 8), True, "itype must be 1, 2 or 3"),
    (_eye(2, 8), _eye(2, 8), _eye(2, 8), 1.0 + 1e-9, "itype must be 1, 2 or 3"),
    (_eye(2, 8), _eye(2, 8), None, 1, "itype 1 reads Rinv, which is None"),
    (_eye(2, 8), None, _eye(2, 8), 3, "itype 3 reads R, which is None"),
    (_eye(2, 8), _eye(2, 8), _eye(2, 8), 1, "CUDA"),
    (_eye(2, 8), _eye(2, 8), None, 2, "CUDA"),
])
def test_sygst_batched_rejects(A, R, Rinv, itype, what):
    with pytest.raises(ValueError, match=what):
        cb.cholinv.sygst_batched(A, R, Rinv, None, itype=itype)


APPLY = [cb.cholinv.apply_Rinv_batched, cb.cholinv.apply_RinvT_batched, cb.cholinv.apply_R_batched, cb.cholinv.apply_RT_batched]


@pytest.mark.parametrize("fn", APPLY, ids=lambda f: f.__name__)
@pytest.mark.parametrize("F,B,what", [
    (_eye(2, 8, torch.float32), torch.zeros(2, 8, dtype=F64), "must be a float64"),
    (_eye(2, 8), torch.zeros(2, 8, dtype=torch.float32), "B must be a float64"),
    (torch.eye(8, dtype=F64), torch.zeros(2, 8, dtype=F64), "has shape"),
    (_eye(2, 8), torch.zeros(16, dtype=F64), "B has shape"),
    (_eye(2, 8), torch.zeros(2, 8, 1, 1, dtype=F64), "B has shape"),
    (torch.zeros(2, 8, 7, dtype=F64), torch.zeros(2, 8, dtype=F64), r"must have shape \(b, n, n\)"),
    (_eye(2, 8), torch.zeros(3, 8, dtype=F64), "B must have shape"),
    (_eye(2, 8), torch.zeros(2, 9, 4, dtype=F64), "B must have shape"),
    (_eye(1, 513), torch.zeros(1, 513, dtype=F64), "513 > 512"),
    (_eye(2, 8), torch.zeros(2, 8, 3, dtype=F64), "CUDA"),
])
def test_apply_batched_rejects(fn, F, B, what):
    with pytest.raises(ValueError, match=what):
        fn(F, B, None)


@pytest.mark.parametrize("A,B,itype,what", [
    (_eye(2, 8, torch.float32), _eye(2, 8), 1, "A must be a float64"),
    (_eye(2, 8), _eye(2, 8).numpy(), 1, "B must be a float64"),
    (torch.eye(8, dtype=F64), _eye(2, 8), 1, "A has shape"),
    (_eye(2, 8), torch.zeros(2, 8, dtype=F64), 1, "B has shape"),
    (torch.zeros(2, 8, 7, dtype=F64), _eye(2, 8), 1, "A must have shape"),
    (_eye(2, 8), _eye(3, 8), 1, r"B must have shape \(2, 8, 8\)"),
    (_eye(2, 8), _eye(2, 7), 1, r"B must have shape \(2, 8, 8\)"),
    (_eye(1, 513), _eye(1, 513), 1, "513 > 512"),
    (_eye(2, 8), _eye(2, 8), False, "itype must be 1, 2 or 3"),
    (_eye(2, 8), _eye(2, 8), "1", "itype must be 1, 2 or 3"),
    (_eye(2, 8), _eye(2, 8), 2, "CUDA"),
])
def test_eigh_batched_rejects(A, B, itype, what):
    with pytest.raises(ValueError, match=what):
        cb.cholinv.eigh_batched(A, B, None, itype=itype)


@pytest.mark.parametrize("n,call,expect", [
    (512, "inverse", 341), (512, "sygst", 256), (512, "sygst_ab", 256), (512, "apply_rinv", 8192), (512, "apply_r", 8192),
    (8, "inverse", 65535), (8, "sygst", 65535), (8, "apply_r", 65535), (17, "sygst", 65535),
    (256, "inverse", 1365), (255, "sygst", 1028), (1, "apply_rinv", 65535),
])
def test_chunk_rule(n, call, expect):
    """matrices per chunk: the 2 GiB cap over the bytes per matrix, at most 65535 (grid z)"""
    assert bs.chunk(call, n, 10 ** 6) == expect
    assert bs.chunk(call, n, 3) == 3
    ld = (n + 15) // 16 * 16
    per = {"inverse": 3 * ld * n, "sygst": 4 * ld * n, "sygst_ab": 4 * ld * n}.get(call, (n + (n + 63) // 64 * 64) * 32) * 8
    assert expect * per <= 2 << 30 and (expect == 65535 or (expect + 1) * per > 2 << 30)


@pytest.mark.parametrize("itype", [1, 2, 3])
@pytest.mark.parametrize("n", [1, 9, 40])
def test_product_bound_rejects_wrong_results(n, itype):
    """the bound the GPU tests gate on holds for the FP64 product and fails for one that drops a class, returns 0 or -C"""
    from batched_reference import chol_ld
    g = np.random.default_rng(n + 10 * itype)
    for kappa in (10.0, 1e8):
        b = bs.spd_spectrum(n, kappa, 7 * n + itype).numpy()
        a = g.standard_normal((n, n))
        a = a + a.T
        r = np.triu(chol_ld(b)[0].astype(np.float64))
        f = np.linalg.inv(r) if itype == 1 else r
        ref = bs.sygst_ld(a, f, itype)
        bound = bs.product_bound(a, f)
        fp = f.T @ (a @ f) if itype == 1 else f @ (a @ f.T)
        assert float(np.linalg.norm((fp - ref).astype(np.float64))) <= bound
        half = bs.sygst_half(a, f, itype)
        for wrong in (half, half.T, np.zeros_like(ref), -ref):
            assert float(np.linalg.norm((wrong - ref).astype(np.float64))) > bound
    ri = np.linalg.inv(r)
    assert float(np.linalg.norm((ri @ ri.T - bs.inverse_ld(ri)).astype(np.float64))) <= bs.inverse_product_bound(ri)
    assert float(np.linalg.norm(bs.inverse_ld(ri).astype(np.float64))) > bs.inverse_product_bound(ri)


@pytest.mark.parametrize("itype", [1, 2, 3])
def test_eigh_bounds_hold_for_scipy(itype):
    """the eigh bounds are met by LAPACK's own generalized eigh on the same pencils"""
    import scipy.linalg as sl
    for n in (1, 17, 64):
        for kappa in (10.0, 1e4):
            b = bs.spd_spectrum(n, kappa, n + 3).numpy()
            g = np.random.default_rng(n)
            a = g.standard_normal((n, n))
            a = a + a.T
            w, x = sl.eigh(a, b, type=itype)
            eb = bs.EighBounds(a, b, itype)
            assert bs.eigh_residual(a, b, w, x, itype) <= eb.residual(w, x)
            assert bs.eigh_orthonormality(b, x, itype) <= eb.orthonormality()
            assert bs.eigh_orthonormality(b, 1.001 * x, itype) > eb.orthonormality()
