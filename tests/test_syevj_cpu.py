"""The batched Jacobi eigensolver without a GPU: the circle-method pairing, the padding invariant, convergence of the schedule's numpy
model (syevj_reference) on every test family, the accuracy bounds the GPU tests gate on against wrong results, and the rejections of
capital_syevj_batched_f64, eig.syevj_batched and eigh_batched's eigensolver keyword (all before any device call)."""
import itertools
import numpy as np
import pytest
import torch
import capital_b200 as cb
from capital_b200 import _lib
import syevj_reference as sr

F64 = torch.float64


@pytest.mark.parametrize("m", sorted({np_ // 32 for np_ in range(64, 513, 64)} | {2, 8, 34, 64}))
def test_pairing_covers_every_pair_once_per_sweep(m):
    """every step pairs all m players (disjoint pairs), and every unordered pair comes up exactly once in the m - 1 steps: the blocks
    N = Np / 32 of every n <= 512 and the inner orders"""
    seen = []
    for s in range(m - 1):
        pairs = sr.pairing(m, s)
        assert len(pairs) == m // 2 and all(p < q for p, q in pairs)
        assert sorted(i for pq in pairs for i in pq) == list(range(m))
        seen += pairs
    assert sorted(seen) == list(itertools.combinations(range(m), 2))


@pytest.mark.parametrize("n", [33, 100])
def test_padding_stays_exactly_decoupled(n):
    """pad rows and columns of the iterate stay exactly zero off the diagonal, pad eigenvectors exactly unit vectors, and the real
    eigenvectors exactly zero in the pad rows (rank-deficient input: zero eigenvalues beside the zero pad)"""
    a = np.stack([sr.family("rankdef", n, 3)[0], sr.family("random", n, 4)[0]])
    r = sr.syevj(a)
    assert r["info"].tolist() == [0, 0]
    Aw, Vw = r["Aw"], r["Vw"]
    m = Aw.shape[1]
    assert m > n
    assert not Aw[:, :n, n:].any() and not Aw[:, n:, :n].any()
    assert np.array_equal(Vw[:, n:, :n], np.zeros((2, m - n, n))) and not Vw[:, :n, n:].any()
    assert np.array_equal(Vw[:, n:, n:], np.tile(np.eye(m - n), (2, 1, 1)))
    assert np.array_equal(Aw[:, n:, n:], np.zeros((2, m - n, m - n)))


# The test prints the sweeps the model needs per family (pytest -s): for n <= 64 the sweeps of the one-CTA solver, for n > 64 the outer
# sweeps, each including the final sweep without a rotation.  At n = 7: random 6, cluster 7, repeated 1, rankdef 6, negdef 6, graded 6,
# diagonal 1, zero 1.
@pytest.mark.parametrize("n", [7, 33, 64, 100, 256])
def test_model_converges_on_every_family(n):
    mats = [sr.family(f, n, 1000 * n + i)[0] for i, f in enumerate(sr.FAMILIES)]
    r = sr.syevj(np.stack(mats))
    print(n, dict(zip(sr.FAMILIES, r["sweeps"].tolist())))
    assert r["info"].tolist() == [0] * len(mats)
    assert (r["sweeps"] <= sr.SWEEPS).all()
    assert r["sweeps"][sr.FAMILIES.index("diagonal")] == 1 and r["sweeps"][sr.FAMILIES.index("zero")] == 1
    for i, f in enumerate(sr.FAMILIES):
        chk = sr.check(mats[i], r["w"][i], r["V"][i])
        assert chk.ok, (f, chk)
        assert sr.vectors_ok(mats[i], r["w"][i], r["V"][i]), f


@pytest.mark.parametrize("n", [33, 65])
def test_bounds_reject_wrong_results(n):
    a = sr.family("random", n, 77)[0]
    r = sr.syevj(a[None], snapshots=True)
    w, V = r["w"][0], r["V"][0]
    assert sr.check(a, w, V).ok
    Vs = V.copy()
    Vs[:, [3, 7]] = Vs[:, [7, 3]]
    assert not sr.check(a, w, Vs).ok                      # two eigenvectors swapped
    assert not sr.check(a, w[::-1], V[:, ::-1]).ok        # consistent pairs, descending order
    assert not sr.check(a, w, np.eye(n)).ok               # V = I
    if n > 64:
        # the iterate after every outer step: once it meets the bounds it keeps meeting them, and the one before is rejected
        ok = [sr.check(a, w_[0], V_[0]).ok for w_, V_ in r["steps"]]
        first = next(k for k in range(len(ok)) if all(ok[k:]))
        assert 0 < first < len(ok) - 1 and not ok[first - 1], ok


def test_chunk_rule():
    assert sr.chunk(512, 10 ** 6) == 481 and sr.chunk(512, 100) == 100
    assert sr.chunk(64, 10 ** 6) == 65535 and sr.chunk(65, 10 ** 6) == 2 ** 31 // ((2 * 128 * 128 + 2 * 4096) * 8)


def test_entry_point_rejects_a_null_context():
    assert _lib.lib().capital_syevj_batched_f64(None, 8, 2, None, None, None, None) == _lib.ERR_INVALID


def _eye(b, n, dtype=F64):
    return torch.eye(n, dtype=dtype).expand(b, n, n).clone()


@pytest.mark.parametrize("A,what", [
    (_eye(2, 8, torch.float32), "float64"),
    (_eye(2, 8).numpy(), "float64"),
    (torch.eye(8, dtype=F64), "shape"),
    (torch.zeros(0, 8, 8, dtype=F64), "shape"),
    (torch.zeros(2, 8, 7, dtype=F64), "shape"),
    (torch.zeros(2, 8, 8, 1, dtype=F64), "shape"),
    (_eye(1, 513), "513 > 512"),
    (_eye(2, 8), "CUDA"),
])
def test_syevj_batched_rejects(A, what):
    with pytest.raises(ValueError, match=what):
        cb.eig.syevj_batched(A, None)


@pytest.mark.parametrize("solver,what", [
    ("x", "eigensolver must be"), ("Jacobi", "eigensolver must be"), (None, "eigensolver must be"), (1, "eigensolver must be"),
    ("jacobi", "CUDA"), ("torch", "CUDA"),
])
def test_eigh_batched_rejects_eigensolver(solver, what):
    with pytest.raises(ValueError, match=what):
        cb.cholinv.eigh_batched(_eye(2, 8), _eye(2, 8), None, eigensolver=solver)
