"""The extended-precision references of the batched Jacobi eigensolver without a GPU: the normalised numpy model of syevj.cu at both
ends of the exponent range, the certified gate of syevj_ld_reference on the model's results and against wrong results, and the mpmath
and long-double Rayleigh-Ritz references against each other."""
import numpy as np
import pytest
import syevj_ld_reference as lr
import syevj_reference as sr

DBL_MAX = float(np.finfo(np.float64).max)
U = 2.0 ** -53


def _powers(a):
    """j of 4^j A: largest entry about 2^-1070, near the bottom of the normal range, 1, ||A||_F and ||A||_2 just below DBL_MAX (as
    in tests/test_gpu_syevj_reference.py)"""
    e = int(np.frexp(np.abs(a).max())[1]) - 1
    f, s2 = sr.fro(a), float(np.linalg.norm(a, 2))
    return sorted({(-1070 - e) // 2, (-1020 - e) // 2, 0, int(np.floor((np.log2(DBL_MAX) - np.log2(f)) / 2)),
                   int(np.floor((np.log2(DBL_MAX) - np.log2(s2) - 1e-9) / 2))})


@pytest.mark.parametrize("n", [7, 33, 65])
def test_model_meets_the_bounds_at_the_ends_of_the_range(n):
    """4^j A, j from a largest entry of 2^-1070 to ||A||_2 just below DBL_MAX: info 0, V bit for bit and w = 4^j w of the exactly
    scaled-back matrix, which meets the a-priori bounds.  Without the normalisation the top scalings overflow ||A||_F (n >= 65, random)
    and the bottom ones round every rotation at the subnormal spacing."""
    for i, f in enumerate(("random", "graded", "rankdef", "diagonal")):
        a = sr.family(f, n, 17 * n + i)[0]
        js = _powers(a)
        A = np.stack([np.ldexp(a, 2 * j) for j in js])
        B = np.stack([np.ldexp(x, -2 * j) for x, j in zip(A, js)])
        r, rb = sr.syevj(A), sr.syevj(B)
        assert r["info"].tolist() == [0] * len(js) and rb["info"].tolist() == [0] * len(js)
        assert np.array_equal(r["V"], rb["V"])
        for k, j in enumerate(js):
            assert np.array_equal(r["w"][k], np.ldexp(rb["w"][k], 2 * j)), (f, j)
            chk = sr.check(B[k], rb["w"][k], rb["V"][k])
            assert chk.ok, (f, j, chk)
        if f == "random" and n >= 65:
            assert sr.fro(A[-1]) == np.inf and np.isfinite(np.ldexp(np.linalg.norm(a, 2), 2 * js[-1]))


def test_model_fro_does_not_overflow():
    a = np.diag([DBL_MAX, -DBL_MAX])
    assert sr.fro(a) == np.inf and abs(sr.fro(np.ldexp(a, -2)) / (np.sqrt(2.0) * np.ldexp(DBL_MAX, -2)) - 1) <= 4 * U
    assert sr.scale_power(a) == 511 and sr.scale_power(np.full((2, 2), 2.0 ** -1074)) == -537
    r = sr.syevj(a[None])
    assert r["info"].tolist() == [0] and r["w"][0].tolist() == [-DBL_MAX, DBL_MAX]
    d, x = 0.5 * DBL_MAX, 0.6 * DBL_MAX
    r = sr.syevj(np.array([[[d, x], [x, -d]]]))
    assert r["info"].tolist() == [0] and abs(r["w"][0][1] / DBL_MAX - np.hypot(0.5, 0.6)) <= 8 * U


@pytest.mark.parametrize("n", [7, 33, 65])
def test_certified_gate_holds_on_the_model(n):
    for i, f in enumerate(sr.FAMILIES):
        a = sr.family(f, n, 1000 * n + i)[0]
        r = sr.syevj(a[None])
        c = lr.certify(a, r["w"][0], r["V"][0])
        assert c.ok, (f, c)


def test_certified_gate_rejects_wrong_results():
    # one eigenvalue moved by 4 x the largest certified bound the gate accepts.  The certified bound holds for every (w, V), so a move
    # is caught by the requirement that the bound stay within that limit, not by the comparison with the reference.
    n = 33
    a = sr.family("random", n, 77)[0]
    r = sr.syevj(a[None])
    w, V = r["w"][0], r["V"][0]
    ref = lr.reference(a)
    c = lr.certify(a, w, V, ref)
    assert c.ok, c
    wm = w.copy()
    wm[n // 2] += 4 * c.apriori[0]
    assert not lr.certify(a, wm, V, ref).ok
    # two eigenvalues swapped inside a 1e-12 cluster, with their vectors
    a = sr.family("cluster", n, 78)[0]
    r = sr.syevj(a[None])
    w, V = r["w"][0], r["V"][0]
    ref = lr.reference(a)
    assert lr.certify(a, w, V, ref).ok
    i, j = n - 3, n - 1
    assert w[i] != w[j] and abs(w[i] - w[j]) < 1e-11
    ws, Vs = w.copy(), V.copy()
    ws[[i, j]], Vs[:, [i, j]] = ws[[j, i]], Vs[:, [j, i]]
    assert not lr.certify(a, ws, Vs, ref).ok
    # the iterate one outer step before the first one the bounds accept
    n = 65
    a = sr.family("random", n, 77)[0]
    r = sr.syevj(a[None], snapshots=True)
    ref = lr.reference(a)
    ok = [sr.check(a, w_[0], V_[0]).ok for w_, V_ in r["steps"]]
    first = next(k for k in range(len(ok)) if all(ok[k:]))
    assert 0 < first
    assert lr.certify(a, r["steps"][first][0][0], r["steps"][first][1][0], ref).ok
    assert not lr.certify(a, r["steps"][first - 1][0][0], r["steps"][first - 1][1][0], ref).ok


@pytest.mark.parametrize("f,n", [("random", 7), ("cluster", 33), ("repeated", 33), ("graded", 64)])
def test_mpmath_and_rayleigh_ritz_references_agree(f, n):
    a = sr.family(f, n, 5 * n)[0]
    m, rr = lr.mp_reference(a), lr.rr_reference(a)
    known = np.isfinite(rr.err)
    assert known.all() or rr.traces
    assert (np.abs(m.lam - rr.lam).astype(float)[known] <= (m.err + rr.err)[known]).all()
    for c, t, e in rr.traces:
        assert abs(float(np.sum(m.lam[c]) - t)) <= e + float(np.sum(m.err[c]))
    # and a small block forced through the trace and through mpmath
    rt = lr.rr_reference(a, mp_block=1)
    for c, t, e in rt.traces:
        assert abs(float(np.sum(m.lam[c]) - t)) <= e + float(np.sum(m.err[c]))
