"""What the grid edge tests share (numpy only): the case tables, the extended-precision reference and the error bounds.

tests/test_grid_edges_cpu.py replays the schedule of these cases on the CPU and tests/mp_worker_grid_edges.py runs them on the GPU;
both take sizes and knob sets from here, so a case the GPU runs is a case the replay has seen."""
import numpy as np

from oracle import capital_oracle as co

U = 2.0 ** -53  # unit roundoff of FP64

GRIDS = {2: (2, 1), 4: (1, 2), 8: (2, 2)}  # ranks -> (c, d)

# d = 2 (local size L = n / 2): L = 501 and 695 are odd (ld = 512, 704), 648 is a multiple of 8 but not of 16, 513 is one past 512;
# 1024 is the aligned control.  d = 1: L = n.
SIZES = {2: (1002, 1390, 1296, 1026, 1024), 1: (777, 1001, 1024)}
ODD_SIZES = {2: (1002, 1390), 1: (777, 1001)}

_LOW = {"CAPITAL_DIST_FAR_MIN": "64", "CAPITAL_DIST_SIDE_MIN": "32", "CAPITAL_DIST_CHUNK_MIN": "128"}
KNOBS = {
    "default": {},
    "low": _LOW,                                          # deferred classes and chunked, pushed products at L ~ 500
    "low3": dict(_LOW, CAPITAL_DIST_CHUNKS="3"),           # three chunks: other chunk widths (at the larger odd size only, see cases)
    "pipe": dict(_LOW, CAPITAL_DIST_PIPELINE="1"),         # chunk j + 1 issued before chunk j is added up
    "nobulk": dict(_LOW, CAPITAL_DIST_BULK="0"),           # node-entry pushes on the chain's push stream
    # no deferred streams at all; with the default CHUNK_MIN this is the default schedule at these sizes, so the chunks stay
    "one": {"CAPITAL_DIST_TWO_STREAM": "0", "CAPITAL_DIST_CHUNK_MIN": "128"},
}
KNOB_NAMES = sorted({k for env in KNOBS.values() for k in env})


# Knob sets beyond default / low that change the schedule of a grid (tests/test_grid_edges_cpu.py asserts that each one does).  With
# d = 1 nothing is pushed, so nothing is chunked, there is no bulk class, and `one` is the default schedule below L = 1024; the pipeline reorders the depth exchange, which needs c > 1.
EXTRA_KNOBS = {2: (), 4: ("nobulk", "one"), 8: ("pipe", "nobulk", "one")}


def cases(size, sizes=None):
    """(n, complete_inv, split, bc_mult_dim, serialize, knob set) of every factorization on the grid of `size` ranks, the `default`
    one of each (n, ci, split, bc, serialize) first.  `sizes` restricts the table to those n."""
    d = GRIDS[size][1]
    out = []
    odd = ODD_SIZES[d]
    for n in (odd if size == 8 else SIZES[d]):  # eight ranks time-slicing one GPU take seconds per factorization: the odd sizes only
        for ci in (0, 1):
            for split in (1, 2):
                for knob in ("default", "low"):
                    out.append((n, ci, split, -3, True, knob))
    for n in odd:
        for ci, split in ((0, 2), (1, 1)):
            # at L ~ 500 three and four chunks cut every block into the same 128-wide chunks: low3 only where it differs from low
            for knob in EXTRA_KNOBS[size] + (("low3",) if d > 1 and n == odd[1] else ()):
                out.append((n, ci, split, -3, True, knob))
            for bcm, serialize in ((-2, True), (-3, False)):
                for knob in ("default", "low"):
                    out.append((n, ci, split, bcm, serialize, knob))
    return [c for c in out if sizes is None or c[0] in sizes]


def case_id(n, ci, split, bcm, serialize, knob):
    return f"n={n} ci={ci} split={split} bc={bcm} {'packed' if serialize else 'rect'} {knob}"


def chol_ld(a):
    """(R, Rinv, R64, Rinv64): the upper Cholesky factor of a (A = R^T R) and its inverse computed row by row in np.longdouble, and
    their float64 roundings.  np.linalg.cholesky and the oracle work in float64 and so share the kernels' rounding error; this does
    not (u = 2^-64 where long double is the x87 format)."""
    n = a.shape[0]
    w = np.asarray(a, dtype=np.longdouble)
    r = np.zeros((n, n), dtype=np.longdouble)
    for i in range(n):
        v = w[i, i:] - r[:i, i] @ r[:i, i:]
        r[i, i] = np.sqrt(v[0])
        r[i, i + 1:] = v[1:] / r[i, i]
    ri = np.zeros((n, n), dtype=np.longdouble)
    for i in range(n - 1, -1, -1):  # row i of R X = I
        ri[i, i:] = -(r[i, i + 1:] @ ri[i + 1:, i:]) / r[i, i]
        ri[i, i] += 1 / r[i, i]
    return r, ri, r.astype(np.float64), ri.astype(np.float64)


def assemble(parts, coords, n, d, serialize):
    """global matrix from the layer-0 local blocks: rect blocks as they are, packed ones through their (global) upper triangle"""
    L = n // d
    a = np.zeros((n, n))
    for part, (x, y, z) in zip(parts, coords):
        if z != 0:
            continue
        loc = co.unpack_upper(part, L) if serialize else part.reshape(L, L).T
        gy, gx = np.meshgrid(y + d * np.arange(L), x + d * np.arange(L), indexing="ij")
        keep = np.ones_like(loc, dtype=bool) if not serialize else gy <= gx
        a[gy[keep], gx[keep]] = loc[keep]
    if serialize:
        a = np.triu(a) + np.triu(a, 1).T
    return a


class Bounds:
    """A-priori rounding bounds of CholInv on the SPD matrix a, from its measured 2-norm and condition number.

    Every entry of every product is a sum of at most n terms, so whatever the tiling and the order, |fl(sum) - sum| <= n u sum|terms|
    to first order.
      backward: textbook Cholesky leaves |R^T R - A| <= (n + 1) u |R^T||R| <= (n + 1) u max|A|.  CholInv forms R12 = Rinv11^T A12 with
        an inverse instead of a triangular solve; with Rinv11 R11 = I + E, |E| <~ n u kappa(R), the block R11^T R12 - A12 = E^T A12 +
        R11^T (rounding of the product) is at most 2 n u kappa(R) ||A||_2 in norm, kappa(R) = sqrt(kappa(A)).  Sum of the two, with
        max|A| <= ||A||_2.
      inverse: Rinv12 = -Rinv11 R12 Rinv22 is two products; with the error of the diagonal blocks, |Rinv R - I| <= 3 n u kappa(A).
      forward: R is the exact factor of A + dA with ||dA||_F <= n * backward; the factor's perturbation bound (Sun 1991; Higham,
        Accuracy and Stability, thm 10.8) gives ||dR||_F <= kappa(A) / sqrt 2 * ||R||_2 ||dA||_F / ||A||_2 to first order (doubled
        here for the higher orders).  Rinv - R^-1 = (Rinv R_c - I) R_c^-1 + (R_c^-1 - R^-1) for the computed R_c, the last term being
        R^-1 dR R^-1 to first order.
    The generator's matrix is diagonally dominant (n on the diagonal, entries in [0, 1) elsewhere), so kappa(A) is about 1.5; it is
    computed, not assumed."""

    def __init__(self, a):
        n = a.shape[0]
        ev = np.linalg.eigvalsh(a)
        self.norm2, self.kappa = float(ev[-1]), float(ev[-1] / ev[0])
        self.backward = (n + 1) * U * (1 + 2 * np.sqrt(self.kappa)) * self.norm2
        self.inverse = 3 * n * U * self.kappa
        norm_r, norm_ri = np.sqrt(ev[-1]), 1 / np.sqrt(ev[0])
        self.forward_r = 2 * self.kappa / np.sqrt(2) * norm_r * (n * self.backward) / self.norm2
        self.forward_rinv = 2 * (n * self.inverse * norm_ri + norm_ri ** 2 * self.forward_r)


def residual_rows(r, ri, a, rows, dtype=np.longdouble):
    """(max|R^T R - A|, max|Rinv R - I|) over the given rows, evaluated in `dtype`.  numpy's long double products run at about
    0.1 Gflop/s, so callers give it a sample of the rows and evaluate the rest in float64, whose own rounding (at most n u max|A| and
    n u kappa(R)) is within the bounds above."""
    rows = np.asarray(rows)
    rl = np.asarray(r, dtype=dtype)
    e_a = np.abs(rl[:, rows].T @ rl - a[rows]).max()
    e_i = np.asarray(ri[rows], dtype=dtype) @ rl
    e_i[np.arange(len(rows)), rows] -= 1
    return float(e_a), float(np.abs(e_i).max())
