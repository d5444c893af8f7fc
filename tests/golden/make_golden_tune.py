"""Generate the golden fixtures of the tunable c x d x c CA-CholeskyQR2 grid (1 < c < d; the reference's sweep_tune,
cacqr.hpp:122-170) by running the reference itself, like tests/golden/make_golden.py, whose driver and helpers it reuses:

    bash oracle/build_ref.sh && python tests/golden/make_golden_tune.py [names...]

16 ranks on the 2 x 4 x 2 grid (two 2x2x2 cubes).  Every layer holds the same A, Q and R blocks, so each fixture stores one rank
per layer pair; meta["replica_of"] maps a left-out rank to the stored one (about 0.5 MB per fixture instead of 1.05 MB).
"""
import json, os, sys, tempfile
import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from make_golden import HERE, REF, dedup_replicas, run  # noqa: E402

TUNE = [  # name, P, variant, m, n, c, complete_inv, split, bc_mult
    ("cacqr_p16_tune_m512_n64", 16, 2, 512, 64, 2, 1, 1, -1),
    ("cacqr_p16_tune_m512_n64_ci0", 16, 2, 512, 64, 2, 0, 1, -1),  # complete_inv = 0: the reference's block `solve` (cacqr.hpp:46-71)
    ("cacqr_p16_tune_m512_n64_it1", 16, 1, 512, 64, 2, 1, 1, -1),  # num_iter = 1: one sweep (CholeskyQR, not QR2)
]


def main():
    only = set(sys.argv[1:])  # optional: regenerate the named fixtures only
    for name, P, var, m, n, c, ci, split, bcm in TUNE:
        if only and name not in only:
            continue
        with tempfile.TemporaryDirectory() as td:
            meta = run([os.path.join(REF, "ref_cacqr"), str(var), str(m), str(n), str(c), str(ci), str(split), str(bcm), "1", os.path.join(td, "d")], P)
            arrs = {}
            for r in range(P):
                for k in ("A", "Q", "R"):
                    arrs[f"{k}_{r}"] = np.fromfile(os.path.join(td, f"d.{k}.{r}.bin"), dtype=np.float64)
            dedup_replicas(meta, arrs, P, ("A", "Q", "R"))
            np.savez_compressed(os.path.join(HERE, name + ".npz"), meta=json.dumps(meta), **arrs)
            print(name, meta)


if __name__ == "__main__":
    main()
