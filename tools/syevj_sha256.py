"""SHA-256 of the batched Jacobi eigensolver's outputs (w, V, info of eig.syevj_batched) on the accuracy inputs of
tests/test_gpu_syevj_reference.py: every family of tests/syevj_reference.FAMILIES at each n of ACCURACY_N, one batch per n, seeded
as in tests/test_gpu_syevj.py.  Every input lies well inside the double range, so a change to the solver's scaling must leave these
bits alone; tests/golden/syevj_sha256.json holds the hashes of the solver before it normalised each matrix by a power of 4.

    python tools/syevj_sha256.py [--out FILE]
"""
import argparse, hashlib, json, os, sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np
import torch
import capital_b200 as cb
import syevj_reference as sr

ACCURACY_N = [1, 2, 3, 7, 31, 32, 33, 63, 64, 65, 100, 127, 128, 129, 255, 256, 257, 383, 511, 512]


def inputs(n):
    return np.stack([sr.family(f, n, 1000 * n + i)[0] for i, f in enumerate(sr.FAMILIES)])


def digest(w, V, info):
    return {k: hashlib.sha256(t.cpu().contiguous().numpy().tobytes()).hexdigest() for k, t in (("w", w), ("V", V), ("info", info))}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("syevj_sha256 needs a GPU (no CPU fallback)")
    topo = cb.topo.square(1, 0, 1)
    recs = [{"n": n, **digest(*cb.eig.syevj_batched(torch.from_numpy(inputs(n)).cuda(), topo))} for n in ACCURACY_N]
    s = "[\n" + ",\n".join(json.dumps(r) for r in recs) + "\n]\n"
    if a.out:
        with open(a.out, "w") as f:
            f.write(s)
    else:
        print(s, end="")


if __name__ == "__main__":
    main()
