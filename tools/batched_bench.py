"""Timing of the batched CholInv (capital_cholinv_factor_batched_f64 / capital_cholinv_solve_batched_f64) on one GPU, against torch.

    python tools/batched_bench.py [--sizes 32,64,128,256,384,512] [--iters 5] [--mem-gb 56] [--out FILE]

For every n the batch is grown until one factor_batched call takes at least 50 ms (or its buffers, and torch's, would pass --mem-gb);
the matrices are seeded, exactly symmetric and well conditioned.  Every timing is the mean of `iters` calls after warm-up, with CUDA
events.  Recorded per n:
  - factor_batched: ms, matrices/s and algorithmic GFLOP/s at 2n^3/3 per matrix (n^3/3 for potrf plus n^3/3 for trtri);
  - torch on the same batch: cholesky_ex(upper=True) followed by solve_triangular(R, I) for the inverse, and cholesky_ex alone;
  - solve_batched at nrhs 1 and 32 against torch.cholesky_solve on torch's own factor;
  - for n in {128, 256}: the width the library picks for its cluster kernel against width 8 (CAPITAL_BATCHED_CW=8), alternated in
    the same run, three rounds each;
  - batch = 1: the latency of one factor_batched call (mean of 200), the base-case kernel of that n on its own.
The card name, power limit and max SM clock are read in the same run.  Writes one JSON document."""
import argparse, json, os, sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import torch
import capital_b200 as cb
from sygst_bench import card, timed


def spd(b, n, seed):
    g = torch.Generator("cuda").manual_seed(seed)
    A = torch.randn(b, n, n, dtype=torch.float64, device="cuda", generator=g) * (0.1 / n ** 0.5)
    return A + A.mT + torch.eye(n, dtype=torch.float64, device="cuda")


def width(n):
    t = (n + 63) // 64
    return 0 if n <= 64 else 2 if t <= 2 else 4 if t <= 4 else 8


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="32,64,128,256,384,512")
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--mem-gb", type=float, default=56.0)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("batched_bench needs a GPU (no CPU fallback)")
    torch.cuda.set_device(0)
    topo = cb.topo.square(1, 0, 1)
    topo.context()
    doc = {"tool": "tools/batched_bench.py", **card(), "iters": a.iters, "records": []}
    for n in [int(s) for s in a.sizes.split(",")]:
        # A, R, Rinv, torch's R, its inverse and the identity right-hand side: six b n n buffers
        bmax = max(1, int(a.mem_gb * 1e9 / (6 * 8 * n * n)))
        batch = min(bmax, 1024)
        while True:
            A = spd(batch, n, n)
            ms = timed(lambda: cb.cholinv.factor_batched(A, topo), 1, warmup=1)
            if ms >= 50 or batch >= bmax:
                break
            batch = min(bmax, int(batch * 70 / max(ms, 1e-3)) + 1)
            del A
            torch.cuda.empty_cache()
        ms = timed(lambda: cb.cholinv.factor_batched(A, topo), a.iters, warmup=2)
        flops = batch * 2 * n ** 3 / 3
        R, Ri, info = cb.cholinv.factor_batched(A, topo)
        assert int(info.abs().sum()) == 0
        rec = {"n": n, "batch": batch, "cluster_width": width(n), "ms": round(ms, 3), "matrices_per_s": round(batch / (ms * 1e-3)),
               "GFLOPs": round(flops / (ms * 1e-3) / 1e9, 1)}
        eye = torch.eye(n, dtype=torch.float64, device="cuda").expand(batch, n, n)

        def torch_inv():
            U, _ = torch.linalg.cholesky_ex(A, upper=True)
            return U, torch.linalg.solve_triangular(U, eye, upper=True)

        ms_ti = timed(torch_inv, a.iters, warmup=2)
        ms_tc = timed(lambda: torch.linalg.cholesky_ex(A, upper=True), a.iters, warmup=2)
        U, Ui = torch_inv()
        rec.update({"torch_cholesky_ex_plus_inverse_ms": round(ms_ti, 3), "torch_cholesky_ex_ms": round(ms_tc, 3),
                    "speedup_vs_torch_cholesky_plus_inverse": round(ms_ti / ms, 2),
                    "speedup_vs_torch_cholesky_ex": round(ms_tc / ms, 2),
                    "rel_diff_R_vs_torch": ((R - U).abs().max() / U.abs().max()).item(),
                    "rel_diff_Rinv_vs_torch": ((Ri - Ui).abs().max() / Ui.abs().max()).item()})
        del U, Ui, eye
        torch.cuda.empty_cache()
        L = R.mT.contiguous()
        rec["solve"] = []
        for k in (1, 32):
            B = torch.randn(batch, n, k, dtype=torch.float64, device="cuda", generator=torch.Generator("cuda").manual_seed(k))
            ms_s = timed(lambda: cb.cholinv.solve_batched(Ri, B, topo), a.iters, warmup=2)
            ms_t = timed(lambda: torch.cholesky_solve(B, L), a.iters, warmup=2)
            X, Xt = cb.cholinv.solve_batched(Ri, B, topo), torch.cholesky_solve(B, L)
            rec["solve"].append({"nrhs": k, "ms": round(ms_s, 3), "torch_cholesky_solve_ms": round(ms_t, 3),
                                 "speedup_vs_torch": round(ms_t / ms_s, 2),
                                 "rel_diff_vs_torch": ((X - Xt).abs().max() / Xt.abs().max()).item()})
            del B, X, Xt
        del L
        if n in (128, 256):
            mine, eight = [], []
            for _ in range(3):
                os.environ.pop("CAPITAL_BATCHED_CW", None)
                mine.append(timed(lambda: cb.cholinv.factor_batched(A, topo), a.iters, warmup=1))
                os.environ["CAPITAL_BATCHED_CW"] = "8"
                R8, Ri8, _ = cb.cholinv.factor_batched(A, topo)
                eight.append(timed(lambda: cb.cholinv.factor_batched(A, topo), a.iters, warmup=1))
                os.environ.pop("CAPITAL_BATCHED_CW", None)
            rec["width_vs_8"] = {"width": width(n), "ms": [round(x, 3) for x in mine], "width8_ms": [round(x, 3) for x in eight],
                                 "same_bits_as_width8": bool(torch.equal(R8, R) and torch.equal(Ri8, Ri))}
            del R8, Ri8
        del A, R, Ri
        torch.cuda.empty_cache()
        A1 = spd(1, n, 5)
        rec["batch1_latency_ms"] = round(timed(lambda: cb.cholinv.factor_batched(A1, topo), 200, warmup=20), 4)
        doc["records"].append(rec)
        print(json.dumps(rec), flush=True)
    text = json.dumps(doc, indent=1)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(text + "\n")
    print(text)


if __name__ == "__main__":
    main()
