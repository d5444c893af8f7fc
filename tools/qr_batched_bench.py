"""Timing of the batched CholeskyQR (capital_cacqr_factor_batched_f64 / capital_cacqr_lstsq_batched_f64) on one GPU, against torch.

    python tools/qr_batched_bench.py [--shapes 1024x32,4096x64,16384x128,32768x256,65536x512] [--iters 5] [--mem-gb 40] [--out FILE]

For every m x n the batch is grown until one factor_batched call (num_iter = 2) takes at least 50 ms (or its buffers, and torch's,
would pass --mem-gb); the matrices are seeded Gaussian (well conditioned).  Every timing is the mean of `iters` calls after warm-up,
with CUDA events.  Recorded per shape:
  - factor_batched: ms, matrices/s, and bytes/s at the model's traffic, 4 passes of 8 m n bytes per sweep, against a device-to-device
    copy of A timed in the same run (read + write: 16 m n bytes per matrix);
  - a loop of cacqr.factor (one matrix per call, rect R) over a subset of the batch, scaled to the whole batch;
  - torch on the same batch: linalg.qr (reduced), and CholeskyQR2 written in batched torch (A^T A, cholesky_ex, solve_triangular);
  - lstsq_batched at nrhs 1 and 32 against torch.linalg.lstsq;
  - the largest residual ||QR - A||_F / ||A||_F and orthogonality ||Q^T Q - I||_F over the batch (torch float64 products).
The card name, power limit and max SM clock are read in the same run.  Writes one JSON document."""
import argparse, json, os, sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import torch
import capital_b200 as cb
from sygst_bench import card, timed


def tall(b, m, n, seed):
    g = torch.Generator("cuda").manual_seed(seed)
    return torch.randn(b, n, m, dtype=torch.float64, device="cuda", generator=g).mT  # column-major matrices: read in place


def torch_cqr2(A):
    R1 = torch.linalg.cholesky_ex(A.mT @ A, upper=True)[0]
    Q1 = torch.linalg.solve_triangular(R1, A, upper=True, left=False)
    R2 = torch.linalg.cholesky_ex(Q1.mT @ Q1, upper=True)[0]
    return torch.linalg.solve_triangular(R2, Q1, upper=True, left=False), R2 @ R1


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shapes", default="1024x32,4096x64,16384x128,32768x256,65536x512")
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--mem-gb", type=float, default=40.0)
    ap.add_argument("--loop-max", type=int, default=64, help="matrices timed through the cacqr.factor loop")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("qr_batched_bench needs a GPU (no CPU fallback)")
    torch.cuda.set_device(0)
    topo = cb.topo.rect(1, 0, 1)
    topo.context()
    doc = {"tool": "tools/qr_batched_bench.py", **card(), "iters": a.iters, "num_iter": 2, "records": []}
    for shape in a.shapes.split(","):
        m, n = (int(s) for s in shape.split("x"))
        # A, Q, torch's Q and its workspaces: about eight b m n buffers
        bmax = max(1, int(a.mem_gb * 1e9 / (8 * 8 * m * n)))
        batch = min(bmax, 64)
        while True:
            A = tall(batch, m, n, m + n)
            ms = timed(lambda: cb.cacqr.factor_batched(A, topo), 1, warmup=1)
            if ms >= 50 or batch >= bmax:
                break
            batch = min(bmax, int(batch * 70 / max(ms, 1e-3)) + 1)
            del A
            torch.cuda.empty_cache()
        ms = timed(lambda: cb.cacqr.factor_batched(A, topo), a.iters, warmup=2)
        Q, R, info = cb.cacqr.factor_batched(A, topo)
        assert int(info.abs().sum()) == 0
        ms_copy = timed(lambda: A.clone(), a.iters, warmup=2)
        model = batch * 2 * 4 * 8 * m * n
        rec = {"m": m, "n": n, "batch": batch, "ms": round(ms, 3), "matrices_per_s": round(batch / (ms * 1e-3)),
               "model_GBps": round(model / (ms * 1e-3) / 1e9, 1), "copy_GBps": round(batch * 16 * m * n / (ms_copy * 1e-3) / 1e9, 1)}
        eye = torch.eye(n, dtype=torch.float64, device="cuda")
        res = float((torch.linalg.norm(Q @ R - A, dim=(1, 2)) / torch.linalg.norm(A, dim=(1, 2))).max())
        orth = float(torch.linalg.norm(Q.mT @ Q - eye, dim=(1, 2)).max())
        rec.update({"max_residual": res, "max_orthogonality": orth})
        del Q, R
        # the same matrices one call at a time (a subset, scaled)
        sub = min(batch, a.loop_max)
        mats = [cb.matrix(n, m, 1, 1, data=A[b].mT.contiguous().reshape(-1)) for b in range(sub)]
        args = [cb.cacqr.info(2, cb.cholinv.info(0, 1, 0, "U"), serialize=False) for _ in range(sub)]

        def loop():
            for M, g in zip(mats, args):
                cb.cacqr.factor(M, g, topo)

        ms_loop = timed(loop, 2, warmup=1) * batch / sub
        del mats, args
        torch.cuda.empty_cache()
        ms_qr = timed(lambda: torch.linalg.qr(A), a.iters, warmup=1)
        torch.cuda.empty_cache()
        ms_tq = timed(lambda: torch_cqr2(A), a.iters, warmup=1)
        torch.cuda.empty_cache()
        rec.update({"loop_of_factor_ms": round(ms_loop, 3), "loop_subset": sub, "speedup_vs_loop": round(ms_loop / ms, 2),
                    "torch_qr_ms": round(ms_qr, 3), "speedup_vs_torch_qr": round(ms_qr / ms, 2),
                    "torch_cholesky_qr2_ms": round(ms_tq, 3), "speedup_vs_torch_cholesky_qr2": round(ms_tq / ms, 2)})
        Q, R, _ = cb.cacqr.factor_batched(A, topo)
        rec["lstsq"] = []
        for k in (1, 32):
            B = torch.randn(batch, m, k, dtype=torch.float64, device="cuda", generator=torch.Generator("cuda").manual_seed(k))
            ms_l = timed(lambda: cb.cacqr.lstsq_batched(Q, R, B, topo), a.iters, warmup=2)
            ms_t = timed(lambda: torch.linalg.lstsq(A, B), a.iters, warmup=1)
            X, Xt = cb.cacqr.lstsq_batched(Q, R, B, topo), torch.linalg.lstsq(A, B).solution
            rec["lstsq"].append({"nrhs": k, "ms": round(ms_l, 3), "torch_lstsq_ms": round(ms_t, 3), "speedup_vs_torch": round(ms_t / ms_l, 2),
                                 "rel_diff_vs_torch": float(torch.linalg.norm(X - Xt) / torch.linalg.norm(Xt))})
            del B, X, Xt
            torch.cuda.empty_cache()
        del A, Q, R
        torch.cuda.empty_cache()
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
