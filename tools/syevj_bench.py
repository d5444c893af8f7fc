"""Timing of the batched Jacobi eigensolver (capital_syevj_batched_f64, eig.syevj_batched) on one GPU, against torch.linalg.eigh.

    python tools/syevj_bench.py [--sizes 16,32,64,128,256,384,512] [--iters 3] [--out FILE]

The batch at each n is the one profiles/h100_sygst_batched.json timed eigh_batched on (torch.linalg.eigh takes about half a second
there; n = 16 takes n = 32's).  The symmetric matrices are seeded, A = G + G^T.  Every timing is the mean of `iters` calls after one
warm-up call, with CUDA events.  Recorded per n:
  - syevj_batched against torch.linalg.eigh on the same batch, and the ratio;
  - the outer sweeps (n > 64), derived from the launch counter: one chunk makes 2 + sweeps (2 (N - 1) + 1) launches, N = Np / 32;
  - the worst ||A V - V diag(w)||_F / (n u ||A||_F) and ||V^T V - I||_F / (n u) over the batch, and the largest eigenvalue
    difference from torch relative to ||A||_2;
  - eigh_batched (itype 1, B seeded SPD) with eigensolver="jacobi" against eigensolver="torch".
The card name, power limit and max SM clock are read in the same run.  Writes one JSON document."""
import argparse, json, os, sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import torch
import capital_b200 as cb
from sygst_bench import card, timed

F64 = torch.float64
U = 2.0 ** -53
BATCH = {16: 9550, 32: 9550, 64: 642, 128: 301, 256: 237, 384: 142, 512: 103}


def sym(b, n, seed):
    g = torch.Generator("cuda").manual_seed(seed)
    A = torch.randn(b, n, n, dtype=F64, device="cuda", generator=g)
    return A + A.mT


def spd(b, n, seed):
    g = torch.Generator("cuda").manual_seed(seed)
    A = torch.randn(b, n, n, dtype=F64, device="cuda", generator=g) * (0.1 / n ** 0.5)
    return A + A.mT + torch.eye(n, dtype=F64, device="cuda")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="16,32,64,128,256,384,512")
    ap.add_argument("--iters", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("syevj_bench needs a GPU (no CPU fallback)")
    torch.cuda.set_device(0)
    topo = cb.topo.square(1, 0, 1)
    ctx = topo.context()
    doc = {"tool": "tools/syevj_bench.py", **card(), "iters": a.iters, "records": []}
    for n in [int(s) for s in a.sizes.split(",")]:
        b = BATCH[n]
        A = sym(b, n, n)
        rec = {"n": n, "batch": b}
        rec["syevj_ms"] = timed(lambda: cb.eig.syevj_batched(A, topo), a.iters, warmup=1)
        rec["torch_eigh_ms"] = timed(lambda: torch.linalg.eigh(A), a.iters, warmup=1)
        rec["speedup_vs_torch"] = rec["torch_eigh_ms"] / rec["syevj_ms"]
        torch.cuda.synchronize()
        ctx.reset_counters()
        w, V, info = cb.eig.syevj_batched(A, topo)
        torch.cuda.synchronize()
        launches = ctx.counters().kernel_launches
        rec["launches"], rec["info_nonzero"] = launches, int((info != 0).sum())
        if n > 64:
            N = -(-n // 64) * 2
            assert b <= cb_chunk(n)  # one chunk: the launch count gives the sweeps
            rec["outer_sweeps"] = (launches - 2) // (2 * N - 1)
        anorm = torch.linalg.matrix_norm(A)
        res = torch.linalg.matrix_norm(A @ V - V * w[:, None, :]) / (n * U * anorm)
        orth = torch.linalg.matrix_norm(V.mT @ V - torch.eye(n, dtype=F64, device="cuda")) / (n * U)
        wt = torch.linalg.eigvalsh(A)
        rec["worst_residual_over_nu_normA"] = res.max().item()
        rec["worst_orth_over_nu"] = orth.max().item()
        rec["worst_eig_diff_over_normA2"] = ((w - wt).abs().amax(1) / torch.linalg.matrix_norm(A, 2)).max().item()
        B = spd(b, n, n + 1)
        rec["eigh_batched_jacobi_ms"] = timed(lambda: cb.cholinv.eigh_batched(A, B, topo, eigensolver="jacobi"), a.iters, warmup=1)
        rec["eigh_batched_torch_ms"] = timed(lambda: cb.cholinv.eigh_batched(A, B, topo), a.iters, warmup=1)
        print(json.dumps(rec), flush=True)
        doc["records"].append(rec)
        del A, V, w, B
        torch.cuda.empty_cache()
    s = json.dumps(doc, indent=1)
    if a.out:
        with open(a.out, "w") as f:
            f.write(s + "\n")
    else:
        print(s)


def cb_chunk(n):
    """matrices per chunk of capital_syevj_batched_f64 (tests/syevj_reference.chunk)"""
    if n <= 64:
        return 65535
    Np = -(-n // 64) * 64
    return min(65535, (2 << 30) // ((2 * Np * Np + Np // 64 * 4096) * 8))


if __name__ == "__main__":
    main()
