"""Timing of cholinv::sygst for itype 2 and 3 (capital_cholinv_sygst_ab_f64) and apply_R (capital_cholinv_apply_r_f64) on one GPU,
against the FP64 tensor-pipe ceiling and torch's dense products.

    python tools/sygst_ab_bench.py [--n 16384] [--bcm -5] [--iters 10] [--out FILE]

B = the generator's SPD matrix, factored once (complete_inv = 1, device buffers, packed; only R is read, so complete_inv does not matter);
A = a seeded random symmetric matrix.  sygst(itype=2) is warmed up, then `iters` calls are timed with CUDA events.  Its algorithmic flops
come from the shapes: n(n+1)(n+2)/3 for W = R U (upper output, k from i to j) and n(n+1)(n+2)/3 for each of W R^T and R W^T (upper
output, k from max(i, j)): n(n+1)(n+2) in all, n^3 to leading order.  The GEMM kernel's own time and flops (capital_profile_*) are set
against the DMMA ceiling probed in the same run (capital_probe_dmma_f64).  Baseline: torch's dense R @ A @ R.T on the same R (4 n^3
flops).  apply_R (X = R B) is timed at nrhs = 1 and 32 against torch's R @ B.  The card name, power limit and max SM clock are read in
the same run.  Writes one JSON document."""
import argparse, json, os, sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import torch
import capital_b200 as cb
from sygst_bench import card, timed


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=16384)
    ap.add_argument("--bcm", type=int, default=-5)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--ref-iters", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("sygst_ab_bench needs a GPU (no CPU fallback)")
    torch.cuda.set_device(0)
    n = a.n
    topo = cb.topo.square(1, 0, 1)
    ctx = topo.context()
    B = cb.matrix(n, n, 1, 1).distribute_symmetric(topo)
    g = torch.randn(n, n, dtype=torch.float64, device="cuda", generator=torch.Generator("cuda").manual_seed(1))
    A = cb.matrix(n, n, 1, 1, data=(g + g.t()).t().contiguous().view(-1))
    del g
    peak, _ = ctx.probe_dmma()
    doc = {"tool": "tools/sygst_ab_bench.py", **card(), "n": n, "bc_mult_dim": a.bcm, "iters": a.iters,
           "dmma_peak_TFLOPs": round(peak, 2), "records": [], "apply_r": []}
    args = cb.cholinv.info(1, 1, a.bcm, "U")
    cb.cholinv.factor(B, args, topo)
    ms = timed(lambda: cb.cholinv.sygst(A, args, topo, itype=2), a.iters)
    ctx.profile_begin()
    Cl = cb.cholinv.sygst(A, args, topo, itype=2)
    gemm_ms, gemm_fl, gemm_n = ctx.profile_end()
    flops = n * (n + 1) * (n + 2)
    R = cb.cholinv.construct_R(args)
    av = A.view2d()
    dense = lambda: R @ av @ R.t()
    ms_dense = timed(dense, a.ref_iters, warmup=1)
    ref = dense()
    iu = torch.triu_indices(n, n, device="cuda")
    err = ((Cl[(iu[1] * (iu[1] + 1)) // 2 + iu[0]] - ref[iu[0], iu[1]]).abs().max() / ref.abs().max()).item()
    del iu, ref, Cl
    rec = {"itype": 2, "ms": round(ms, 3), "flops": flops,
           "TFLOPs": round(flops / (ms * 1e-3) / 1e12, 2), "of_dmma_peak": round(flops / (ms * 1e-3) / 1e12 / peak, 3),
           "gemm_launches": gemm_n, "gemm_ms": round(gemm_ms, 3), "gemm_TFLOPs": round(gemm_fl / (gemm_ms * 1e-3) / 1e12, 2),
           "gemm_of_dmma_peak": round(gemm_fl / (gemm_ms * 1e-3) / 1e12 / peak, 3),
           "torch_dense_ms": round(ms_dense, 2), "speedup_vs_torch_dense": round(ms_dense / ms, 2), "rel_diff_vs_torch_dense": err}
    doc["records"].append(rec)
    print(json.dumps(rec), flush=True)
    for k in (1, 32):
        rhs = torch.randn(n, k, dtype=torch.float64, device="cuda", generator=torch.Generator("cuda").manual_seed(k))
        ms_a = timed(lambda: cb.cholinv.apply_R(args, rhs, topo), 20)
        ms_t = timed(lambda: R @ rhs, 20)
        X = cb.cholinv.apply_R(args, rhs, topo)
        Xt = R @ rhs
        e = ((X - Xt).abs().max() / Xt.abs().max()).item()
        # the packed triangle is read once per panel of 32 right-hand sides: n(n+1)/2 doubles, plus B and X
        byt = 8 * (n * (n + 1) / 2 + 2 * n * k)
        r2 = {"nrhs": k, "ms": round(ms_a, 3), "GBs": round(byt / (ms_a * 1e-3) / 1e9, 1), "torch_matmul_ms": round(ms_t, 3),
              "speedup_vs_torch_matmul": round(ms_t / ms_a, 2), "rel_diff_vs_torch_matmul": e}
        doc["apply_r"].append(r2)
        print(json.dumps(r2), flush=True)
    text = json.dumps(doc, indent=1)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(text + "\n")
    print(text)


if __name__ == "__main__":
    main()
