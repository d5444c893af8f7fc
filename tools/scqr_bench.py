"""Timing and accuracy of shifted CholeskyQR3 (cacqr num_iter = 3) on one GPU.

    python tools/scqr_bench.py [--m 131072,1048576] [--n 256] [--iters 10] [--out FILE]

For each m, on the generator's well-conditioned A (distribute_random, device buffers), CUDA-event means of `iters` calls after
warm-up:
  * cacqr.factor with num_iter 2 (CholeskyQR2) and 3 (shifted CholeskyQR3), and torch.linalg.qr (cuSOLVER geqrf + orgqr);
  * cacqr.factor(3) + lstsq against torch.linalg.lstsq (one right-hand side).
At the first m, A = U diag(logspace(0, -10, n)) V^T (kappa = 1e10): the validator's residual and orthogonality of the num_iter 3
factors and the forward error of lstsq on a consistent system.  The card name and power limit are read in the same run.  Writes one
JSON document (default profiles/h100_scqr3_m131072_n256.json)."""
import argparse, json, os, sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import torch
import capital_b200 as cb
from solve_bench import card, timed


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--m", default="131072,1048576")
    ap.add_argument("--n", type=int, default=256)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_scqr3_m131072_n256.json"))
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("scqr_bench needs a GPU (no CPU fallback)")
    torch.cuda.set_device(0)
    n = a.n
    topo = cb.topo.rect(1, 0, 1)
    doc = {"card": card(), "n": n, "iters": a.iters, "runs": []}
    for i, m in enumerate(int(s) for s in a.m.split(",")):
        A = cb.matrix(n, m, 1, 1).distribute_random(topo, 5)
        args = {it: cb.cacqr.info(it, cb.cholinv.info(0, 1, 0, "U")) for it in (2, 3)}
        run = {"m": m}
        for it in (2, 3):
            run[f"factor_num_iter{it}_ms"] = timed(lambda: cb.cacqr.factor(A, args[it], topo), a.iters)
        A2 = A.view2d()
        run["torch_linalg_qr_ms"] = timed(lambda: torch.linalg.qr(A2), a.iters)
        B = torch.rand(m, 1, dtype=torch.float64, device="cuda", generator=torch.Generator(device="cuda").manual_seed(1)) - 0.5

        def ours():
            cb.cacqr.factor(A, args[3], topo)
            return cb.cacqr.lstsq(args[3], B, topo)

        run["factor3_plus_lstsq_ms"] = timed(ours, a.iters)
        run["torch_linalg_lstsq_ms"] = timed(lambda: torch.linalg.lstsq(A2, B), a.iters)
        run["factor3_over_factor2"] = run["factor_num_iter3_ms"] / run["factor_num_iter2_ms"]
        del A, A2, args
        torch.cuda.empty_cache()
        if i == 0:  # kappa = 1e10 from a chosen SVD
            g = torch.Generator(device="cuda").manual_seed(3)
            u, _ = torch.linalg.qr(torch.randn(m, n, dtype=torch.float64, device="cuda", generator=g))
            v, _ = torch.linalg.qr(torch.randn(n, n, dtype=torch.float64, device="cuda", generator=g))
            ill = (u * torch.logspace(0, -10, n, dtype=torch.float64, device="cuda")) @ v.T
            Ai = cb.matrix(n, m, 1, 1, data=ill.t().contiguous().view(-1))
            ai = cb.cacqr.info(3, cb.cholinv.info(0, 1, 0, "U"))
            cb.cacqr.factor(Ai, ai, topo)
            res, orth = cb.cacqr.validate(Ai, ai, topo)
            xt = torch.randn(n, 1, dtype=torch.float64, device="cuda", generator=g)
            X = cb.cacqr.lstsq(ai, ill @ xt, topo)
            run["kappa_1e10"] = {"residual": res, "orthogonality": orth,
                                 "lstsq_forward_error": ((X - xt).abs().max() / xt.abs().max()).item()}
            del u, ill, Ai, ai, X
            torch.cuda.empty_cache()
        doc["runs"].append(run)
        print(json.dumps(run), flush=True)
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "w") as f:
        json.dump(doc, f, indent=1)
    print(json.dumps(doc["card"]))


if __name__ == "__main__":
    main()
