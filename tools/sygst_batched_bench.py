"""Timing of the batched inverse, sygst, products with the factors and eigh_batched (capital_cholinv_inverse_batched_f64,
_sygst_batched_f64, _sygst_ab_batched_f64, _apply_rinv_batched_f64, _apply_r_batched_f64) on one GPU, against torch.

    python tools/sygst_batched_bench.py [--sizes 32,64,128,256,384,512] [--iters 5] [--mem-gb 48] [--out FILE]

For every n the batch is grown until one sygst_batched call takes at least 50 ms (or the buffers of the comparison would pass --mem-gb);
B is seeded, exactly symmetric and well conditioned, A a seeded symmetric matrix.  Every timing is the mean of `iters` calls after
warm-up, with CUDA events.  Recorded per n, on the same batch and the same factors R = torch's upper Cholesky factor shape:
  - inverse_batched against torch.cholesky_inverse(R, upper=True), algorithmic GFLOP/s at n^3 / 3 per matrix;
  - sygst_batched itype 1 against torch's two batched solve_triangular on R (R^-T A R^-1), itype 2 against R @ A @ R.mT, at n^3 per matrix;
  - apply_Rinv_batched and apply_RT_batched at nrhs 1 and 32 against solve_triangular and matmul;
  - eigh_batched (itype 1) against the torch pipeline cholesky_ex + two solve_triangular + eigh + solve_triangular, on a batch sized so
    that torch.linalg.eigh takes about half a second, with the time torch.linalg.eigh alone takes on that batch (the same in both);
  - a loop of the single-matrix sygst over up to 64 matrices, scaled to the batch;
  - the largest difference from torch's result, relative to its largest entry.
The card name, power limit and max SM clock are read in the same run.  Writes one JSON document."""
import argparse, json, os, sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import torch
import capital_b200 as cb
from sygst_bench import card, timed

F64 = torch.float64


def spd(b, n, seed):
    g = torch.Generator("cuda").manual_seed(seed)
    A = torch.randn(b, n, n, dtype=F64, device="cuda", generator=g) * (0.1 / n ** 0.5)
    return A + A.mT + torch.eye(n, dtype=F64, device="cuda")


def sym(b, n, seed):
    g = torch.Generator("cuda").manual_seed(seed)
    A = torch.randn(b, n, n, dtype=F64, device="cuda", generator=g)
    return A + A.mT


def rel(x, ref):
    return ((x - ref).abs().max() / ref.abs().max()).item()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="32,64,128,256,384,512")
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--mem-gb", type=float, default=48.0)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("sygst_batched_bench needs a GPU (no CPU fallback)")
    torch.cuda.set_device(0)
    topo = cb.topo.square(1, 0, 1)
    topo.context()
    doc = {"tool": "tools/sygst_batched_bench.py", **card(), "iters": a.iters, "records": []}
    tri = torch.linalg.solve_triangular
    for n in [int(s) for s in a.sizes.split(",")]:
        # A, B, R, Rinv, the library's output, torch's output and its intermediate: about eight b n n buffers
        bmax = max(1, int(a.mem_gb * 1e9 / (8 * 8 * n * n)))
        batch = min(bmax, 256)
        while True:
            Bm = spd(batch, n, n)
            A = sym(batch, n, n + 1)
            R, Ri, info = cb.cholinv.factor_batched(Bm, topo)
            ms = timed(lambda: cb.cholinv.sygst_batched(A, R, Ri, topo, itype=1), 1, warmup=1)
            if ms >= 50 or batch >= bmax:
                break
            batch = min(bmax, int(batch * 70 / max(ms, 1e-3)) + 1)
            del Bm, A, R, Ri, info
            torch.cuda.empty_cache()
        assert int(info.abs().sum()) == 0
        n3 = batch * float(n) ** 3
        rec = {"n": n, "batch": batch}

        def pair(name, mine, theirs, flops=None):
            ms_m = timed(mine, a.iters, warmup=2)
            ms_t = timed(theirs, a.iters, warmup=2)
            r = {"ms": round(ms_m, 3), "torch_ms": round(ms_t, 3), "speedup_vs_torch": round(ms_t / ms_m, 2),
                 "rel_diff_vs_torch": rel(mine(), theirs())}
            if flops:
                r["GFLOPs"] = round(flops / (ms_m * 1e-3) / 1e9, 1)
                r["torch_GFLOPs"] = round(flops / (ms_t * 1e-3) / 1e9, 1)
            rec[name] = r
            torch.cuda.empty_cache()

        pair("inverse", lambda: cb.cholinv.inverse_batched(Ri, topo), lambda: torch.cholesky_inverse(R, upper=True), n3 / 3)
        pair("sygst_itype1", lambda: cb.cholinv.sygst_batched(A, R, Ri, topo, itype=1),
             lambda: tri(R, tri(R, A, upper=True, left=False).mT, upper=True, left=False).mT, n3)
        pair("sygst_itype2", lambda: cb.cholinv.sygst_batched(A, R, Ri, topo, itype=2), lambda: R @ A @ R.mT, n3)
        for k in (1, 32):
            Y = torch.randn(batch, n, k, dtype=F64, device="cuda", generator=torch.Generator("cuda").manual_seed(k))
            pair(f"apply_Rinv_nrhs{k}", lambda: cb.cholinv.apply_Rinv_batched(Ri, Y, topo), lambda: tri(R, Y, upper=True))
            pair(f"apply_RT_nrhs{k}", lambda: cb.cholinv.apply_RT_batched(R, Y, topo), lambda: R.mT @ Y)
            del Y
        # eigh: a batch on which torch.linalg.eigh takes about half a second
        C = cb.cholinv.sygst_batched(A[:8], R[:8], Ri[:8], topo, itype=1)
        ms8 = timed(lambda: torch.linalg.eigh(C), 1, warmup=1)
        be = max(1, min(batch, int(8 * 500 / max(ms8, 1e-3))))
        Ae, Be = A[:be], Bm[:be]

        def torch_eigh():
            L, _ = torch.linalg.cholesky_ex(Be)
            Ct = tri(L, tri(L, Ae, upper=False).mT, upper=False)
            w, Y = torch.linalg.eigh(Ct)
            return w, tri(L.mT, Y, upper=True)

        iters_e = max(1, min(a.iters, 3))
        ms_e = timed(lambda: cb.cholinv.eigh_batched(Ae, Be, topo), iters_e, warmup=1)
        ms_te = timed(torch_eigh, iters_e, warmup=1)
        Ce = cb.cholinv.sygst_batched(Ae, R[:be], Ri[:be], topo, itype=1)
        ms_eig = timed(lambda: torch.linalg.eigh(Ce), iters_e, warmup=1)
        w, X, _ = cb.cholinv.eigh_batched(Ae, Be, topo)
        wt, Xt = torch_eigh()
        rec["eigh"] = {"batch": be, "ms": round(ms_e, 3), "torch_pipeline_ms": round(ms_te, 3), "speedup_vs_torch": round(ms_te / ms_e, 2),
                       "torch_eigh_alone_ms": round(ms_eig, 3), "reduction_and_back_ms": round(ms_e - ms_eig, 3),
                       "torch_reduction_and_back_ms": round(ms_te - ms_eig, 3), "rel_diff_eigenvalues_vs_torch": rel(w, wt),
                       "rel_diff_abs_eigenvectors_vs_torch": rel(X.abs(), Xt.abs())}
        del C, Ce, w, X, wt, Xt
        # the single-matrix sygst in a loop, scaled to the batch
        m = min(batch, 64)
        singles = []
        for i in range(m):
            args = cb.cholinv.info(1, 1, 0, "U", serialize=False)
            args.R, args.Rinv = R[i].mT.contiguous().reshape(-1), Ri[i].mT.contiguous().reshape(-1)
            args.local_dim = args.global_dim = n
            singles.append((cb.matrix(n, n, 1, 1, data=A[i].mT.contiguous().reshape(-1)), args))

        def loop():
            for Am, args in singles:
                cb.cholinv.sygst(Am, args, topo)

        ms_loop = timed(loop, a.iters, warmup=1) * batch / m
        rec["sygst_itype1"]["single_call_loop_ms_scaled"] = round(ms_loop, 3)
        rec["sygst_itype1"]["speedup_vs_single_call_loop"] = round(ms_loop / rec["sygst_itype1"]["ms"], 2)
        del singles, Bm, A, R, Ri, info
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
