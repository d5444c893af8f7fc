"""Timing of cacqr::apply_QT / lstsq (capital_cacqr_apply_qt_f64, capital_cacqr_lstsq_f64) on one GPU against the copy bandwidth and
torch.

    python tools/lstsq_bench.py [--m 1048576,131072] [--n 256] [--nrhs 1,8,32,128] [--iters 20] [--out FILE]

For each m: factor A (distribute_random, CholeskyQR2, device buffers) once, time a device-to-device copy of Q's bytes, then for each
nrhs time with CUDA events (mean of `iters` calls after warm-up):
  * apply_QT (Q^T B), with the bandwidth it reaches on Q's bytes (Q is read once per panel of 32) against the copy's;
  * lstsq (Q^T B, then the substitution with R);
  * the substitution alone: the device time of its kernels (tri_block_solve_kernel and the op-N update), from torch.profiler;
  * torch on the same Q and R: Q.T @ B (cuBLAS) and torch.linalg.solve_triangular;
  * cacqr.factor + lstsq against torch.linalg.lstsq(A, B) (cuSOLVER's QR-based gels).
The card name and power limit are read in the same run.  Writes one JSON document."""
import argparse, ctypes as C, json, os, sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import torch
import capital_b200 as cb
from capital_b200 import _lib
from solve_bench import card, timed

W = 32  # panel width of the kernels (SOLVE_W)


def substitution_ms(fn, iters):
    """device time per call of the substitution's kernels inside fn (the update of rows above a block is the op-N, non-full
    instantiation of tri_apply_kernel, which nothing else in lstsq launches)"""
    from torch.profiler import profile, ProfilerActivity
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(iters):
            fn()
        torch.cuda.synchronize()
    us = 0.0
    for ev in prof.key_averages():
        name = ev.key
        if "tri_block_solve_kernel" in name or ("tri_apply_kernel<" in name and ", false, false>" in name) or \
                "tri_finish_kernel<false>" in name:
            us += ev.device_time_total if hasattr(ev, "device_time_total") else ev.cuda_time_total
    return us / 1e3 / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--m", default="1048576,131072")
    ap.add_argument("--n", type=int, default=256)
    ap.add_argument("--nrhs", default="1,8,32,128")
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("lstsq_bench needs a GPU (no CPU fallback)")
    torch.cuda.set_device(0)
    n = a.n
    topo = cb.topo.rect(1, 0, 1)
    ctx = topo.context()
    L = _lib.lib()
    doc = {"tool": "tools/lstsq_bench.py", **card(), "n": n, "iters": a.iters, "panel_width": W, "runs": []}
    g = torch.Generator(device="cuda").manual_seed(1)
    for m in [int(s) for s in a.m.split(",")]:
        A = cb.matrix(n, m, 1, 1).distribute_random(topo, 3)
        args = cb.cacqr.info(2, cb.cholinv.info(0, 1, 0, "U"))
        cb.cacqr.factor(A, args, topo)
        q_bytes = m * n * 8
        dst = torch.empty_like(args.Q)
        copy_ms = timed(lambda: dst.copy_(args.Q), a.iters)
        del dst
        copy_bw = 2 * q_bytes / (copy_ms * 1e-3)  # read + write
        Qv, Rd = cb.cacqr.construct_Q(args), cb.cacqr.construct_R(args)
        Av = A.view2d()
        run = {"m": m, "q_bytes": q_bytes, "copy_q_ms": round(copy_ms, 4), "copy_bandwidth_GBps": round(copy_bw / 1e9, 1),
               "factor_ms": round(timed(lambda: cb.cacqr.factor(A, args, topo), 5, warmup=1), 3), "records": []}
        for k in [int(s) for s in a.nrhs.split(",")]:
            B = torch.rand(k, m, dtype=torch.float64, device="cuda", generator=g) - 0.5  # column-major m x k
            Y = torch.empty(k, n, dtype=torch.float64, device="cuda")
            X = torch.empty_like(Y)
            qt = lambda: ctx.check(L.capital_cacqr_apply_qt_f64(ctx.handle, m, n, args.Q.data_ptr(), k, B.data_ptr(), m, Y.data_ptr(), n))
            ls = lambda: ctx.check(L.capital_cacqr_lstsq_f64(ctx.handle, m, n, args.Q.data_ptr(), _lib.UPPERTRI_PACKED, args.R.data_ptr(),
                                                             k, B.data_ptr(), m, X.data_ptr(), n))
            ms_qt, ms_ls = timed(qt, a.iters), timed(ls, a.iters)
            ms_sub = substitution_ms(ls, a.iters)
            Bt = B.t()
            ms_t_qt = timed(lambda: Qv.t() @ Bt, a.iters)
            Yt = Qv.t() @ Bt
            ms_t_sub = timed(lambda: torch.linalg.solve_triangular(Rd, Yt, upper=True), a.iters)
            ref = torch.linalg.solve_triangular(Rd, Yt, upper=True)
            diff = ((X.t() - ref).abs().max() / ref.abs().max()).item()
            panels = -(-k // W)
            rate = panels * q_bytes / (ms_qt * 1e-3)
            ms_t_lstsq = timed(lambda: torch.linalg.lstsq(Av, Bt), 3, warmup=1)
            ms_ours_e2e = run["factor_ms"] + ms_ls
            rec = {"nrhs": k, "apply_qt_ms": round(ms_qt, 4), "apply_qt_q_GBps": round(rate / 1e9, 1),
                   "apply_qt_of_copy_bw": round(rate / copy_bw, 3), "tri_solve_ms": round(ms_sub, 4), "lstsq_ms": round(ms_ls, 4),
                   "torch_qt_matmul_ms": round(ms_t_qt, 4), "torch_solve_triangular_ms": round(ms_t_sub, 4),
                   "torch_products_ms": round(ms_t_qt + ms_t_sub, 4), "rel_diff_vs_torch": diff,
                   "factor_plus_lstsq_ms": round(ms_ours_e2e, 3), "torch_linalg_lstsq_ms": round(ms_t_lstsq, 3),
                   "speedup_vs_torch_linalg_lstsq": round(ms_t_lstsq / ms_ours_e2e, 2)}
            run["records"].append(rec)
            print(json.dumps({"m": m, **rec}), flush=True)
            del B, Bt, Yt, ref
        doc["runs"].append(run)
        del A, args, Qv, Rd, Av
        torch.cuda.empty_cache()
    text = json.dumps(doc, indent=1)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(text + "\n")
    print(text)


if __name__ == "__main__":
    main()
