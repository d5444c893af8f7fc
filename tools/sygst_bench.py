"""Timing of cholinv::sygst (capital_cholinv_sygst_f64) and apply_Rinv (capital_cholinv_apply_rinv_f64) on one GPU, against the FP64
tensor-pipe ceiling and torch's triangular solves.

    python tools/sygst_bench.py [--n 16384] [--bcm -5] [--iters 10] [--out FILE]

B = the generator's SPD matrix, factored once per complete_inv in {1, 0} (device buffers, packed); A = a seeded random symmetric matrix.
sygst is warmed up, then `iters` calls are timed with CUDA events.  Its algorithmic flops come from the shapes: n(n+1)(n+2)/3 for
V = U Rinv (upper output, k from i to j) and n(n+1)(n+2)/3 for each of Rinv^T V and V^T Rinv (upper output, k up to min(i, j)):
n(n+1)(n+2) in all, n^3 to leading order, plus the two products that rebuild a skipped top-level Rinv12.  The GEMM kernel's own time and flops
(capital_profile_*) are set against the DMMA ceiling probed in the same run (capital_probe_dmma_f64).  Baseline: torch's TRSM on the
same R, R^-T (A R^-1) with solve_triangular on the right, then on the left (2 n^3 flops).  apply_Rinv (X = R^-1 B) is timed at nrhs = 1
and 32 against solve_triangular.  The card name, power limit and max SM clock are read in the same run.  Writes one JSON document."""
import argparse, json, os, subprocess, sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch
import capital_b200 as cb
from capital_b200 import _lib


def card():
    q = "name,power.limit,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()), f"--query-gpu={q}", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        name, power, clk = [s.strip() for s in out.split(",")]
        return {"gpu": name, "power_limit": power, "sm_max_clock": clk}
    except Exception as e:  # noqa: reported, not fatal
        return {"gpu": torch.cuda.get_device_name(), "power_limit": f"not read ({e!r})"}


def timed(fn, iters, warmup=3):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def sygst_flops(n, s1, skipped):
    """algorithmic flops of one call (see the module docstring)"""
    f = n * (n + 1) * (n + 2) / 3 + 2 * n * (n + 1) * (n + 2) / 3
    if skipped:
        s2 = n - s1
        f += s2 * s1 * (s1 + 1) + s1 * s2 * (s2 + 1)
    return f


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=16384)
    ap.add_argument("--bcm", type=int, default=-5)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--ref-iters", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("sygst_bench needs a GPU (no CPU fallback)")
    torch.cuda.set_device(0)
    n = a.n
    topo = cb.topo.square(1, 0, 1)
    ctx = topo.context()
    B = cb.matrix(n, n, 1, 1).distribute_symmetric(topo)
    g = torch.randn(n, n, dtype=torch.float64, device="cuda", generator=torch.Generator("cuda").manual_seed(1))
    A = cb.matrix(n, n, 1, 1, data=(g + g.t()).t().contiguous().view(-1))
    del g
    peak, _ = ctx.probe_dmma()
    doc = {"tool": "tools/sygst_bench.py", **card(), "n": n, "bc_mult_dim": a.bcm, "iters": a.iters,
           "dmma_peak_TFLOPs": round(peak, 2), "records": [], "apply_rinv": []}
    bc = _lib.lib().capital_cholinv_bc_dimension(n, 1, 1, a.bcm)
    for ci in (1, 0):
        args = cb.cholinv.info(ci, 1, a.bcm, "U")
        cb.cholinv.factor(B, args, topo)
        skipped = ci == 0 and n > bc
        ms = timed(lambda: cb.cholinv.sygst(A, args, topo), a.iters)
        ctx.profile_begin()
        Cl = cb.cholinv.sygst(A, args, topo)
        gemm_ms, gemm_fl, gemm_n = ctx.profile_end()
        flops = sygst_flops(n, n >> 1, skipped)
        R = cb.cholinv.construct_R(args)
        av = A.view2d()
        trsm = lambda: torch.linalg.solve_triangular(R.t(), torch.linalg.solve_triangular(R, av, upper=True, left=False), upper=False)
        ms_trsm = timed(trsm, a.ref_iters, warmup=1)
        ref = trsm()
        iu = torch.triu_indices(n, n, device="cuda")
        err = ((Cl[(iu[1] * (iu[1] + 1)) // 2 + iu[0]] - ref[iu[0], iu[1]]).abs().max() / ref.abs().max()).item()
        del iu, ref, Cl
        rec = {"complete_inv": ci, "rinv12_rebuilt": skipped, "ms": round(ms, 3), "flops": flops,
               "TFLOPs": round(flops / (ms * 1e-3) / 1e12, 2), "of_dmma_peak": round(flops / (ms * 1e-3) / 1e12 / peak, 3),
               "gemm_launches": gemm_n, "gemm_ms": round(gemm_ms, 3), "gemm_TFLOPs": round(gemm_fl / (gemm_ms * 1e-3) / 1e12, 2),
               "gemm_of_dmma_peak": round(gemm_fl / (gemm_ms * 1e-3) / 1e12 / peak, 3),
               "torch_trsm_ms": round(ms_trsm, 2), "speedup_vs_torch_trsm": round(ms_trsm / ms, 2),
               "rel_diff_vs_torch_trsm": err}
        doc["records"].append(rec)
        print(json.dumps(rec), flush=True)
        if ci == 1:
            for k in (1, 32):
                rhs = torch.randn(n, k, dtype=torch.float64, device="cuda", generator=torch.Generator("cuda").manual_seed(k))
                ms_a = timed(lambda: cb.cholinv.apply_Rinv(args, rhs, topo), 20)
                ms_t = timed(lambda: torch.linalg.solve_triangular(R, rhs, upper=True), 20)
                X = cb.cholinv.apply_Rinv(args, rhs, topo)
                Xt = torch.linalg.solve_triangular(R, rhs, upper=True)
                e = ((X - Xt).abs().max() / Xt.abs().max()).item()
                # the packed triangle is read once per panel of 32 right-hand sides: n(n+1)/2 doubles, plus B and X
                byt = 8 * (n * (n + 1) / 2 + 2 * n * k)
                r2 = {"nrhs": k, "ms": round(ms_a, 3), "GBs": round(byt / (ms_a * 1e-3) / 1e9, 1), "torch_trsm_ms": round(ms_t, 3),
                      "speedup_vs_torch_trsm": round(ms_t / ms_a, 2), "rel_diff_vs_torch_trsm": e}
                doc["apply_rinv"].append(r2)
                print(json.dumps(r2), flush=True)
        del R
    text = json.dumps(doc, indent=1)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(text + "\n")
    print(text)


if __name__ == "__main__":
    main()
