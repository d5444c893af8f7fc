"""Timing of cholinv::inverse (capital_cholinv_inverse_f64) on one GPU against the FP64 tensor-pipe ceiling, cuSOLVER and torch.

    python tools/inverse_bench.py [--n 16384] [--bcm -5] [--iters 20] [--out FILE]

For complete_inv in {1, 0}: factor once (device buffers, packed), warm up, then time `iters` inverse calls with CUDA events.  The
algorithmic flops are computed from the shapes: n(n+1)(n+2)/3 for the product of Rinv^T with itself (upper tiles, k from max(i, j)),
plus the two products that rebuild a skipped top-level Rinv12.  The GEMM kernel's own time and flops (capital_profile_*) are set against
the DMMA ceiling probed in the same run (capital_probe_dmma_f64).  Baselines: torch.cholesky_inverse on the same factor R (cuSOLVER
potri) and torch.linalg.inv(A).  The card name, power limit and max SM clock are read in the same run.  Writes one JSON document."""
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


def inverse_flops(n, s1, skipped):
    """algorithmic flops: sum over the upper output entries (i <= j) of 2 (n - j); a rebuilt Rinv12 adds T^T = R12^T Rinv11^T
    (s2 x s1, k from the column) and Rinv12 = -(T^T)^T Rinv22 (s1 x s2, k up to the column)"""
    f = n * (n + 1) * (n + 2) / 3
    if skipped:
        s2 = n - s1
        f += s2 * s1 * (s1 + 1) + s1 * s2 * (s2 + 1)
    return f


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=16384)
    ap.add_argument("--bcm", type=int, default=-5)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--ref-iters", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("inverse_bench needs a GPU (no CPU fallback)")
    torch.cuda.set_device(0)
    n = a.n
    topo = cb.topo.square(1, 0, 1)
    ctx = topo.context()
    A = cb.matrix(n, n, 1, 1).distribute_symmetric(topo)
    peak, _ = ctx.probe_dmma()
    doc = {"tool": "tools/inverse_bench.py", **card(), "n": n, "bc_mult_dim": a.bcm, "iters": a.iters,
           "dmma_peak_TFLOPs": round(peak, 2), "records": []}
    V = A.view2d()
    Afull = torch.triu(V) + torch.triu(V, 1).t()  # the factor reads the upper triangle only
    ms_inv = timed(lambda: torch.linalg.inv(Afull), a.ref_iters, warmup=1)
    for ci in (1, 0):
        args = cb.cholinv.info(ci, 1, a.bcm, "U")
        cb.cholinv.factor(A, args, topo)
        bc = _lib.lib().capital_cholinv_bc_dimension(n, 1, 1, a.bcm)
        s1 = n >> 1
        skipped = ci == 0 and n > bc
        ms = timed(lambda: cb.cholinv.inverse(args, topo), a.iters)
        ctx.profile_begin()
        Ainv = cb.cholinv.inverse(args, topo)
        gemm_ms, gemm_fl, gemm_n = ctx.profile_end()
        flops = inverse_flops(n, s1, skipped)
        R = cb.cholinv.construct_R(args)
        ms_potri = timed(lambda: torch.cholesky_inverse(R, upper=True), a.ref_iters, warmup=1)
        ref = torch.cholesky_inverse(R, upper=True)
        del R
        iu = torch.triu_indices(n, n, device="cuda")
        mine = torch.zeros(n, n, dtype=torch.float64, device="cuda")
        mine[iu[0], iu[1]] = Ainv[(iu[1] * (iu[1] + 1)) // 2 + iu[0]]
        del iu
        err = ((mine - torch.triu(ref)).abs().max() / ref.abs().max()).item()
        del mine, ref, Ainv
        res = cb.cholinv.inverse_residual(A, cb.cholinv.inverse(args, topo), args, topo)
        rec = {"complete_inv": ci, "rinv12_rebuilt": skipped, "ms": round(ms, 3), "flops": flops,
               "TFLOPs": round(flops / (ms * 1e-3) / 1e12, 2), "of_dmma_peak": round(flops / (ms * 1e-3) / 1e12 / peak, 3),
               "gemm_launches": gemm_n, "gemm_ms": round(gemm_ms, 3), "gemm_TFLOPs": round(gemm_fl / (gemm_ms * 1e-3) / 1e12, 2),
               "gemm_of_dmma_peak": round(gemm_fl / (gemm_ms * 1e-3) / 1e12 / peak, 3),
               "cholesky_inverse_ms": round(ms_potri, 2), "speedup_vs_cholesky_inverse": round(ms_potri / ms, 2),
               "linalg_inv_ms": round(ms_inv, 2), "speedup_vs_linalg_inv": round(ms_inv / ms, 2),
               "rel_diff_vs_cholesky_inverse": err, "residual": res}
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
