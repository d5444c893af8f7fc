"""Timing of cholinv::solve (capital_cholinv_solve_f64) on one GPU against the copy bandwidth and cuSOLVER.

    python tools/solve_bench.py [--n 16384] [--bcm -5] [--iters 50] [--out FILE]

For complete_inv in {0, 1} and nrhs in {1, 8, 16, 32, 256}: factor once (device buffers), warm up, then time `iters` solves with CUDA
events.  The bytes a solve must move are computed from the shapes (every factor element of every window once per product and panel,
plus B in and X out) and set against a device-to-device copy timed in the same run.  The baseline is torch.cholesky_solve (cuSOLVER
potrs) on the same factor R.  The card name and power limit are read in the same run.  Writes one JSON document."""
import argparse, ctypes as C, json, os, subprocess, sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch
import capital_b200 as cb
from capital_b200 import _lib

W = 32  # panel width of the kernel (SOLVE_W)


def card():
    q = "name,power.limit,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()), f"--query-gpu={q}", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        name, power, clk = [s.strip() for s in out.split(",")]
        return {"gpu": name, "power_limit": power, "sm_max_clock": clk}
    except Exception as e:  # noqa: reported, not fatal
        return {"gpu": torch.cuda.get_device_name(), "power_limit": f"not read ({e!r})"}


def timed(fn, iters, warmup=5):
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


def copy_bandwidth(nbytes=1 << 30, iters=20):
    x = torch.empty(nbytes // 8, dtype=torch.float64, device="cuda").uniform_()
    y = torch.empty_like(x)
    ms = timed(lambda: y.copy_(x), iters)
    return 2 * nbytes / (ms * 1e-3)  # read + write


def tri(m):
    return m * (m + 1) // 2


def solve_bytes(n, s1, skipped, k):
    """HBM bytes a solve of k right-hand sides needs: each product reads its factor window once per panel of W; B in, X out."""
    panels = -(-k // W)
    if skipped:
        elems = 2 * tri(s1) + 2 * tri(n - s1) + 2 * s1 * (n - s1)
    else:
        elems = 2 * tri(n)
    return 8 * (elems * panels + 2 * n * k)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=16384)
    ap.add_argument("--bcm", type=int, default=-5)
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--nrhs", default="1,8,16,32,256")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("solve_bench needs a GPU (no CPU fallback)")
    torch.cuda.set_device(0)
    n = a.n
    topo = cb.topo.square(1, 0, 1)
    ctx = topo.context()
    A = cb.matrix(n, n, 1, 1).distribute_symmetric(topo)
    bw = copy_bandwidth()
    doc = {"tool": "tools/solve_bench.py", **card(), "n": n, "bc_mult_dim": a.bcm, "iters": a.iters, "panel_width": W,
           "copy_bandwidth_GBps": round(bw / 1e9, 1), "records": []}
    g = torch.Generator(device="cuda").manual_seed(1)
    for ci in (1, 0):
        args = cb.cholinv.info(ci, 1, a.bcm, "U")
        cb.cholinv.factor(A, args, topo)
        bc = _lib.lib().capital_cholinv_bc_dimension(n, 1, 1, a.bcm)
        s1 = n >> 1
        skipped = ci == 0 and n > bc
        Rd = cb.cholinv.construct_R(args)  # dense upper R for the cuSOLVER baseline (same factor)
        ca = args._c()
        for k in [int(s) for s in a.nrhs.split(",")]:
            Bc = torch.rand(k, n, dtype=torch.float64, device="cuda", generator=g) - 0.5  # column-major n x k
            Xc = torch.empty_like(Bc)

            def ours():
                ctx.check(_lib.lib().capital_cholinv_solve_f64(ctx.handle, n, C.byref(ca), _lib.UPPERTRI_PACKED, args.R.data_ptr(),
                                                               args.Rinv.data_ptr(), k, Bc.data_ptr(), n, Xc.data_ptr(), n))

            ms = timed(ours, a.iters)
            Bt = Bc.t().contiguous()
            ms_ref = timed(lambda: torch.cholesky_solve(Bt, Rd, upper=True), a.iters)
            err = ((Xc.t() - torch.cholesky_solve(Bt, Rd, upper=True)).abs().max() / Xc.abs().max()).item()
            nbytes = solve_bytes(n, s1, skipped, k)
            rate = nbytes / (ms * 1e-3)
            elems = (nbytes // 8 - 2 * n * k) // -(-k // W)  # factor elements of all products (one panel's pass)
            rec = {"complete_inv": ci, "nrhs": k, "ms": round(ms, 4), "bytes": nbytes, "GBps": round(rate / 1e9, 1),
                   "of_copy_bw": round(rate / bw, 3), "fp64_TFLOPs": round(2 * elems * k / (ms * 1e-3) / 1e12, 2),
                   "cusolver_ms": round(ms_ref, 4), "speedup_vs_cusolver": round(ms_ref / ms, 2), "rel_diff_vs_cusolver": err}
            doc["records"].append(rec)
            print(json.dumps(rec), flush=True)
        del Rd
    text = json.dumps(doc, indent=1)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(text + "\n")
    print(text)


if __name__ == "__main__":
    main()
