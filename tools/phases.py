"""Where a warm one-GPU cholinv::factor step goes: prologue, recursion and tail, from CUDA events around every launch.
    python tools/phases.py [n] [bc_mult_dim] [out.json]
prologue  = step start -> end of the last zeroing / input copy on the caller's stream, and the start of the first base case;
recursion = first base case -> last launch of the chain and the deferred streams;
tail      = what runs after that (the packing of the columns not packed early), i.e. the exposed end of the step.
Also: the plain step time (no timeline), the card's name and power limit, and whether a device-to-device cudaMemcpy2DAsync runs on
a copy engine (its time barely changes while a long FP64 GEMM holds every SM) or on the SMs (it waits for the GEMM)."""
import ctypes as C, glob, json, os, subprocess, sys
import numpy as np
import torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import capital_b200 as cb

CHAIN, DEFERRED, USER, COPYIN, COPYOUT = 1, (2, 3, 4), 0, 10, 11


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as ex:  # noqa
        q = f"nvidia-smi failed: {ex!r}"
    return q


def phases(tl):
    t0 = tl[:, 2].min()
    tl = tl.copy()
    tl[:, 2:4] -= t0
    sid, kind, sub = tl[:, 0].astype(int), tl[:, 1].astype(int), tl[:, 4].astype(int)
    bc = tl[(kind == 3) | (kind == 4)]
    first_bc = float(bc[:, 2].min())
    pro = tl[(kind == 8) & np.isin(sub, (2, 4, 5)) & (tl[:, 2] < first_bc) & ((sid == USER) | (sid == COPYIN))]
    rec_mask = (sid == CHAIN) | np.isin(sid, DEFERRED)
    rec_end = float(tl[rec_mask, 3].max())
    end = float(tl[:, 3].max())
    tail = tl[(tl[:, 3] > rec_end) & (kind == 8) & (sub == 3)]
    copy = tl[(kind == 8) & (sub == 2)]
    return {"first_base_case_start_ms": first_bc,
            "prologue_end_ms": float(pro[:, 3].max()) if len(pro) else 0.0,
            "prologue_busy_ms": float((pro[:, 3] - pro[:, 2]).sum()) if len(pro) else 0.0,
            "input_copy_ms": [round(float(b - a), 4) for a, b in copy[:, 2:4]],
            "recursion_ms": rec_end - first_bc,
            "tail_ms": end - rec_end,
            "tail_packs": [[int(r[5]), int(r[6]), round(float(r[3] - r[2]), 4)] for r in tail],
            "span_ms": end, "launches": int(len(tl))}


def copy_engine_probe(n=16384):
    import nvidia.cuda_runtime
    rt = C.CDLL(glob.glob(os.path.join(nvidia.cuda_runtime.__path__[0], "lib", "libcudart.so*"))[0])
    src = torch.empty((n, n), dtype=torch.float64, device="cuda")
    dst = torch.empty_like(src)
    a = torch.randn(8192, 8192, dtype=torch.float64, device="cuda")
    s_cp, s_mm = torch.cuda.Stream(), torch.cuda.Stream()

    def cp():  # upper-triangle-sized 2D copy with a pitch: n/2 columns of n rows
        rt.cudaMemcpy2DAsync(C.c_void_p(dst.data_ptr()), C.c_size_t(n * 8), C.c_void_p(src.data_ptr()), C.c_size_t(n * 8),
                             C.c_size_t(n * 8), C.c_size_t(n // 2), 3, C.c_void_p(s_cp.cuda_stream))

    def timed(with_mm):
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        if with_mm:
            with torch.cuda.stream(s_mm):
                for _ in range(3):
                    torch.mm(a, a)
        with torch.cuda.stream(s_cp):
            e0.record()
            cp()
            e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1)

    for w in (False, True):
        timed(w)
    alone = min(timed(False) for _ in range(3))
    busy = min(timed(True) for _ in range(3))
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(3):
        torch.mm(a, a)
    e1.record()
    torch.cuda.synchronize()
    return {"bytes": n * n // 2 * 8, "alone_ms": alone, "beside_gemm_ms": busy, "gemm_x3_ms": e0.elapsed_time(e1)}


def main():
    n = int(sys.argv[1]) if len(sys.argv) > 1 else 16384
    bcm = int(sys.argv[2]) if len(sys.argv) > 2 else -5
    out = sys.argv[3] if len(sys.argv) > 3 else None
    torch.cuda.set_device(0)
    topo = cb.topo.square(1, 0, 1)
    ctx = topo.context()
    A = cb.matrix(n, n, 1, 1).distribute_symmetric(topo)
    args = cb.cholinv.info(0, 1, bcm, "U")
    for _ in range(3):
        cb.cholinv.factor(A, args, topo)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(5):
        cb.cholinv.factor(A, args, topo)
    e1.record()
    torch.cuda.synchronize()
    rec = {"card": card(), "n": n, "bc_mult_dim": bcm, "step_ms": e0.elapsed_time(e1) / 5,
           "counters_per_step": None, "timeline": []}
    ctx.reset_counters()
    cb.cholinv.factor(A, args, topo)
    c = ctx.counters()
    rec["counters_per_step"] = {"kernel_launches": c.kernel_launches, "gemm_launches": c.gemm_launches, "gemm_flops": c.gemm_flops}
    for _ in range(3):
        ctx.timeline_begin()
        cb.cholinv.factor(A, args, topo)
        rec["timeline"].append(phases(ctx.timeline_end()))
    del A, args
    ctx.release_workspace()
    torch.cuda.empty_cache()
    rec["memcpy2d_d2d"] = copy_engine_probe(n)
    s = json.dumps(rec)
    print(s)
    if out:
        os.makedirs(os.path.dirname(os.path.abspath(out)), exist_ok=True)
        with open(out, "w") as f:
            f.write(s + "\n")


if __name__ == "__main__":
    main()
