"""Timeline of one cholinv::factor (CUDA events around every launch; the image has no nsys).
    python tools/timeline.py [n] [bc_mult_dim]                       one GPU
    torchrun --nproc-per-node N tools/timeline.py [n] [bcm] [c]      N GPUs (rank 0 prints; every rank writes $CAPITAL_OUT_DIR/timeline_r<rank>.npy, default .)
Prints per-stream busy time, per-kind totals, the chain's idle gaps and its longest flag waits."""
import os, sys
import numpy as np
import torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import capital_b200 as cb

KIND = {1: "gemm128", 2: "gemm64", 3: "basecase", 4: "leaf", 5: "wait", 6: "signal", 7: "dma", 8: "layout"}
SID = {0: "user", 1: "chain", 2: "far0", 3: "far1", 4: "far2", 5: "push0", 6: "push1", 7: "push2", 8: "push3", 9: "pushB", 10: "copyin", 11: "copyout"}


def covered(a, b, iv):
    """length of [a, b] covered by the union of the intervals iv (rows of start, end)"""
    seg = sorted((max(a, x), min(b, y)) for x, y in iv if y > a and x < b)
    tot, cs, ce = 0.0, None, None
    for x, y in seg:
        if cs is None or x > ce:
            tot += (ce - cs) if cs is not None else 0.0
            cs, ce = x, y
        else:
            ce = max(ce, y)
    return tot + ((ce - cs) if cs is not None else 0.0)


def main():
    world = int(os.environ.get("WORLD_SIZE", "1")); rank = int(os.environ.get("RANK", "0")); lr = int(os.environ.get("LOCAL_RANK", "0"))
    n = int(sys.argv[1]) if len(sys.argv) > 1 else 16384
    bcm = int(sys.argv[2]) if len(sys.argv) > 2 else -5
    c = int(sys.argv[3]) if len(sys.argv) > 3 else 1
    torch.cuda.set_device(lr)
    if world > 1:
        import torch.distributed as dist
        dist.init_process_group("nccl", device_id=torch.device("cuda", lr))
    topo = cb.topo.square(world, rank, c)
    ctx = topo.context()
    A = cb.matrix(n, n, topo.d, topo.d).distribute_symmetric(topo)
    args = cb.cholinv.info(0, 1, bcm, "U")
    for _ in range(3):
        cb.cholinv.factor(A, args, topo)
    if world > 1:
        dist.barrier()
    torch.cuda.synchronize()
    ctx.timeline_begin()
    cb.cholinv.factor(A, args, topo)
    tl = ctx.timeline_end()
    out = os.environ.get("CAPITAL_OUT_DIR", ".")
    os.makedirs(out, exist_ok=True)
    np.save(os.path.join(out, f"timeline_r{rank}.npy"), tl)
    if rank == 0:
        t0, t1 = tl[:, 2].min(), tl[:, 3].max()
        print(f"n={n} bcm={bcm} world={world}: {len(tl)} launches, span {t1 - t0:.2f} ms (with event overhead)")
        # one GPU: far updates (and bands) of the top-level node / of the other nodes, T^T products, packing of finished columns
        sids = {**SID, **({2: "far-top", 3: "far-low", 4: "tt", 11: "pack"} if world == 1 else {})}
        for sid in sorted(set(tl[:, 0].astype(int))):
            s = tl[tl[:, 0] == sid]
            busy = (s[:, 3] - s[:, 2]).sum()
            print(f"  stream {sids.get(sid, sid):8s}: {len(s):5d} launches, busy {busy:8.2f} ms, first {s[:, 2].min():7.2f} last {s[:, 3].max():7.2f}")
            for k in sorted(set(s[:, 1].astype(int))):
                kk = s[s[:, 1] == k]
                print(f"      {KIND.get(k, k):9s} x{len(kk):5d}  total {(kk[:, 3] - kk[:, 2]).sum():8.2f} ms  max {(kk[:, 3] - kk[:, 2]).max():7.3f}")
        ch = tl[tl[:, 0] == 1]
        ch = ch[np.argsort(ch[:, 2])]
        gaps = ch[1:, 2] - ch[:-1, 3]
        print(f"  chain idle between launches: {gaps[gaps > 0].sum():.2f} ms over {np.sum(gaps > 0.01)} gaps > 10 us; largest {np.sort(gaps)[-5:]}")
        # how much of the base cases' time has a GEMM of another stream running beside it (first / second half in issue order)
        bc = ch[ch[:, 1] == 3]
        other = tl[(tl[:, 0] != 1) & np.isin(tl[:, 1], (1, 2))][:, 2:4]
        if len(bc):
            cov = np.array([covered(a, b, other) for a, b in bc[:, 2:4]])
            d = bc[:, 3] - bc[:, 2]
            h = len(bc) // 2
            print(f"  basecase with a deferred GEMM beside it: first half {cov[:h].sum():.2f} of {d[:h].sum():.2f} ms, "
                  f"second half {cov[h:].sum():.2f} of {d[h:].sum():.2f} ms")
        w = ch[ch[:, 1] == 5]
        if len(w):
            d = w[:, 3] - w[:, 2]
            print(f"  chain flag waits: {len(w)} total {d.sum():.2f} ms; longest {np.sort(d)[-8:]}")
    if world > 1:
        dist.barrier()
        cb.topo.release_contexts()
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
