"""Grid worker of cholinv::solve (run under torch.distributed.run, one process per rank).  Exits non-zero on a mismatch.

2 ranks: the 2x1x1 grid, 4: 1x2x2, 8: 2x2x2.  For n in {512, 768}, complete_inv in {0, 1} and nrhs in {1, 33}: X against the numpy
solve, X bit-identical on every rank, the host-pointer path equal to the device path; and d not dividing n is rejected."""
import os, sys
import numpy as np
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import capital_b200 as cb
from capital_b200 import _lib
from oracle import capital_oracle as co


def main():
    rank, world, lr = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    if os.environ.get("CAPITAL_MP_SAME_DEVICE"):
        torch.cuda.set_device(0)
        dist.init_process_group("gloo")
    else:
        torch.cuda.set_device(lr)
        dist.init_process_group("nccl", device_id=torch.device("cuda", lr))
    c = {2: 2, 4: 1, 8: 2}[world]
    topo = cb.topo.square(world, rank, c)
    d = topo.d
    ok = True
    msgs = []
    for n in (512, 768):
        a = co.spd_global(n)
        A = cb.matrix(n, n, d, d).distribute_symmetric(topo)
        for ci in (0, 1):
            args = cb.cholinv.info(ci, 1, -2, "U")
            cb.cholinv.factor(A, args, topo)
            for k in (1, 33):
                B = torch.from_numpy(np.random.default_rng(n + k).standard_normal((n, k))).cuda()
                X = cb.cholinv.solve(args, B, topo)
                ref = np.linalg.solve(a, B.cpu().numpy())
                err = float(np.abs(X.cpu().numpy() - ref).max() / np.abs(ref).max())
                # every rank holds the same bits
                mine = X if dist.get_backend() != "gloo" else X.cpu()
                parts = [torch.empty_like(mine) for _ in range(world)]
                dist.all_gather(parts, mine)
                same = all(torch.equal(parts[0], p) for p in parts)
                # host pointers: factors, B and X on the host
                h = cb.cholinv.info(ci, 1, -2, "U")
                h.R, h.Rinv, h.local_dim, h.global_dim = args.R.cpu(), args.Rinv.cpu(), args.local_dim, n
                Xh = cb.cholinv.solve(h, B.cpu(), topo)
                host_same = (not Xh.is_cuda) and torch.equal(Xh, X.cpu())
                ok &= err <= 1e-12 and same and host_same
                msgs.append(f"n={n} ci={ci} k={k}: err={err:.1e} ranks-identical={same} host==device={host_same}")
    if d > 1:
        n = 2 * 256 + 1  # d = 2 does not divide it
        L = -(-n // d)
        args = cb.cholinv.info(1, 1, -2, "U")
        args.R = torch.zeros(L * (L + 1) // 2, dtype=torch.float64, device="cuda")
        args.Rinv = torch.zeros_like(args.R)
        args.local_dim, args.global_dim = L, n
        try:
            cb.cholinv.solve(args, torch.zeros(n, 1, dtype=torch.float64, device="cuda"), topo)
            rejected = False
        except _lib.CapitalError as e:
            rejected = e.status == _lib.ERR_UNSUPPORTED
        ok &= rejected
        msgs.append(f"d does not divide n: rejected={rejected}")
    flag = torch.tensor([0 if ok else 1], device="cuda")
    if dist.get_backend() == "gloo":
        flag = flag.cpu()
    dist.all_reduce(flag)
    if rank == 0:
        print(("MP_OK " if flag.item() == 0 else "MP_FAIL ") + " | ".join(msgs), flush=True)
    dist.barrier()
    cb.topo.release_contexts()
    dist.destroy_process_group()
    sys.exit(0 if flag.item() == 0 else 1)


if __name__ == "__main__":
    main()
