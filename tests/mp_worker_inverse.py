"""Grid worker of cholinv::inverse (run under torch.distributed.run, one process per rank).  Exits non-zero on a mismatch.

2 ranks: the 2x1x1 grid, 4: 1x2x2, 8: 2x2x2.  For n in {512, 768}, complete_inv in {0, 1} and both output structures: the assembled
A^-1 against numpy, bit-identical layer replicas, a rect output whose lower half is the transpose partner's upper half bit for bit
(the assembled matrix is exactly symmetric), the residual, the host-pointer path equal to the device path; and d not dividing n is
rejected."""
import os, sys
import numpy as np
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import capital_b200 as cb
from capital_b200 import _lib
from oracle import capital_oracle as co
from grid_edges_reference import assemble


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
    gloo = dist.get_backend() == "gloo"
    me = torch.tensor([topo.x, topo.y, topo.z], dtype=torch.int64, device="cpu" if gloo else "cuda")
    coords = [torch.empty_like(me) for _ in range(world)]
    dist.all_gather(coords, me)
    coords = [tuple(int(v) for v in t.cpu()) for t in coords]
    ok = True
    msgs = []
    for n in (512, 768):
        ref = np.linalg.inv(co.spd_global(n))
        A = cb.matrix(n, n, d, d).distribute_symmetric(topo)
        for ci in (0, 1):
            for serialize in (True, False):
                args = cb.cholinv.info(ci, 1, -2, "U", serialize=serialize)
                cb.cholinv.factor(A, args, topo)
                Ainv = cb.cholinv.inverse(args, topo)
                mine = Ainv.cpu() if gloo else Ainv
                parts = [torch.empty_like(mine) for _ in range(world)]
                dist.all_gather(parts, mine)
                parts = [p.cpu() for p in parts]
                # layer replicas: the same bits on every z of a face position
                layers = all(torch.equal(parts[i], parts[j]) for i in range(world) for j in range(world)
                             if coords[i][:2] == coords[j][:2])
                M = assemble([p.numpy() for p in parts], coords, n, d, serialize)
                err = float(np.abs(M - ref).max() / np.abs(ref).max())
                sym = serialize or np.array_equal(M, M.T)  # rect: lower half = the partner's upper half, bit for bit
                # packed: zeros on the local-diagonal slots of ranks below the global diagonal (y > x), as in R
                sym &= all(np.all(np.diag(co.unpack_upper(p.numpy(), n // d)) == 0) for p, (x, y, _) in zip(parts, coords)
                           if serialize and y > x)
                res = cb.cholinv.inverse_residual(A, Ainv, args, topo)
                # host pointers: factors and output on the host
                h = cb.cholinv.info(ci, 1, -2, "U", serialize=serialize)
                h.R, h.Rinv, h.local_dim, h.global_dim = args.R.cpu(), args.Rinv.cpu(), args.local_dim, n
                Xh = cb.cholinv.inverse(h, topo)
                host_same = (not Xh.is_cuda) and torch.equal(Xh, Ainv.cpu())
                ok &= err <= 1e-12 and layers and sym and res <= 1e-14 and host_same
                msgs.append(f"n={n} ci={ci} packed={serialize}: err={err:.1e} res={res:.1e} layers-identical={layers} symmetric={sym} "
                            f"host==device={host_same}")
    if d > 1:
        n = 2 * 256 + 1  # d = 2 does not divide it
        L = -(-n // d)
        args = cb.cholinv.info(1, 1, -2, "U")
        args.R = torch.zeros(L * (L + 1) // 2, dtype=torch.float64, device="cuda")
        args.Rinv = torch.zeros_like(args.R)
        args.local_dim, args.global_dim = L, n
        try:
            cb.cholinv.inverse(args, topo)
            rejected = False
        except _lib.CapitalError as e:
            rejected = e.status == _lib.ERR_UNSUPPORTED
        ok &= rejected
        msgs.append(f"d does not divide n: rejected={rejected}")
    flag = torch.tensor([0 if ok else 1], device="cuda")
    if gloo:
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
