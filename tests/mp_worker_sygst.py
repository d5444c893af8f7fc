"""Grid worker of cholinv::sygst and apply_Rinv / apply_RinvT (run under torch.distributed.run, one process per rank).  Exits non-zero
on a mismatch.

2 ranks: the 2x1x1 grid, 4: 1x2x2, 8: 2x2x2.  B = the diagonally dominant generator matrix, A = the plain symmetric generator matrix.
For n in {512, 768}, complete_inv in {0, 1} and both output structures: the assembled C against LAPACK's dsygst of the assembled
global matrices, bit-identical layer replicas, an exactly symmetric rect output, NaN in A's strict global upper triangle changing no bit,
the host-pointer path equal to the device path, factor -> sygst -> factor giving identical factors, and apply_Rinv(apply_RinvT(B))
equal to solve(B) bit for bit; and d not dividing n is rejected."""
import os, sys
import numpy as np
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import capital_b200 as cb
from capital_b200 import _lib
from oracle import capital_oracle as co
from grid_edges_reference import assemble
from sygst_reference import bound, dsygst_full


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

    def gather(t):
        mine = t.cpu() if gloo else t
        parts = [torch.empty_like(mine) for _ in range(world)]
        dist.all_gather(parts, mine)
        return [p.cpu() for p in parts]

    ok = True
    msgs = []
    for n in (512, 768):
        b = co.spd_global(n)
        a = b - n * np.eye(n)  # the generator's plain symmetric matrix: the same draws without the diagonal shift
        Bm = cb.matrix(n, n, d, d).distribute_symmetric(topo)
        Am = cb.matrix(n, n, d, d).distribute_symmetric(topo, False)
        L = Am.num_rows_local
        # A with NaN in its strict global upper triangle: local (r, c) is global (y + d r, x + d c)
        gy = topo.y + d * torch.arange(L, device="cuda").view(L, 1)
        gx = topo.x + d * torch.arange(L, device="cuda").view(1, L)
        poisoned = Am.view2d().clone()
        poisoned[gy < gx] = float("nan")
        Ap = cb.matrix(n, n, d, d, data=poisoned.t().contiguous().view(-1))
        r = None
        for ci in (0, 1):
            for serialize in (True, False):
                args = cb.cholinv.info(ci, 1, -2, "U", serialize=serialize)
                cb.cholinv.factor(Bm, args, topo)
                R0, Ri0 = args.R.clone(), args.Rinv.clone()
                if r is None:
                    r = assemble([p.numpy() for p in gather(args.R)], coords, n, d, serialize) if serialize else None
                Cl = cb.cholinv.sygst(Am, args, topo)
                parts = gather(Cl)
                layers = all(torch.equal(parts[i], parts[j]) for i in range(world) for j in range(world) if coords[i][:2] == coords[j][:2])
                M = assemble([p.numpy() for p in parts], coords, n, d, serialize)
                ref = dsygst_full(a, np.triu(r))
                within = bool(np.all(np.abs(M - ref) <= bound(a, np.linalg.inv(np.triu(r)))))
                err = float(np.abs(M - ref).max() / np.abs(ref).max())
                sym = serialize or np.array_equal(M, M.T)
                sym &= all(np.all(np.diag(co.unpack_upper(p.numpy(), L)) == 0) for p, (x, y, _) in zip(parts, coords)
                           if serialize and y > x)
                nan_free = torch.equal(cb.cholinv.sygst(Ap, args, topo), Cl)
                h = cb.cholinv.info(ci, 1, -2, "U", serialize=serialize)
                h.R, h.Rinv, h.local_dim, h.global_dim = args.R.cpu(), args.Rinv.cpu(), args.local_dim, n
                Ch = cb.cholinv.sygst(cb.matrix(n, n, d, d, data=Am.data.cpu()), h, topo)
                host_same = (not Ch.is_cuda) and torch.equal(Ch, Cl.cpu())
                cb.cholinv.factor(Bm, args, topo)
                refactor = torch.equal(R0, args.R) and torch.equal(Ri0, args.Rinv)
                ok &= within and layers and sym and nan_free and host_same and refactor
                msgs.append(f"n={n} ci={ci} packed={serialize}: err={err:.1e} within-bound={within} layers-identical={layers} "
                            f"symmetric={sym} nan-free={nan_free} host==device={host_same} refactor-identical={refactor}")
            # the two halves of the solve, applied in turn, are the solve
            args = cb.cholinv.info(ci, 1, -2, "U")
            cb.cholinv.factor(Bm, args, topo)
            for k in (1, 33):
                Bv = torch.from_numpy(np.random.default_rng(n + k).standard_normal((n, k))).cuda()
                Y = cb.cholinv.apply_RinvT(args, Bv, topo)
                X = cb.cholinv.apply_Rinv(args, Y, topo)
                S = cb.cholinv.solve(args, Bv, topo)
                halves = torch.equal(X, S)
                err = float(np.abs(Y.cpu().numpy() - np.linalg.solve(np.triu(r).T, Bv.cpu().numpy())).max())
                same = all(torch.equal(gather(X)[0], p) for p in gather(X))
                ok &= halves and same and err <= 1e-12
                msgs.append(f"n={n} ci={ci} k={k}: apply_Rinv(apply_RinvT(B)) == solve(B): {halves} ranks-identical={same} "
                            f"R^-T B err={err:.1e}")
    if d > 1:
        n = 2 * 256 + 1  # d = 2 does not divide it
        L = -(-n // d)
        args = cb.cholinv.info(1, 1, -2, "U")
        args.R = torch.zeros(L * (L + 1) // 2, dtype=torch.float64, device="cuda")
        args.Rinv = torch.zeros_like(args.R)
        args.local_dim, args.global_dim = L, n
        try:
            cb.cholinv.sygst(cb.matrix(n, n, d, d), args, topo)
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
