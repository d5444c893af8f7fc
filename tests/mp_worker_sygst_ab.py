"""Grid worker of cholinv::sygst for itype 2 and 3 and of apply_R / apply_RT (run under torch.distributed.run, one process per rank).
Exits non-zero on a mismatch.

2 ranks: the 2x1x1 grid, 4: 1x2x2, 8: 2x2x2.  B = the diagonally dominant generator matrix, A = the plain symmetric generator matrix.
For n in {512, 768}, complete_inv in {0, 1} and both output structures: the factor's R holds zeros on the local-diagonal slots of ranks
with y > x (apply_R reads its full window); the assembled C against LAPACK's dsygst (itype 2 and 3) of the assembled global matrices,
bit-identical layer replicas, an exactly symmetric rect output, NaN in A's strict global upper triangle changing no bit, the host-pointer
path equal to the device path; apply_R and apply_RT against numpy and bit-identical on every rank, in place too.  And d not dividing n
is rejected."""
import ctypes as C
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
from sygst_ab_reference import bound, dsygst_full
from sygst_reference import U
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
        for ci in (0, 1):
            for serialize in (True, False):
                args = cb.cholinv.info(ci, 1, -2, "U", serialize=serialize)
                cb.cholinv.factor(Bm, args, topo)
                # apply_R reads the full local window of R: below the global diagonal it must hold zeros
                zdiag = bool((torch.diagonal(cb.cholinv.construct_R(args)) == 0).all()) if topo.y > topo.x else True
                zdiag = all(gather(torch.tensor([int(zdiag)], device="cpu" if gloo else "cuda"))[i].item() for i in range(world))
                r = np.triu(assemble([p.numpy() for p in gather(args.R)], coords, n, d, serialize))
                refs = {it: dsygst_full(a, r, it) for it in (2, 3)}
                bnd = bound(a, r)
                Cl = cb.cholinv.sygst(Am, args, topo, itype=2)
                parts = gather(Cl)
                layers = all(torch.equal(parts[i], parts[j]) for i in range(world) for j in range(world) if coords[i][:2] == coords[j][:2])
                M = assemble([p.numpy() for p in parts], coords, n, d, serialize)
                # the GPU result and LAPACK's each lie within the first-order bound of the exact C
                ratio = max(float((np.abs(M - refs[it]) / bnd).max()) for it in (2, 3))
                within = ratio <= 2
                err = float(np.abs(M - refs[2]).max() / np.abs(refs[2]).max())
                sym = serialize or np.array_equal(M, M.T)
                sym &= all(np.all(np.diag(co.unpack_upper(p.numpy(), L)) == 0) for p, (x, y, _) in zip(parts, coords)
                           if serialize and y > x)
                same3 = torch.equal(cb.cholinv.sygst(Am, args, topo, itype=3), Cl)
                nan_free = torch.equal(cb.cholinv.sygst(Ap, args, topo, itype=2), Cl)
                h = cb.cholinv.info(ci, 1, -2, "U", serialize=serialize)
                h.R, h.Rinv, h.local_dim, h.global_dim = args.R.cpu(), args.Rinv.cpu(), args.local_dim, n
                Ch = cb.cholinv.sygst(cb.matrix(n, n, d, d, data=Am.data.cpu()), h, topo, itype=2)
                host_same = (not Ch.is_cuda) and torch.equal(Ch, Cl.cpu())
                ok &= zdiag and within and layers and sym and same3 and nan_free and host_same
                msgs.append(f"n={n} ci={ci} packed={serialize}: R-zero-below={zdiag} err={err:.1e} err/bound={ratio:.2f} within-2-bounds={within} "
                            f"layers-identical={layers} symmetric={sym} itype3-same={same3} nan-free={nan_free} host==device={host_same}")
                # X = R B and X = R^T B: bit-identical everywhere, in place as well
                for k in (1, 33):
                    Bv = torch.from_numpy(np.random.default_rng(n + k).standard_normal((n, k))).cuda()
                    for trans, fn, F in ((0, cb.cholinv.apply_R, r), (1, cb.cholinv.apply_RT, r.T)):
                        X = fn(args, Bv, topo)
                        bv = Bv.cpu().numpy()
                        ref = F @ bv
                        dev = np.abs(X.cpu().numpy() - ref)
                        e = float(dev.max() / np.abs(ref).max())
                        within_r = bool(np.all(dev <= 2 * n * U * (np.abs(F) @ np.abs(bv))))  # two dot products of n terms
                        Xs = gather(X)
                        same = all(torch.equal(Xs[0], p) for p in Xs)
                        buf = Bv.t().clone(memory_format=torch.contiguous_format)
                        ctx = topo.context()
                        ca = args._c()
                        ctx.check(_lib.lib().capital_cholinv_apply_r_f64(ctx.handle, n, C.byref(ca),
                                                                         _lib.UPPERTRI_PACKED if serialize else _lib.RECT,
                                                                         args.R.data_ptr(), trans, k, buf.data_ptr(), n, buf.data_ptr(), n))
                        inplace = torch.equal(buf.t(), X)
                        ok &= within_r and same and inplace
                        msgs.append(f"n={n} ci={ci} packed={serialize} k={k} trans={trans}: err={e:.1e} within-bound={within_r} ranks-identical={same} "
                                    f"in-place={inplace}")
    if d > 1:
        n = 2 * 256 + 1  # d = 2 does not divide it
        L = -(-n // d)
        args = cb.cholinv.info(1, 1, -2, "U")
        args.R = torch.zeros(L * (L + 1) // 2, dtype=torch.float64, device="cuda")
        args.Rinv = torch.zeros_like(args.R)
        args.local_dim, args.global_dim = L, n
        rejected = True
        for call in (lambda: cb.cholinv.sygst(cb.matrix(n, n, d, d), args, topo, itype=2),
                     lambda: cb.cholinv.apply_R(args, torch.zeros(n, dtype=torch.float64, device="cuda"), topo)):
            try:
                call()
                rejected = False
            except _lib.CapitalError as e:
                rejected &= e.status == _lib.ERR_UNSUPPORTED
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
