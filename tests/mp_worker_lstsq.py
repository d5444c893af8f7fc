"""Grid worker of cacqr::lstsq / apply_QT / apply_Q on the 1D row grid topo.rect(P, rank, 1) (run under torch.distributed.run, one
process per rank).  Exits non-zero on a mismatch.

For m in {4096, 4099 (d does not divide it)}, n = 96, nrhs in {1, 33}: X and Y against numpy on the assembled global A, each rank's
rows of Q Z against numpy, X bit-identical on every rank, the host-pointer path equal to the device path, and factor -> lstsq ->
factor bit-identical.  On 8 ranks, the 2 x 2 x 2 grid rect(8, rank, 2) is rejected with CAPITAL_ERR_UNSUPPORTED."""
import os, sys
import numpy as np
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import capital_b200 as cb
from capital_b200 import _lib


def main():
    rank, world, lr = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    if os.environ.get("CAPITAL_MP_SAME_DEVICE"):
        torch.cuda.set_device(0)
        dist.init_process_group("gloo")
    else:
        torch.cuda.set_device(lr)
        dist.init_process_group("nccl", device_id=torch.device("cuda", lr))
    gloo = dist.get_backend() == "gloo"

    def gather(t):
        mine = t.cpu() if gloo else t
        parts = [torch.empty_like(mine) for _ in range(world)]
        dist.all_gather(parts, mine)
        return [p.cpu() for p in parts]

    topo = cb.topo.rect(world, rank, 1)
    d = world
    ok = True
    msgs = []
    n = 96
    for m in (4096, 4099):
        rows = -(-m // d)
        A = cb.matrix(n, m, 1, d).distribute_random(topo, rank)
        args = cb.cacqr.info(2, cb.cholinv.info(0, 1, 0, "U"))
        cb.cacqr.factor(A, args, topo)
        Q0, R0 = args.Q.clone(), args.R.clone()
        # the global A from every rank's rows (global row gy on rank gy mod d, local row gy / d)
        blocks = gather(A.view2d().contiguous())
        a = np.zeros((m, n))
        for y in range(d):
            cnt = len(range(y, m, d))
            a[y::d] = blocks[y].numpy()[:cnt]
        for k in (1, 33):
            rng = np.random.default_rng(m + k)
            b = rng.standard_normal((m, k))
            z = rng.standard_normal((n, k))
            mine = np.zeros((rows, k))
            mine[:len(range(rank, m, d))] = b[rank::d]
            B = torch.from_numpy(mine).cuda()
            X = cb.cacqr.lstsq(args, B, topo)
            Y = cb.cacqr.apply_QT(B, args, topo)
            Cq = cb.cacqr.apply_Q(torch.from_numpy(z).cuda(), args, topo)
            ref = np.linalg.lstsq(a, b, rcond=None)[0]
            err = float(np.abs(X.cpu().numpy() - ref).max() / np.abs(ref).max())
            qs = gather(cb.cacqr.construct_Q(args).contiguous())
            q = np.zeros((m, n))
            for y in range(d):
                q[y::d] = qs[y].numpy()[:len(range(y, m, d))]
            qtb = q.T @ b
            err_y = float(np.abs(Y.cpu().numpy() - qtb).max() / np.abs(qtb).max())
            qz = (q @ z)[rank::d]
            err_c = float(np.abs(Cq.cpu().numpy()[:len(qz)] - qz).max() / np.abs(qz).max())
            pad_zero = bool((Cq.cpu()[len(qz):] == 0).all())  # the pad row of Q is zero, so is its row of Q Z
            same = all(torch.equal(p, X.cpu()) for p in gather(X)) and all(torch.equal(p, Y.cpu()) for p in gather(Y))
            h = cb.cacqr.info(2, cb.cholinv.info(0, 1, 0, "U"))
            h.Q, h.R, h.n, h.rows_local, h.m_global, h.n_global = args.Q.cpu(), args.R.cpu(), n, rows, m, n
            Xh = cb.cacqr.lstsq(h, B.cpu(), topo)
            host_same = (not Xh.is_cuda) and torch.equal(Xh, X.cpu()) and torch.equal(cb.cacqr.apply_QT(B.cpu(), h, topo), Y.cpu())
            ok &= err <= 1e-11 and err_y <= 1e-12 and err_c <= 1e-12 and pad_zero and same and host_same
            msgs.append(f"m={m} k={k}: err={err:.1e} errY={err_y:.1e} errQZ={err_c:.1e} ranks-identical={same} host==device={host_same}")
        cb.cacqr.factor(A, args, topo)
        again = torch.equal(Q0, args.Q) and torch.equal(R0, args.R)
        ok &= again
        msgs.append(f"m={m}: factor -> lstsq -> factor identical={again}")
    if world == 8:
        t3 = cb.topo.rect(8, rank, 2)
        A = cb.matrix(n, 256, 2, 2).distribute_random(t3, rank // 2)
        qa = cb.cacqr.info(2, cb.cholinv.info(1, 1, -1, "U"))
        cb.cacqr.factor(A, qa, t3)
        ctx = t3.context()
        buf = torch.zeros(n * A.num_rows_local, dtype=torch.float64, device="cuda")
        st = _lib.lib().capital_cacqr_lstsq_f64(ctx.handle, 256, n, qa.Q.data_ptr(), _lib.UPPERTRI_PACKED, qa.R.data_ptr(), 1,
                                                buf.data_ptr(), A.num_rows_local, buf.data_ptr(), n)
        rejected = st == _lib.ERR_UNSUPPORTED
        ok &= rejected
        msgs.append(f"rect(8, rank, 2): rejected={rejected}")
    flag = torch.tensor([0 if ok else 1], device="cuda")
    if gloo:
        flag = flag.cpu()
    dist.all_reduce(flag)
    if rank == 0:
        print(("MP_OK " if flag.item() == 0 else "MP_FAIL ") + " | ".join(msgs), flush=True)
    else:
        print(" | ".join(msgs), flush=True)
    dist.barrier()
    cb.topo.release_contexts()
    dist.destroy_process_group()
    sys.exit(0 if flag.item() == 0 else 1)


if __name__ == "__main__":
    main()
