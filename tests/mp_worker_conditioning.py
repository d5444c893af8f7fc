"""Grid worker of the conditioning tests (run under torch.distributed.run with 2 ranks, one process per rank).  Exits non-zero on
a mismatch.

cholinv on the 2x1x1 grid and CholeskyQR2 on the 2-rank 1D row grid, with inputs scaled so that the products of neighbouring
pivots leave the double range: R(2^(2k) A) 2^-k and Rinv(2^(2k) A) 2^k against the factors of A on the same grid and against
scipy; Q(A 2^k) against Q(A) and R(A 2^k) 2^-k against R(A) and the numpy restatement."""
import math, os, sys
import numpy as np
import scipy.linalg as sla
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import capital_b200 as cb
from oracle import capital_oracle as co


def rel(x, ref):
    return float(np.abs(np.asarray(x) - ref).max() / np.abs(ref).max())


def main():
    rank, world, lr = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    if os.environ.get("CAPITAL_MP_SAME_DEVICE"):
        torch.cuda.set_device(0)
        dist.init_process_group("gloo")
    else:
        torch.cuda.set_device(lr)
        dist.init_process_group("nccl", device_id=torch.device("cuda", lr))
    assert world == 2
    ok, msgs = True, []
    # cholinv on 2x1x1: d = 1, every rank holds the whole matrix
    topo = cb.topo.square(2, rank, 2)
    n = 1024
    a = co.spd_global(n)
    r_ref = sla.cholesky(a)
    outs = {}
    for k in (0, -412, 412):
        data = torch.from_numpy(np.asfortranarray(a * math.ldexp(1.0, 2 * k)).ravel(order="F").copy()).cuda()
        A = cb.matrix(n, n, 1, 1, data=data)
        args = cb.cholinv.info(1, 1, -2, "U")
        cb.cholinv.factor(A, args, topo)
        outs[k] = (cb.cholinv.construct_R(args).cpu().numpy() * math.ldexp(1.0, -k),
                   cb.cholinv.construct_Rinv(args).cpu().numpy() * math.ldexp(1.0, k))
    for k in (-412, 412):
        eR, eX = rel(outs[k][0], outs[0][0]), rel(outs[k][1], outs[0][1])
        eS = rel(outs[k][0], r_ref)
        good = eR <= 1e-14 and eX <= 1e-14 and eS <= 1e-12
        ok &= good
        msgs.append(f"cholinv 2x1x1 k={k}: errR={eR:.1e} errRinv={eX:.1e} vs scipy {eS:.1e}")
    # CholeskyQR2 on the 1D row grid: rows rank, rank + 2, ... of the global A
    qt = cb.topo.rect(world, rank, 1)
    m, nq = 4096, 256
    A = cb.matrix(nq, m, 1, world).distribute_random(qt, rank)
    blocks = [co.random_local(m, nq, 1, world, 0, y, y) for y in range(world)]
    _, r2 = co.cacqr_1d(blocks, 2)
    res = {}
    for k in (0, -300, 270):
        As = cb.matrix(nq, m, 1, world, data=A.data * math.ldexp(1.0, k))
        args = cb.cacqr.info(2, cb.cholinv.info(0, 1, 0, "U"))
        cb.cacqr.factor(As, args, qt)
        res[k] = (cb.cacqr.construct_Q(args).cpu().numpy(), cb.cacqr.construct_R(args).cpu().numpy() * math.ldexp(1.0, -k))
    for k in (-300, 270):
        eQ, eR, eN = rel(res[k][0], res[0][0]), rel(res[k][1], res[0][1]), rel(res[k][1], r2)
        good = eQ <= 1e-13 and eR <= 1e-13 and eN <= 1e-11
        ok &= good
        msgs.append(f"cacqr2 1D k={k}: errQ={eQ:.1e} errR={eR:.1e} vs numpy {eN:.1e}")
    flag = torch.tensor([0 if ok else 1], device="cpu" if dist.get_backend() == "gloo" else "cuda")
    dist.all_reduce(flag)
    print(("MP_OK " if flag.item() == 0 else "MP_FAIL ") + " | ".join(msgs), flush=True)
    dist.barrier()
    cb.topo.release_contexts()
    dist.destroy_process_group()
    sys.exit(0 if flag.item() == 0 else 1)


if __name__ == "__main__":
    main()
