"""Grid worker of shifted CholeskyQR3 (cacqr num_iter = 3), run under torch.distributed.run with one process per rank.  Exits
non-zero on a failed check.

CAPITAL_SCQR3_GRID picks the grid: "1d" = topo.rect(P, rank, 1), "3d" = the 2 x 2 x 2 grid rect(8, rank, 2), "tune" = the 2 x 4 x 2
grid rect(16, rank, 2).  Every rank builds the same seeded global A with kappa = 1e10 in numpy and takes its cyclic local block.
Checks: residual <= 1e-14 and orthogonality <= 1e-15, R bit-identical wherever it is replicated (every rank on the 1D grid, the
layers and cubes of the 3D / tunable grids), and on the 1D grid lstsq on a consistent system (forward error <= 1e-6) with X
bit-identical on every rank.  CAPITAL_MP_SAME_DEVICE=1 puts every rank on cuda:0 (the ranks bootstrap through the gloo group)."""
import os, sys
import numpy as np
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import capital_b200 as cb
from oracle import capital_oracle as co
from scqr3_reference import ill_conditioned


def main():
    rank, world, lr = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    grid = os.environ.get("CAPITAL_SCQR3_GRID", "1d")
    torch.cuda.set_device(0 if os.environ.get("CAPITAL_MP_SAME_DEVICE") else lr)
    dist.init_process_group("gloo")
    c = 1 if grid == "1d" else 2
    topo = cb.topo.rect(world, rank, c)
    d = world // (c * c)
    m, n = 8192, 128
    a = ill_conditioned(m, n, 1e10, 21)
    loc = co.cyclic_local(a, c, d, topo.x, topo.y)
    A = cb.matrix(n, m, c, d, data=torch.from_numpy(loc.ravel(order="F").copy()).cuda())
    args = cb.cacqr.info(3, cb.cholinv.info(1, 1, -1, "U"))
    cb.cacqr.factor(A, args, topo)
    res, orth = cb.cacqr.validate(A, args, topo)
    ok = res <= 1e-14 and orth <= 1e-15
    msgs = [f"{grid} P={world}: res={res:.1e} orth={orth:.1e}"]
    # R is replicated on the ranks with the same (x, y mod c)
    parts = [None] * world
    dist.all_gather_object(parts, (topo.x, topo.y % c, args.R.cpu().numpy()))
    same_r = all(np.array_equal(p[2], q[2]) for p in parts for q in parts if p[:2] == q[:2])
    ok &= same_r
    msgs.append(f"R replica-identical={same_r}")
    if grid == "1d":
        xt = np.random.default_rng(22).standard_normal((n, 3))
        b = (a @ xt)[topo.y::d]
        X = cb.cacqr.lstsq(args, torch.from_numpy(b.copy()).cuda(), topo).cpu().numpy()
        err = float(np.abs(X - xt).max() / np.abs(xt).max())
        xs = [None] * world
        dist.all_gather_object(xs, X)
        same_x = all(np.array_equal(x, X) for x in xs)
        ok &= err <= 1e-6 and same_x
        msgs.append(f"lstsq err={err:.1e} X rank-identical={same_x}")
    if not ok:
        print(f"rank {rank}: " + " | ".join(msgs), flush=True)
    flag = torch.tensor([0 if ok else 1])
    dist.all_reduce(flag)
    if rank == 0:
        print(("MP_OK " if flag.item() == 0 else "MP_FAIL ") + " | ".join(msgs), flush=True)
    dist.barrier()
    cb.topo.release_contexts()
    dist.destroy_process_group()
    sys.exit(0 if flag.item() == 0 else 1)


if __name__ == "__main__":
    main()
