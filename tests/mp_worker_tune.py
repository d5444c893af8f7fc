"""16-rank worker for CA-CholeskyQR2 on the tunable 2 x 4 x 2 grid (run under torch.distributed.run).  Exits non-zero on mismatch.

Every rank runs on cuda:0 by default (gloo; the peer layer bootstraps through the host all-gather, and CUDA IPC works between
processes on one device); CAPITAL_MP_RANKS_PER_GPU=2 puts two ranks on each of 8 GPUs instead.  Checks the reference's own dumps
(tests/golden/cacqr_p16_tune_*.npz), the numpy restatement at a larger size, the validators, the bit-identity of R across the two
cubes, the host-pointer path and the rejection of a shape the grid cannot take.  Rank 0 prints one summary line.
"""
import json, os, sys, time
import numpy as np
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import capital_b200 as cb
from capital_b200 import _lib
from oracle import capital_oracle as co

GOLD = os.path.join(ROOT, "tests", "golden")
C_, D_ = 2, 4


def load(name):
    z = dict(np.load(os.path.join(GOLD, name + ".npz")))
    meta = json.loads(str(z["meta"]))
    for r, s in meta.get("replica_of", {}).items():  # layer replicas are stored once (tests/golden/make_golden_tune.py)
        for k in [k for k in z if k.endswith(f"_{s}")]:
            z[k[: -len(str(s))] + r] = z[k]
    return meta, z


def main():
    t_start = time.time()
    rank, world, lr = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    assert world == 16
    per_gpu = int(os.environ.get("CAPITAL_MP_RANKS_PER_GPU", "16"))
    dev = lr // per_gpu
    torch.cuda.set_device(dev)
    dist.init_process_group("gloo")
    ok = True
    msgs = []
    peak_used = 0

    def sample_memory():
        nonlocal peak_used
        free, total = torch.cuda.mem_get_info(dev)
        peak_used = max(peak_used, total - free)

    topo = cb.topo.rect(world, rank, C_)
    yc = topo.y % C_  # row coordinate on the cube's square grid
    # --- the reference's dumps, elementwise ---
    for name in ("cacqr_p16_tune_m512_n64", "cacqr_p16_tune_m512_n64_ci0", "cacqr_p16_tune_m512_n64_it1"):
        meta, z = load(name)
        m, n = meta["m"], meta["n"]
        ci = 0 if name.endswith("_ci0") else 1
        A = cb.matrix(n, m, C_, D_).distribute_random(topo, rank // C_)
        same_a = np.array_equal(A.data.cpu().numpy(), z[f"A_{rank}"])
        qa = cb.cacqr.info(meta["variant"], cb.cholinv.info(ci, 1, -1, "U"))
        cb.cacqr.factor(A, qa, topo)
        sample_memory()
        eq = np.abs(qa.Q.cpu().numpy() - z[f"Q_{rank}"]).max()
        er = np.abs(qa.R.cpu().numpy() - z[f"R_{rank}"]).max() / np.abs(z[f"R_{rank}"]).max()
        Rl = cb.cacqr.construct_R(qa).cpu().numpy()
        zeros = yc <= topo.x or bool(np.all(np.diag(Rl) == 0))
        res, orth = cb.cacqr.validate(A, qa, topo)
        good = same_a and eq < 1e-12 and er < 1e-12 and zeros and res < 1e-14 and orth < 1e-15
        ok &= good
        if not good:
            print(f"rank {rank} {name}: A={same_a} dQ={eq:.1e} dR={er:.1e} zeros={zeros} res={res:.1e} orth={orth:.1e}", flush=True)
        msgs.append(f"{name}: dQ={eq:.1e} dR={er:.1e} res={res:.1e} orth={orth:.1e}")
    # --- a larger case against the restatement; R bit-identical in both cubes; host-pointer path == device path ---
    m, n = 1 << 14, 256
    for ci in (1, 0):
        A = cb.matrix(n, m, C_, D_).distribute_random(topo, rank // C_)
        qa = cb.cacqr.info(2, cb.cholinv.info(ci, 1, -1, "U"))
        cb.cacqr.factor(A, qa, topo)
        sample_memory()
        res, orth = cb.cacqr.validate(A, qa, topo)
        parts = [None] * world if rank == 0 else None
        dist.gather_object((topo.x, topo.y, A.data.cpu().numpy(), qa.Q.cpu().numpy(), qa.R.cpu().numpy()), parts, dst=0)
        lr_, lc_ = m // D_, n // C_
        blk = lambda a: a.reshape(lc_, lr_).T
        eq, same_r = 0.0, True
        if rank == 0:  # one restatement, not sixteen
            same_r = all(np.array_equal(parts[r][4], parts[r + world // 2][4]) for r in range(world // 2))
            Ag = co.cyclic_assemble({(p[0], p[1]): blk(p[2]) for p in parts}, m, n, C_, D_)
            Qg = co.cyclic_assemble({(p[0], p[1]): blk(p[3]) for p in parts}, m, n, C_, D_)
            q_o, _ = co.cacqr_3d(Ag, C_, 2, bool(ci), 1, -1)
            eq = float(np.abs(Qg - q_o).max())
        hostA = cb.matrix(n, m, C_, D_, data=A.data.cpu().pin_memory())
        hq = cb.cacqr.info(2, cb.cholinv.info(ci, 1, -1, "U"))
        cb.cacqr.factor(hostA, hq, topo)
        same_host = (not hq.Q.is_cuda) and torch.equal(hq.Q, qa.Q.cpu()) and torch.equal(hq.R, qa.R.cpu())
        good = eq < 1e-12 and res < 1e-13 and orth < 1e-14 and same_r and same_host
        ok &= good
        if not good:
            print(f"rank {rank} m={m} n={n} ci={ci}: dQ={eq:.1e} res={res:.1e} orth={orth:.1e} R same in both cubes={same_r} "
                  f"host path identical={same_host}", flush=True)
        msgs.append(f"m={m} n={n} ci={ci}: dQ={eq:.1e} res={res:.1e} orth={orth:.1e} R cube-identical={same_r} host identical={same_host}")
    # --- a shape the grid cannot take: d = 4 does not divide m ---
    A = cb.matrix(64, 510, C_, D_).distribute_random(topo, rank // C_)
    try:
        cb.cacqr.factor(A, cb.cacqr.info(2, cb.cholinv.info(1, 1, -1, "U")), topo)
        rejected = False
    except _lib.CapitalError as ex:
        rejected = ex.status == _lib.ERR_UNSUPPORTED and "must divide m" in str(ex)
    ok &= rejected
    msgs.append(f"m=510 rejected={rejected}")
    flag = torch.tensor([0 if ok else 1])
    dist.all_reduce(flag)
    peak = torch.tensor([peak_used], dtype=torch.int64)
    dist.all_reduce(peak, op=dist.ReduceOp.MAX)
    if rank == 0:
        msgs.append(f"peak device memory in use {peak.item() / 2**30:.1f} GiB (all processes on the device)")
        msgs.append(f"worker wall {time.time() - t_start:.0f} s; peer flag waits: {topo.context().peer_wait_mode()}")
        print(("MP_OK " if flag.item() == 0 else "MP_FAIL ") + " | ".join(msgs), flush=True)
    dist.barrier()
    cb.topo.release_contexts()
    dist.destroy_process_group()
    sys.exit(0 if flag.item() == 0 else 1)


if __name__ == "__main__":
    main()
