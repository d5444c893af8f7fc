"""Grid worker of the schedule's edges (run under torch.distributed.run, one process per rank).  Exits non-zero on a mismatch.

2 ranks: the 2x1x1 grid, 4: 1x2x2, 8: 2x2x2.  Runs the table of tests/grid_edges_reference.py: ragged local sizes (L = 501, 513, 648, 695;
777 and 1001 with d = 1), split 1 and 2, both output structures, and knob sets that lower the schedule's thresholds so that sizes one GPU
holds take the chunked, deferred, pipelined and single-stream paths of the large ones (CAPITAL_DIST_* are read on every call).

Under the default knobs every case is checked against the extended-precision reference within derived bounds, against the oracle
(2e-13, and the same zero pattern), for exact zeros where the structure promises them, for bit-identical layer replicas, and by the
library's own validator.  Every other knob set must reproduce the default's bits: the knobs move work between streams and cut outputs
at multiples of 128 columns, no tile's k range or order changes.  `low` must also launch more kernels for the same GEMM flops.
Then factorizations of different ragged sizes in turn on one context, and solve / inverse / sygst on ragged factors.
CAPITAL_GRID_EDGES_SIZES=n,n restricts the table; each case prints a digest of all ranks' bits so that runs can be compared."""
import hashlib
import os, sys
import numpy as np
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import capital_b200 as cb
from oracle import capital_oracle as co
import grid_edges_reference as ge
import sygst_reference, sygst_ab_reference

LD_ROWS = 16  # rows per rank whose residuals are evaluated in long double (the others in float64)


class knobs:
    """the knob set in the environment for the calls inside, identically on every rank"""

    def __init__(self, name):
        self.env = ge.KNOBS[name]

    def __enter__(self):
        os.environ.update(self.env)

    def __exit__(self, *exc):
        for k in self.env:
            del os.environ[k]


def main():
    rank, world, lr = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    if os.environ.get("CAPITAL_MP_SAME_DEVICE"):
        torch.cuda.set_device(0)
        dist.init_process_group("gloo")
    else:
        torch.cuda.set_device(lr)
        dist.init_process_group("nccl", device_id=torch.device("cuda", lr))
    assert not any(k in os.environ for k in ge.KNOB_NAMES)
    c, d = ge.GRIDS[world]
    topo = cb.topo.square(world, rank, c)
    ctx = topo.context()
    gloo = dist.get_backend() == "gloo"
    only = os.environ.get("CAPITAL_GRID_EDGES_SIZES")
    only = tuple(int(v) for v in only.split(",")) if only else None
    table = ge.cases(world, only)
    sizes = sorted({t[0] for t in table})

    def gather(t):
        mine = t.cpu() if gloo else t
        parts = [torch.empty_like(mine) for _ in range(world)]
        dist.all_gather(parts, mine)
        return [p.cpu() for p in parts]

    def reduce_max(vals):
        t = torch.tensor(vals, dtype=torch.float64, device="cpu" if gloo else "cuda")
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
        return [float(v) for v in t.cpu()]

    coords = [tuple(int(v) for v in t) for t in gather(torch.tensor([topo.x, topo.y, topo.z], dtype=torch.int64, device="cuda"))]

    # the extended-precision factors take seconds per size: the ranks share the sizes and broadcast
    refs, mats = {}, {}
    for i, n in enumerate(sizes):
        a = co.spd_global(n)
        ld = torch.zeros(2, n, n, dtype=torch.float64)
        if i % world == rank:
            _, _, r64, ri64 = ge.chol_ld(a)
            ld[0], ld[1] = torch.from_numpy(r64), torch.from_numpy(ri64)
        if not gloo:
            ld = ld.cuda()
        dist.broadcast(ld, i % world)
        refs[n] = (a, ge.Bounds(a), ld[0].cpu().numpy(), ld[1].cpu().numpy())
        mats[n] = cb.matrix(n, n, d, d).distribute_symmetric(topo)

    def factor(n, ci, split, bcm, serialize, knob, count=False):
        args = cb.cholinv.info(ci, split, bcm, "U", serialize=serialize)
        cnt = None
        with knobs(knob):
            cb.cholinv.factor(mats[n], args, topo)
            if count:  # the first call allocated outputs and workspaces
                first = (args.R.clone(), args.Rinv.clone())
                ctx.reset_counters()
                cb.cholinv.factor(mats[n], args, topo)
                torch.cuda.synchronize()
                cnt = ctx.counters()
                cnt = (cnt.kernel_launches, cnt.gemm_flops, torch.equal(first[0], args.R) and torch.equal(first[1], args.Rinv))
        torch.cuda.synchronize()
        return args, cnt

    def digest(*tensors):
        h = hashlib.sha256()
        for t in tensors:
            h.update(t.cpu().numpy().tobytes())
        mine = torch.tensor([int.from_bytes(h.digest()[:7], "big")], dtype=torch.int64, device="cuda")
        return hashlib.sha256(b"".join(p.numpy().tobytes() for p in gather(mine))).hexdigest()[:12]

    ok = True
    msgs = []

    # --- different ragged sizes in turn on one context: the arena is cleared again and the grow-only workspaces see a changing ld ---
    n0, n1 = ge.ODD_SIZES[d]
    if only is None or (n0 in only and n1 in only):
        seq = [factor(n, 1, 1, -3, True, "default")[0] for n in (n0, n1, n0)]
        again = torch.equal(seq[0].R, seq[2].R) and torch.equal(seq[0].Rinv, seq[2].Rinv)
        ok &= again
        msgs.append(f"n={n0} then {n1} then {n0}: third==first={again}")

    base, counts = {}, {}
    for n, ci, split, bcm, serialize, knob in table:
        key = (n, ci, split, bcm, serialize)
        countable = bcm == -3 and serialize and knob in ("default", "low")
        args, cnt = factor(n, ci, split, bcm, serialize, knob, countable)
        finite = bool(torch.isfinite(args.R).all() and torch.isfinite(args.Rinv).all())
        good = finite and (cnt is None or cnt[2])
        msg = ge.case_id(*key, knob) + ":"
        if knob == "default":
            base[key] = (args.R.clone(), args.Rinv.clone())
            a, bnd, r_ld, ri_ld = refs[n]
            L = n // d
            pr, pi = gather(args.R), gather(args.Rinv)
            layers = all(torch.equal(p[i], p[j]) for p in (pr, pi) for i in range(world) for j in range(world)
                         if coords[i][:2] == coords[j][:2])
            R = ge.assemble([p.numpy() for p in pr], coords, n, d, serialize)
            Ri = ge.assemble([p.numpy() for p in pi], coords, n, d, serialize)
            if serialize:  # exact zeros on the local-diagonal slots of ranks below the global diagonal
                zeros = all(np.all(np.diag(co.unpack_upper(p.numpy(), L)) == 0) for ps in (pr, pi) for p, (x, y, _) in zip(ps, coords) if y > x)
                R, Ri = np.triu(R), np.triu(Ri)
            else:          # exact zeros strictly below the global diagonal
                zeros = not np.tril(R, -1).any() and not np.tril(Ri, -1).any()
            ro, rio = co.cholinv(a, bool(ci), split, co.bc_dimension(L, c, d, bcm), d=d)
            e_o = max(np.abs(R - ro).max() / np.abs(ro).max(), np.abs(Ri - rio).max() / np.abs(rio).max())
            zeros &= np.array_equal(Ri == 0, rio == 0)  # the block complete_inv = 0 skips moves with split
            done = rio != 0
            f_r, f_i = np.abs(R - r_ld).max(), np.abs(np.where(done, Ri - ri_ld, 0)).max()
            # residuals of the assembled factors: this rank's rows in float64 (its own rounding is within one more bound), some in long double
            rows = np.arange(rank, n, world)
            full_ri = Ri if ci else ri_ld  # an incomplete Rinv has no R^-1 residual: its rows are checked against the reference above
            b64 = ge.residual_rows(R, full_ri, a, rows, np.float64)
            bld = ge.residual_rows(R, full_ri, a, rows[:: max(1, len(rows) // LD_ROWS)])
            within = b64[0] <= 2 * bnd.backward and bld[0] <= bnd.backward and f_r <= bnd.forward_r and f_i <= bnd.forward_rinv
            if ci:
                within &= b64[1] <= 2 * bnd.inverse and bld[1] <= bnd.inverse
            e_a, e_i = reduce_max(list(bld))
            res = cb.cholinv.residual(mats[n], args, topo)
            good &= bool(within) and e_o <= 2e-13 and bool(zeros) and layers and res <= 1e-12
            if (n, ci, split, bcm, serialize) == (n0, 1, 1, -3, True) and only is None:
                good &= torch.equal(seq[0].R, args.R) and torch.equal(seq[0].Rinv, args.Rinv)
            msg += (f" |RtR-A|={e_a:.1e}/{bnd.backward:.1e}" + (f" |RinvR-I|={e_i:.1e}/{bnd.inverse:.1e}" if ci else "") +
                    f" dR={f_r:.1e}/{bnd.forward_r:.1e} dRinv={f_i:.1e}/{bnd.forward_rinv:.1e} oracle={e_o:.1e} zeros={bool(zeros)}"
                    f" layers-identical={layers} res={res:.1e}")
        else:
            same = torch.equal(base[key][0], args.R) and torch.equal(base[key][1], args.Rinv)
            good &= same
            msg += f" bits==default={same}"
        if cnt is not None:
            counts[key + (knob,)] = cnt
            if knob == "low":  # the lowered thresholds ran: more launches for the same flops
                l0, f0, _ = counts[key + ("default",)]
                good &= cnt[0] > l0 and cnt[1] == f0
                msg += f" launches={cnt[0]}>{l0} flops-equal={cnt[1] == f0}"
            msg += f" rerun-identical={cnt[2]}"
        ok &= good
        msgs.append(msg + f" finite={finite} sha={digest(args.R, args.Rinv)}" + ("" if good else " FAILED"))
        if rank == 0:  # progress, so that a case that does not come back can be named
            print(msgs[-1], file=sys.stderr, flush=True)

    # --- downstream calls on ragged factors; complete_inv = 0 under `low` rebuilds Rinv12 in chunks ---
    if only is None or n0 in only:
        n = n0
        b = refs[n][0]
        a = b - n * np.eye(n)  # the generator's plain symmetric matrix: the same draws without the diagonal shift
        Am = cb.matrix(n, n, d, d).distribute_symmetric(topo, False)
        rhs = {k: torch.from_numpy(np.random.default_rng(n + k).standard_normal((n, k))).cuda() for k in (1, 33)}
        outs = {}
        for knob in ("default", "low"):
            with knobs(knob):
                args = cb.cholinv.info(0, 1, -3, "U")
                cb.cholinv.factor(mats[n], args, topo)
                outs[knob] = {"solve k=1": cb.cholinv.solve(args, rhs[1], topo), "solve k=33": cb.cholinv.solve(args, rhs[33], topo),
                              "inverse": cb.cholinv.inverse(args, topo), "sygst itype=1": cb.cholinv.sygst(Am, args, topo),
                              "sygst itype=2": cb.cholinv.sygst(Am, args, topo, itype=2)}
                torch.cuda.synchronize()
        r = np.triu(ge.assemble([p.numpy() for p in gather(args.R)], coords, n, d, True))
        for what, out in outs["default"].items():
            same = torch.equal(out, outs["low"][what])
            if what.startswith("solve"):
                ref = np.linalg.solve(b, rhs[out.shape[1]].cpu().numpy())
                err = float(np.abs(out.cpu().numpy() - ref).max() / np.abs(ref).max())
                good = err <= 1e-12 and all(torch.equal(out.cpu(), p) for p in gather(out))
            else:
                M = ge.assemble([p.numpy() for p in gather(out)], coords, n, d, True)
                if what == "inverse":
                    ref = np.linalg.inv(b)
                    good = np.abs(M - ref).max() <= 1e-12 * np.abs(ref).max()
                else:
                    # against the float64 restatement of the library's n^3 form, normwise: no entry is further from it than the largest
                    # entry of the elementwise first-order bound (doubled: the restatement has its own rounding).  The elementwise
                    # ratio is printed, not held: at n = 1002 entry (2, 2), where a diagonal draw of 2.6e-4 cancels to -1.8e-6, the
                    # grids' itype 1 result sits at several bounds while the restatement is within 1e-3 of one.
                    if what == "sygst itype=1":
                        ri = np.linalg.inv(r)
                        ref, q = sygst_reference.sygst(a, r, ri, True, 1, n, d), 2 * sygst_reference.bound(a, ri)
                    else:
                        ref, q = sygst_ab_reference.sygst_ab(a, r), 2 * sygst_ab_reference.bound(a, r)
                    good = np.abs(M - ref).max() <= q.max()
                    q = np.abs(M - ref) / q
                    at = np.unravel_index(q.argmax(), q.shape)
                    what += f" (elementwise err/bound={q[at]:.2f} at {tuple(int(v) for v in at)})"
                err = float(np.abs(M - ref).max() / np.abs(ref).max())
            ok &= bool(good) and same
            msgs.append(f"n={n} ci=0 {what}: err={err:.1e} within={bool(good)} low-bits==default={same}")

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
