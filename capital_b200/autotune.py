"""Base-case size sweep for cholinv::factor -- the job of the reference's autotune/cholesky/cholinv/tune.cpp:153-253.

The reference loops `bcMultiplier + k`, k < space_dim (tune.cpp:239-253), over its three base-case policies and lets critter
model the kernel times.  Here one base-case policy exists (replicate-everything, the semantics of ReplicateCommComp,
cholinv/policy.h:160-224), the timing is the library's own CUDA-event bracket around `factor` (capital_last_factor_ms, max
over ranks), and configurations whose multipliers clamp to the same base-case dimension (cholinv.hpp:15-18) are run once.

    python -m torch.distributed.run --nproc-per-node 8 -m capital_b200.autotune 49152 1 0 1 -6 0 0 3 0 5
    (arguments as tune.cpp:164-176: num_rows rep_div complete_inv split bcMultiplier layout num_chunks num_iter compare [space_dim])

`sweep()` is a pure function of a timing callback, so the selection logic is tested without a GPU (tests/test_autotune.py)."""
from __future__ import annotations
import json, os, statistics, sys
from . import _lib


def configurations(local_dim: int, c: int, d: int, bc_mult_dim: int, space_dim: int) -> list:
    """[{k, bc_mult_dim, bc_dim}] for k < space_dim, one entry per distinct base-case dimension (first multiplier reaching it)."""
    out, seen = [], set()
    for k in range(space_dim):
        bc = int(_lib.lib().capital_cholinv_bc_dimension(local_dim, c, d, bc_mult_dim + k))
        if bc in seen:
            continue
        seen.add(bc)
        out.append({"k": k, "bc_mult_dim": bc_mult_dim + k, "bc_dim": bc})
    return out


def sweep(time_ms, configs: list, num_iter: int, warmup: int = 1) -> list:
    """time_ms(config) -> milliseconds of one factorization (already reduced over ranks).  Returns the configs annotated with
    min / median over num_iter timed calls after `warmup` untimed ones, in the order given."""
    rows = []
    for cfg in configs:
        for _ in range(warmup):
            time_ms(cfg)
        t = [float(time_ms(cfg)) for _ in range(max(1, num_iter))]
        rows.append({**cfg, "ms_min": min(t), "ms_median": statistics.median(t), "samples": len(t)})
    return rows


def best(rows: list, key: str = "ms_median") -> dict:
    """fastest configuration; ties go to the larger base case (fewer recursion levels, fewer launches)."""
    return min(rows, key=lambda r: (r[key], -r["bc_dim"]))


def grid_depth(world: int, rep_div: int = 1) -> int:
    """c of the c x d x d grid: the cube root of the process count cut by rep_div (tune.cpp:182-183); process counts that are not
    cubes (2, 4 GPUs) take the library's own 2x1x1 / 1x2x2 grids."""
    cube = round(world ** (1.0 / 3.0))
    if cube ** 3 == world:
        return max(1, cube // max(1, rep_div))
    return 2 if world == 2 else 1


def tune_cholinv(topo, num_rows: int, complete_inv: int, split: int, bc_mult_dim: int, space_dim: int = 5, num_iter: int = 3) -> list:
    """Runs the sweep on this process' GPU (all ranks of the grid call it together).  Residual of every configuration is checked
    against the reference's validator bound so that a fast-but-wrong configuration can never be selected."""
    import torch
    import torch.distributed as dist
    from . import cholinv
    from .matrix import matrix
    A = matrix(num_rows, num_rows, topo.d, topo.d).distribute_symmetric(topo)
    ctx = topo.context()
    multi = topo.size > 1

    def run(cfg):
        args = run.args.setdefault(cfg["bc_mult_dim"], cholinv.info(complete_inv, split, cfg["bc_mult_dim"], "U"))
        cholinv.factor(A, args, topo)
        ms = torch.tensor([ctx.last_factor_ms()], dtype=torch.float64, device="cuda")
        if multi:
            dist.all_reduce(ms, op=dist.ReduceOp.MAX)
        return ms.item()
    run.args = {}
    rows = sweep(run, configurations(A.num_rows_local, topo.c, topo.d, bc_mult_dim, space_dim), num_iter)
    for r in rows:
        r["residual"] = cholinv.residual(A, run.args[r["bc_mult_dim"]], topo)
        r["tflops"] = num_rows ** 3 / 3.0 / (r["ms_median"] * 1e-3) / 1e12
        if not r["residual"] <= 1e-12:
            r["ms_median"] = r["ms_min"] = float("inf")
    return rows


def main(argv=None):
    argv = list(sys.argv[1:] if argv is None else argv)
    if len(argv) < 9:
        print("usage: autotune num_rows rep_div complete_inv split bcMultiplier layout num_chunks num_iter compare [space_dim]", file=sys.stderr)
        return 2
    num_rows, rep_div, complete_inv, split, bcm, layout, num_chunks, num_iter, _compare = (int(a) for a in argv[:9])
    space_dim = int(argv[9]) if len(argv) > 9 else 5  # tune.cpp:177-178
    import torch
    import torch.distributed as dist
    from . import topology as topo_mod
    rank, world = int(os.environ.get("RANK", 0)), int(os.environ.get("WORLD_SIZE", 1))
    torch.cuda.set_device(int(os.environ.get("LOCAL_RANK", 0)))
    if world > 1:
        dist.init_process_group("nccl", device_id=torch.device("cuda", torch.cuda.current_device()))
    c = grid_depth(world, rep_div)
    topo = topo_mod.square(world, rank, c, layout, num_chunks)
    rows = tune_cholinv(topo, num_rows, complete_inv, split, bcm, space_dim, num_iter)
    if rank == 0:
        for r in rows:
            print(json.dumps(r))
        print(json.dumps({"best": best(rows), "grid": [topo.c, topo.d, topo.d], "num_rows": num_rows, "complete_inv": complete_inv}))
    topo_mod.release_contexts()
    if world > 1:
        dist.destroy_process_group()
    return 0


if __name__ == "__main__":
    sys.exit(main())
