"""Grid worker of the split-k Gram product on the 1D row grid, run under torch.distributed.run with 2 processes.  Exits non-zero on a
failed check.

Every rank builds the same seeded global A in torch and takes its cyclic rows (rank y: rows y, y + P, ...).  In one context the
ranks factor (num_iter = 1) A with P * (k - 1) rows and then with P * k rows, where k is the first local row count at which the
n = 128 Gram product leaves a split-k chunk empty (same chunking as k - 1): the second factorization must not pick up the first
one's partial sums.  Checks, on each: the backward-error bound |R^T R - A^T A| <= 2 (gamma_m |A|^T |A| + gamma_{n+1} |R|^T |R|) of
the replicated R against the global A, and the validator's orthogonality against ||Q^T Q - I||_F / n summed over the ranks in
torch (|difference| <= 2 m u).  CAPITAL_MP_SAME_DEVICE=1 puts every rank on cuda:0 (the ranks bootstrap through the gloo group)."""
import os, sys
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import capital_b200 as cb
from test_gpu_gram import U, first_empty_k, gram_bound_ratio, splitk_chunks


def main():
    rank, world, lr = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(0 if os.environ.get("CAPITAL_MP_SAME_DEVICE") else lr)
    dist.init_process_group("gloo")
    topo = cb.topo.rect(world, rank, 1)
    n = 128
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    kq = first_empty_k(n, True, sms)
    ok, msgs = True, []
    for k, seed in ((kq - 1, 31), (kq, 32)):
        m = world * k
        g = torch.Generator(device="cuda").manual_seed(seed)
        a = torch.randn(m, n, dtype=torch.float64, device="cuda", generator=g)
        A = cb.matrix(n, m, 1, world, data=a[rank::world].t().contiguous().view(-1))
        args = cb.cacqr.info(1, cb.cholinv.info(0, 1, 0, "U"))
        cb.cacqr.factor(A, args, topo)
        ratio = gram_bound_ratio(a, cb.cacqr.construct_R(args))
        _, orth = cb.cacqr.validate(A, args, topo)
        q = cb.cacqr.construct_Q(args)
        qtq = (q.T @ q).cpu()
        dist.all_reduce(qtq)
        ref = (torch.linalg.matrix_norm(qtq - torch.eye(n, dtype=torch.float64)) / n).item()
        good = ratio <= 1.0 and abs(orth - ref) <= 2 * m * U
        ok &= good
        msgs.append(f"m={m} (k={k}, chunks {splitk_chunks(n, k, True, sms)}): bound ratio {ratio:.2g} orth {orth:.3g} torch {ref:.3g}")
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
