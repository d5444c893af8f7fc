"""Child process of tests/test_gpu_zz_late.py (and of bench.py's optional `tf32` record): runs the EXPERIMENTAL TF32 tensor-core path in
its own CUDA context, so that a fault in it cannot poison the parent's context, and prints ONE
JSON line.  usage: tf32_worker.py gemm | cholinv n bcm | bench n bcm steps"""
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import capital_b200 as cb  # noqa: E402
from capital_b200 import _lib  # noqa: E402


def colmajor(rows, cols, ld, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    buf = torch.rand(ld * cols, dtype=torch.float64, device="cuda", generator=g) - 0.5
    return buf, buf.view(cols, ld).t()[:rows]


def gemm_cases(ctx):
    out = []
    for (m, n, k, flags, passes) in [(128, 128, 32, 0, 1), (128, 128, 256, 0, 1), (256, 384, 1024, 0, 1), (300, 200, 1000, 0, 1),
                                     (1024, 1024, 4096, _lib.GEMM_C_UPPER, 1), (640, 640, 777, _lib.GEMM_C_UPPER, 3), (256, 384, 1024, 0, 3),
                                     (2048, 2048, 8192, _lib.GEMM_C_UPPER, 3)]:
        lda, ldb, ldc = k + 6, k + 2, m + 3
        fa, A = colmajor(k, m, lda, 1)
        fb, B = colmajor(k, n, ldb, 2)
        fc, Cm = colmajor(m, n, ldc, 3)
        alpha, beta = -1.0, 1.0
        ref = alpha * (A.t() @ B) + beta * Cm
        if flags & _lib.GEMM_C_UPPER:
            ref = torch.where(torch.ones_like(ref, dtype=torch.bool).triu(), ref, Cm)
        den = (A.abs().t() @ B.abs()).max().item()
        st = _lib.lib().capital_blas_gemm_tn_tf32(ctx.handle, m, n, k, alpha, fa.data_ptr(), lda, fb.data_ptr(), ldb, beta, fc.data_ptr(), ldc,
                                                  flags, passes)
        ctx.synchronize()
        fresh, _ = colmajor(m, n, ldc, 3)
        out.append({"m": m, "n": n, "k": k, "flags": flags, "passes": passes, "status": int(st),
                    "error": _lib.lib().capital_last_error(ctx.handle).decode() if st else "",
                    "rel_err": (Cm - ref).abs().max().item() / den,
                    "padding_untouched": bool(torch.equal(fc.view(n, ldc)[:, m:], fresh.view(n, ldc)[:, m:]))})
    return out


def cholinv_case(topo, ctx, n, bcm, mode):
    ctx.set_trailing_precision(mode)
    A = cb.matrix(n, n, 1, 1).distribute_symmetric(topo)
    args = cb.cholinv.info(1, 1, bcm, "U", serialize=False)
    l0, _ = ctx.tf32_stats()
    cb.cholinv.factor(A, args, topo)
    l1, _ = ctx.tf32_stats()
    res = cb.cholinv.residual(A, args, topo)
    R = cb.cholinv.construct_R(args).clone()
    ctx.set_trailing_precision(0)
    return res, l1 - l0, R


def main():
    what = sys.argv[1]
    topo = cb.topo.square(1, 0, 1)
    ctx = topo.context()
    if what == "gemm":
        print(json.dumps({"gemm": gemm_cases(ctx)}))
    elif what == "cholinv":
        n, bcm = int(sys.argv[2]), int(sys.argv[3])
        r0, l0, R0 = cholinv_case(topo, ctx, n, bcm, 0)
        r1, l1, R1 = cholinv_case(topo, ctx, n, bcm, 1)
        r3, l3, R3 = cholinv_case(topo, ctx, n, bcm, 3)
        sc = R0.abs().max().item()
        print(json.dumps({"n": n, "residual": {"f64": r0, "tf32": r1, "tf32x3": r3}, "tf32_launches": {"f64": l0, "tf32": l1, "tf32x3": l3},
                          "R_rel_diff": {"tf32": (R1 - R0).abs().max().item() / sc, "tf32x3": (R3 - R0).abs().max().item() / sc}}))
    elif what == "bench":
        n, bcm, steps = int(sys.argv[2]), int(sys.argv[3]), int(sys.argv[4])
        A = cb.matrix(n, n, 1, 1).distribute_symmetric(topo)
        rec = {"n": n, "bc_mult_dim": bcm}
        for name, mode in (("f64", 0), ("tf32", 1), ("tf32x3", 3)):
            ctx.set_trailing_precision(mode)
            args = cb.cholinv.info(0, 1, bcm, "U")
            for _ in range(2):
                cb.cholinv.factor(A, args, topo)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            l0, f0 = ctx.tf32_stats()
            torch.cuda.synchronize()
            e0.record()
            for _ in range(steps):
                cb.cholinv.factor(A, args, topo)
            e1.record()
            torch.cuda.synchronize()
            l1, f1 = ctx.tf32_stats()
            ms = e0.elapsed_time(e1) / steps
            rec[name] = {"ms_per_step": ms, "tflops_n3_over_3": n ** 3 / 3 / (ms * 1e-3) / 1e12, "residual": cb.cholinv.residual(A, args, topo),
                         "tf32_kernel_launches_per_step": (l1 - l0) // steps, "tf32_kernel_flops_per_step": (f1 - f0) / steps}
        ctx.set_trailing_precision(0)
        print(json.dumps(rec))


if __name__ == "__main__":
    main()
