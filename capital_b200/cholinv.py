"""cholesky::cholinv -- host-side mirror of the reference's entry points (src/alg/cholesky/cholinv/cholinv.h:46-53).

    args = cholinv.info(complete_inv, split, bc_mult_dim, 'U')      # cholinv.h:25-30
    cholinv.factor(A, args, topo)                                    # cholinv.hpp:6-28  -> args.R, args.Rinv
    R = cholinv.construct_R(args, topo)                              # cholinv.hpp:30-37 -> rect, zero lower
    X = cholinv.solve(args, B, topo)                                 # A X = B from the factors (capital_cholinv_solve_f64)
    Ainv = cholinv.inverse(args, topo)                               # A^-1 = Rinv Rinv^T (capital_cholinv_inverse_f64)
    res = cholinv.inverse_residual(A, Ainv, args, topo)              # ||A Ainv - I||_F / ||I||_F (test/inverse/validate.hpp)
    C = cholinv.sygst(A2, args, topo)                                # C = R^-T A2 R^-1 for A2 x = l A x (capital_cholinv_sygst_f64)
    X = cholinv.apply_Rinv(args, Y, topo)                            # R^-1 Y, the back-transform (capital_cholinv_apply_rinv_f64)
    W = cholinv.apply_RinvT(args, B, topo)                           # R^-T B, whitening
    C = cholinv.sygst(A2, args, topo, itype=2)                       # C = R A2 R^T for A2 A x = l x or A A2 x = l x (itype 3)
    X = cholinv.apply_R(args, Z, topo)                               # R Z (capital_cholinv_apply_r_f64)
    X = cholinv.apply_RT(args, Y, topo)                              # R^T Y, the itype 3 back-transform
    R, Rinv, info = cholinv.factor_batched(A, topo)                  # many SPD matrices A[b] (n <= 512) at once
    X = cholinv.solve_batched(Rinv, B, topo)                         # A[b] X[b] = B[b] from the batched factors

Outputs are packed upper-triangular local blocks (policy::cholinv::Serialize) unless serialize=False."""
from __future__ import annotations
import ctypes as C
import torch
from . import _lib
from .matrix import matrix


class info:
    def __init__(self, complete_inv, split: int, bc_mult_dim: int, dir: str = "U", serialize: bool = True):
        if split <= 0 or dir != "U":
            raise ValueError("cholinv requires split > 0 and dir == 'U' (cholinv.hpp:9)")
        self.complete_inv, self.split, self.bc_mult_dim, self.dir = int(bool(complete_inv)), int(split), int(bc_mult_dim), dir
        self.serialize = serialize
        self.R = None      # torch tensors: packed upper L(L+1)/2 (or L*L rect)
        self.Rinv = None
        self.local_dim = 0
        self.global_dim = 0

    def _c(self) -> _lib.CholinvArgs:
        return _lib.CholinvArgs(self.complete_inv, self.split, self.bc_mult_dim, self.dir.encode())


def _register(args: info, L: int, device):
    count = L * (L + 1) // 2 if args.serialize else L * L
    for name in ("R", "Rinv"):  # matrix::_register_: allocate on first use only (matrix.hpp:141-155)
        t = getattr(args, name)
        if t is None or t.numel() != count or t.device != device:
            pin = device.type == "cpu"
            setattr(args, name, torch.empty(count, dtype=torch.float64, device=device, pin_memory=pin))


def factor(A: matrix, args: info, topo):
    """A is never modified (const&).  Results land in args.R / args.Rinv, on the same device kind as A."""
    ctx = topo.context()
    n = A.num_rows_global
    assert A.num_columns_global == n
    L = A.num_rows_local
    _register(args, L, A.data.device)
    args.local_dim, args.global_dim = L, n
    cargs = args._c()
    st = _lib.lib().capital_cholinv_factor_f64(ctx.handle, A.data.data_ptr(), n, C.byref(cargs),
                                               _lib.UPPERTRI_PACKED if args.serialize else _lib.RECT,
                                               args.R.data_ptr(), args.Rinv.data_ptr())
    ctx.check(st)


def _expand(packed: torch.Tensor, L: int, serialize: bool) -> torch.Tensor:
    if not serialize:
        return packed.view(L, L).t()
    out = torch.zeros(L, L, dtype=torch.float64, device=packed.device)
    iu = torch.triu_indices(L, L, device=packed.device)
    # column-packed upper: (col i, row j<=i) at i(i+1)/2 + j  (structure.h:39)
    out[iu[0], iu[1]] = packed[(iu[1] * (iu[1] + 1)) // 2 + iu[0]]
    return out


def construct_R(args: info, topo=None) -> torch.Tensor:
    """rows x cols local block with zero lower part (serialize<uppertri, rect>, cholinv.hpp:30-37)."""
    return _expand(args.R, args.local_dim, args.serialize)


def construct_Rinv(args: info, topo=None) -> torch.Tensor:
    return _expand(args.Rinv, args.local_dim, args.serialize)


def residual(A: matrix, args: info, topo) -> float:
    """cholesky::validate<Alg>::residual (test/cholesky/validate.hpp:7-49)."""
    ctx = topo.context()
    r = C.c_double()
    ctx.check(_lib.lib().capital_cholinv_residual_f64(ctx.handle, A.data.data_ptr(), A.num_rows_global,
                                                      _lib.UPPERTRI_PACKED if args.serialize else _lib.RECT,
                                                      args.R.data_ptr(), C.byref(r)))
    return float(r.value)


def solve(args: info, B: torch.Tensor, topo) -> torch.Tensor:
    """A X = B with the factors of a previous `factor(A, args, topo)` (capital_cholinv_solve_f64).  B: float64, shape (n,) or (n, k),
    on CUDA or on the host; the full right-hand side, the same on every rank of a grid.  Returns X with B's shape and device
    (bit-identical on every rank)."""
    if args.R is None or args.Rinv is None or args.global_dim <= 0:
        raise ValueError("cholinv.solve: `args` holds no factors (run cholinv.factor first)")
    if not isinstance(B, torch.Tensor) or B.dtype != torch.float64:
        raise ValueError("cholinv.solve: B must be a float64 tensor")
    if B.dim() not in (1, 2) or B.shape[0] != args.global_dim or B.numel() == 0:
        raise ValueError(f"cholinv.solve: B must have shape ({args.global_dim},) or ({args.global_dim}, k), got {tuple(B.shape)}")
    L = args.local_dim
    if args.R.numel() != args.Rinv.numel() or args.Rinv.numel() != (L * (L + 1) // 2 if args.serialize else L * L):
        raise ValueError("cholinv.solve: args.R / args.Rinv do not hold factors of the local dimension args.local_dim")
    n = args.global_dim
    k = 1 if B.dim() == 1 else B.shape[1]
    Bc = B.contiguous() if B.dim() == 1 else B.t().contiguous()  # column-major n x k, ld n
    Xc = torch.empty_like(Bc)
    ctx = topo.context()
    cargs = args._c()
    ctx.check(_lib.lib().capital_cholinv_solve_f64(ctx.handle, n, C.byref(cargs), _lib.UPPERTRI_PACKED if args.serialize else _lib.RECT,
                                                   args.R.data_ptr(), args.Rinv.data_ptr(), k, Bc.data_ptr(), n, Xc.data_ptr(), n))
    return Xc if B.dim() == 1 else Xc.t().contiguous()


def _check_factors(args: info, what: str) -> int:
    """the local element count of args.R / args.Rinv, or ValueError when `args` holds no factors of args.local_dim"""
    if args.R is None or args.Rinv is None or args.global_dim <= 0:
        raise ValueError(f"cholinv.{what}: `args` holds no factors (run cholinv.factor first)")
    L = args.local_dim
    count = L * (L + 1) // 2 if args.serialize else L * L
    if args.R.numel() != count or args.Rinv.numel() != count:
        raise ValueError(f"cholinv.{what}: args.R / args.Rinv do not hold factors of the local dimension args.local_dim")
    return count


def inverse(args: info, topo) -> torch.Tensor:
    """A^-1 = Rinv Rinv^T from the factors of a previous `factor(A, args, topo)` (capital_cholinv_inverse_f64).  Returns the local block
    as a flat float64 tensor with args.Rinv's length and device (pinned on the host): packed upper when args.serialize, else the full,
    exactly symmetric rect block.  The same bits on every layer of a grid."""
    count = _check_factors(args, "inverse")
    dev = args.Rinv.device
    out = torch.empty(count, dtype=torch.float64, device=dev, pin_memory=dev.type == "cpu")
    ctx = topo.context()
    cargs = args._c()
    ctx.check(_lib.lib().capital_cholinv_inverse_f64(ctx.handle, args.global_dim, C.byref(cargs),
                                                     _lib.UPPERTRI_PACKED if args.serialize else _lib.RECT,
                                                     args.R.data_ptr(), args.Rinv.data_ptr(), out.data_ptr()))
    return out


def sygst(A: matrix, args: info, topo, itype: int = 1) -> torch.Tensor:
    """A generalized symmetric-definite eigenproblem reduced to C y = lambda y with the factors of a previous `factor(B, args, topo)`,
    B = R^T R (LAPACK dsygst, upper), with the same eigenvalues:
      itype 1: A x = lambda B x,  C = R^-T A R^-1 (capital_cholinv_sygst_f64),    back-transform x = apply_Rinv(args, y, topo);
      itype 2: A B x = lambda x,  C = R A R^T     (capital_cholinv_sygst_ab_f64), back-transform x = apply_Rinv(args, y, topo);
      itype 3: B A x = lambda x,  C = R A R^T     (capital_cholinv_sygst_ab_f64), back-transform x = apply_RT(args, y, topo).
    A: the symmetric matrix, a `matrix` shaped like the factored B; only its global lower triangle (diagonal included) is read.  Returns
    the local block of C like `inverse` does: a flat float64 tensor with args.Rinv's length and device (pinned on the host), packed upper
    when args.serialize, else the full, exactly symmetric rect block.  The same bits on every layer of a grid."""
    if isinstance(itype, bool) or itype not in (1, 2, 3):
        raise ValueError(f"cholinv.sygst: itype must be 1, 2 or 3, got {itype!r}")
    count = _check_factors(args, "sygst")
    if not isinstance(A, matrix) or A.num_rows_global != args.global_dim or A.num_columns_global != args.global_dim \
            or A.num_rows_local != args.local_dim or A.num_columns_local != args.local_dim:
        raise ValueError("cholinv.sygst: A must be a matrix shaped like the factored one")
    if A.data.dtype != torch.float64 or A.data.numel() != args.local_dim * args.local_dim or not A.data.is_contiguous():
        raise ValueError("cholinv.sygst: A must hold a contiguous float64 local block")
    dev = args.Rinv.device
    out = torch.empty(count, dtype=torch.float64, device=dev, pin_memory=dev.type == "cpu")
    ctx = topo.context()
    cargs = args._c()
    structure = _lib.UPPERTRI_PACKED if args.serialize else _lib.RECT
    if itype == 1:
        ctx.check(_lib.lib().capital_cholinv_sygst_f64(ctx.handle, args.global_dim, C.byref(cargs), structure,
                                                       args.R.data_ptr(), args.Rinv.data_ptr(), A.data.data_ptr(), out.data_ptr()))
    else:
        ctx.check(_lib.lib().capital_cholinv_sygst_ab_f64(ctx.handle, args.global_dim, C.byref(cargs), structure,
                                                          args.R.data_ptr(), A.data.data_ptr(), out.data_ptr()))
    return out


def _apply(args: info, B: torch.Tensor, topo, trans: int, what: str, factor_r: bool) -> torch.Tensor:
    """X = op(F) B with F = R (factor_r) or Rinv: the right-hand-side checks and layout shared by the apply_* entry points"""
    _check_factors(args, what)
    if not isinstance(B, torch.Tensor) or B.dtype != torch.float64:
        raise ValueError(f"cholinv.{what}: B must be a float64 tensor")
    if B.dim() not in (1, 2) or B.shape[0] != args.global_dim or B.numel() == 0:
        raise ValueError(f"cholinv.{what}: B must have shape ({args.global_dim},) or ({args.global_dim}, k), got {tuple(B.shape)}")
    n = args.global_dim
    k = 1 if B.dim() == 1 else B.shape[1]
    Bc = B.contiguous() if B.dim() == 1 else B.t().contiguous()  # column-major n x k, ld n
    Xc = torch.empty_like(Bc)
    ctx = topo.context()
    cargs = args._c()
    structure = _lib.UPPERTRI_PACKED if args.serialize else _lib.RECT
    if factor_r:
        ctx.check(_lib.lib().capital_cholinv_apply_r_f64(ctx.handle, n, C.byref(cargs), structure, args.R.data_ptr(), trans, k,
                                                         Bc.data_ptr(), n, Xc.data_ptr(), n))
    else:
        ctx.check(_lib.lib().capital_cholinv_apply_rinv_f64(ctx.handle, n, C.byref(cargs), structure, args.R.data_ptr(),
                                                            args.Rinv.data_ptr(), trans, k, Bc.data_ptr(), n, Xc.data_ptr(), n))
    return Xc if B.dim() == 1 else Xc.t().contiguous()


def apply_Rinv(args: info, B: torch.Tensor, topo) -> torch.Tensor:
    """X = R^-1 B from the factors of a previous `factor` (capital_cholinv_apply_rinv_f64, trans = 0): the back-transform x = R^-1 y of
    `sygst`.  B as for `solve`; returns X with B's shape and device, bit-identical on every rank."""
    return _apply(args, B, topo, 0, "apply_Rinv", False)


def apply_RinvT(args: info, B: torch.Tensor, topo) -> torch.Tensor:
    """X = R^-T B (capital_cholinv_apply_rinv_f64, trans = 1): whitening.  apply_Rinv(args, apply_RinvT(args, B)) is solve(args, B),
    bit for bit."""
    return _apply(args, B, topo, 1, "apply_RinvT", False)


def apply_R(args: info, Z: torch.Tensor, topo) -> torch.Tensor:
    """X = R Z with the factor R of a previous `factor(B, args, topo)` (capital_cholinv_apply_r_f64, trans = 0); B Z = apply_RT(args,
    apply_R(args, Z)).  Z as B for `solve`; returns X with Z's shape and device, bit-identical on every rank."""
    return _apply(args, Z, topo, 0, "apply_R", True)


def apply_RT(args: info, Z: torch.Tensor, topo) -> torch.Tensor:
    """X = R^T Z (capital_cholinv_apply_r_f64, trans = 1): the back-transform x = R^T y of `sygst(..., itype=3)`, and samples of
    covariance B from white noise Z."""
    return _apply(args, Z, topo, 1, "apply_RT", True)


def inverse_residual(A: matrix, Ainv: torch.Tensor, args: info, topo) -> float:
    """inverse::validate (test/inverse/validate.hpp:7-34): ||A Ainv - I||_F / ||I||_F, with Ainv as `inverse(args, topo)` returned it."""
    count = _check_factors(args, "inverse_residual")
    if not isinstance(A, matrix) or A.num_rows_global != args.global_dim or A.num_columns_global != args.global_dim \
            or A.num_rows_local != args.local_dim:
        raise ValueError("cholinv.inverse_residual: A is not the factored matrix's local block")
    if not isinstance(Ainv, torch.Tensor) or Ainv.dtype != torch.float64 or Ainv.numel() != count or not Ainv.is_contiguous():
        raise ValueError(f"cholinv.inverse_residual: Ainv must be a contiguous float64 tensor of {count} elements")
    ctx = topo.context()
    r = C.c_double()
    ctx.check(_lib.lib().capital_cholinv_inverse_residual_f64(ctx.handle, A.data.data_ptr(), args.global_dim,
                                                              _lib.UPPERTRI_PACKED if args.serialize else _lib.RECT,
                                                              Ainv.data_ptr(), C.byref(r)))
    return float(r.value)


_BATCHED_MAX_N = 512


def _check_batched(t, what: str, name: str, ranks):
    """ValueError unless t is a non-empty float64 tensor of one of the ranks in `ranks` (the device is checked by the caller, last)"""
    if not isinstance(t, torch.Tensor) or t.dtype != torch.float64:
        raise ValueError(f"cholinv.{what}: {name} must be a float64 tensor")
    if t.dim() not in ranks or t.numel() == 0:
        raise ValueError(f"cholinv.{what}: {name} has shape {tuple(t.shape)}")


def factor_batched(A: torch.Tensor, topo):
    """Factor a batch of SPD matrices at once (capital_cholinv_factor_batched_f64): A[b] = R[b].mT @ R[b] and Rinv[b] = R[b]^-1.
    A: a CUDA float64 tensor of shape (b, n, n) with 1 <= n <= 512.  Only the LOWER triangle of each A[b] in torch indexing is read
    (A[b, i, j] with i >= j, the diagonal included); A is never written.  Returns (R, Rinv, info): R and Rinv of shape (b, n, n), upper
    triangular in torch indexing with exact zeros below the diagonal, and info, an int32 tensor of shape (b,): 0 where the factor
    succeeded, else the 1-based pivot that was not positive.  A matrix that is not positive definite does not raise: check info, as
    for torch.linalg.cholesky_ex.  Enqueued on the current stream without a host synchronisation.  On a grid, each rank factors its
    own batch on its own GPU."""
    _check_batched(A, "factor_batched", "A", (3,))
    b, n = A.shape[0], A.shape[1]
    if A.shape[2] != n:
        raise ValueError(f"cholinv.factor_batched: A must have shape (b, n, n), got {tuple(A.shape)}")
    if n > _BATCHED_MAX_N:
        raise ValueError(f"cholinv.factor_batched: n = {n} > {_BATCHED_MAX_N} (factor such matrices one by one with cholinv.factor)")
    if not A.is_cuda:
        raise ValueError("cholinv.factor_batched: A must be a CUDA tensor")
    # a row-major A[b] is the column-major A[b]^T: the upper triangle the library reads is A[b]'s lower triangle in torch indexing
    Ac = A.contiguous()
    Rc = torch.empty_like(Ac)
    Ric = torch.empty_like(Ac)
    info = torch.empty(b, dtype=torch.int32, device=A.device)
    ctx = topo.context()
    ctx.check(_lib.lib().capital_cholinv_factor_batched_f64(ctx.handle, n, b, Ac.data_ptr(), Rc.data_ptr(), Ric.data_ptr(),
                                                            info.data_ptr()))
    # column-major R[b] in a row-major buffer reads as R[b]^T: hand back the transposed views
    return Rc.mT, Ric.mT, info


def solve_batched(Rinv: torch.Tensor, B: torch.Tensor, topo) -> torch.Tensor:
    """X[b] = A[b]^-1 B[b] with Rinv from `factor_batched` (capital_cholinv_solve_batched_f64): X = Rinv (Rinv^T B).  Rinv: CUDA float64
    (b, n, n), upper triangular in torch indexing (only that triangle is read); B: CUDA float64 (b, n) or (b, n, k).  Returns X with B's
    shape.  Enqueued on the current stream; deterministic."""
    _check_batched(Rinv, "solve_batched", "Rinv", (3,))
    _check_batched(B, "solve_batched", "B", (2, 3))
    b, n = Rinv.shape[0], Rinv.shape[1]
    if Rinv.shape[2] != n:
        raise ValueError(f"cholinv.solve_batched: Rinv must have shape (b, n, n), got {tuple(Rinv.shape)}")
    if n > _BATCHED_MAX_N:
        raise ValueError(f"cholinv.solve_batched: n = {n} > {_BATCHED_MAX_N}")
    if B.shape[0] != b or B.shape[1] != n:
        raise ValueError(f"cholinv.solve_batched: B must have shape ({b}, {n}) or ({b}, {n}, k), got {tuple(B.shape)}")
    if not Rinv.is_cuda or not B.is_cuda or Rinv.device != B.device:
        raise ValueError("cholinv.solve_batched: Rinv and B must be CUDA tensors on the same device")
    k = 1 if B.dim() == 2 else B.shape[2]
    Uc = Rinv.mT.contiguous()                                # column-major Rinv[b] (no copy for factor_batched's output)
    Bc = B.contiguous() if B.dim() == 2 else B.mT.contiguous()  # column-major n x k per matrix
    Xc = torch.empty_like(Bc)
    ctx = topo.context()
    ctx.check(_lib.lib().capital_cholinv_solve_batched_f64(ctx.handle, n, b, Uc.data_ptr(), k, Bc.data_ptr(), Xc.data_ptr()))
    return Xc if B.dim() == 2 else Xc.mT.contiguous()
