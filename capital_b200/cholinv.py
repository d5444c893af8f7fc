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
    Ainv = cholinv.inverse_batched(Rinv, topo)                       # A[b]^-1 from the batched factors
    C = cholinv.sygst_batched(A2, R, Rinv, topo, itype=1)            # the batched sygst, itypes 1, 2 and 3
    X = cholinv.apply_Rinv_batched(Rinv, Y, topo)                    # and apply_RinvT_batched, apply_R_batched(R, Z), apply_RT_batched
    w, X, info = cholinv.eigh_batched(A2, A, topo, itype=1)          # A2[b] x = l A[b] x (scipy.linalg.eigh conventions)

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


def _square_batch(t, what: str, name: str, like=None):
    """(b, n) of a (b, n, n) tensor, or ValueError; with `like` = (b, n) the shapes must agree"""
    b, n = t.shape[0], t.shape[1]
    if t.shape[2] != n or (like is not None and (b, n) != like):
        want = "(b, n, n)" if like is None else f"({like[0]}, {like[1]}, {like[1]})"
        raise ValueError(f"cholinv.{what}: {name} must have shape {want}, got {tuple(t.shape)}")
    return b, n


def _check_n(n: int, what: str):
    if n > _BATCHED_MAX_N:
        raise ValueError(f"cholinv.{what}: n = {n} > {_BATCHED_MAX_N}")


def _check_itype(itype, what: str):
    if isinstance(itype, bool) or itype not in (1, 2, 3):
        raise ValueError(f"cholinv.{what}: itype must be 1, 2 or 3, got {itype!r}")


def _check_cuda(what: str, *ts):
    if not all(t.is_cuda for t in ts) or len({t.device for t in ts}) != 1:
        raise ValueError(f"cholinv.{what}: every tensor must be a CUDA tensor, all on the same device")


def inverse_batched(Rinv: torch.Tensor, topo) -> torch.Tensor:
    """A[b]^-1 = Rinv[b] @ Rinv[b].mT (LAPACK potri) with Rinv from `factor_batched` (capital_cholinv_inverse_batched_f64).  Rinv: CUDA
    float64 (b, n, n), 1 <= n <= 512, upper triangular in torch indexing (only that triangle is read; factor_batched's output goes in
    without a copy).  Returns (b, n, n), exactly symmetric.  Each matrix gets the bits of `inverse` on the same factor.  Enqueued on the
    current stream without a host synchronisation."""
    what = "inverse_batched"
    _check_batched(Rinv, what, "Rinv", (3,))
    b, n = _square_batch(Rinv, what, "Rinv")
    _check_n(n, what)
    _check_cuda(what, Rinv)
    Ui = Rinv.mT.contiguous()  # column-major Rinv[b]
    out = torch.empty(b, n, n, dtype=torch.float64, device=Rinv.device)
    ctx = topo.context()
    ctx.check(_lib.lib().capital_cholinv_inverse_batched_f64(ctx.handle, n, b, Ui.data_ptr(), out.data_ptr()))
    return out  # column-major and symmetric bit for bit: the buffer reads the same either way


def sygst_batched(A: torch.Tensor, R: torch.Tensor | None, Rinv: torch.Tensor | None, topo, itype: int = 1) -> torch.Tensor:
    """Many generalized symmetric-definite eigenproblems reduced to C[b] y = lambda y with the factors of `factor_batched(B)`,
    B[b] = R[b].mT @ R[b] (LAPACK dsygst, upper), with the eigenvalues of the pencil:
      itype 1: A x = lambda B x,  C = Rinv^T A Rinv (capital_cholinv_sygst_batched_f64),    back-transform x = apply_Rinv_batched(Rinv, y);
      itype 2: A B x = lambda x,  C = R A R^T       (capital_cholinv_sygst_ab_batched_f64), back-transform x = apply_Rinv_batched(Rinv, y);
      itype 3: B A x = lambda x,  C = R A R^T       (capital_cholinv_sygst_ab_batched_f64), back-transform x = apply_RT_batched(R, y).
    A: CUDA float64 (b, n, n), symmetric; only its lower triangle in torch indexing (A[b, i, j], i >= j) is read, as in factor_batched.
    itype 1 reads only Rinv, itypes 2 and 3 only R (the other may be None); only their upper triangles are read.  Returns C (b, n, n),
    exactly symmetric, with the bits of `sygst` on the same factors.  Enqueued on the current stream without a host synchronisation."""
    what = "sygst_batched"
    _check_batched(A, what, "A", (3,))
    for name, t in (("R", R), ("Rinv", Rinv)):
        if t is not None:
            _check_batched(t, what, name, (3,))
    like = _square_batch(A, what, "A")
    for name, t in (("R", R), ("Rinv", Rinv)):
        if t is not None:
            _square_batch(t, what, name, like)
    b, n = like
    _check_n(n, what)
    _check_itype(itype, what)
    F = Rinv if itype == 1 else R
    if F is None:
        raise ValueError(f"cholinv.{what}: itype {itype} reads {'Rinv' if itype == 1 else 'R'}, which is None")
    _check_cuda(what, A, F)
    Ac = A.contiguous()  # row-major A[b] is column-major A[b]^T: the library's upper triangle is A[b]'s lower one
    Fc = F.mT.contiguous()
    out = torch.empty(b, n, n, dtype=torch.float64, device=A.device)
    ctx = topo.context()
    fn = _lib.lib().capital_cholinv_sygst_batched_f64 if itype == 1 else _lib.lib().capital_cholinv_sygst_ab_batched_f64
    ctx.check(fn(ctx.handle, n, b, Fc.data_ptr(), Ac.data_ptr(), out.data_ptr()))
    return out


def _apply_batched(F: torch.Tensor, B: torch.Tensor, topo, trans: int, what: str, fname: str, factor_r: bool) -> torch.Tensor:
    """X[b] = op(F[b]) B[b] with F = R (factor_r) or Rinv from factor_batched: the checks and layout shared by the apply_*_batched calls"""
    _check_batched(F, what, fname, (3,))
    _check_batched(B, what, "B", (2, 3))
    b, n = _square_batch(F, what, fname)
    if B.shape[0] != b or B.shape[1] != n:
        raise ValueError(f"cholinv.{what}: B must have shape ({b}, {n}) or ({b}, {n}, k), got {tuple(B.shape)}")
    _check_n(n, what)
    _check_cuda(what, F, B)
    k = 1 if B.dim() == 2 else B.shape[2]
    Fc = F.mT.contiguous()                                      # column-major F[b] (no copy for factor_batched's output)
    Bc = B.contiguous() if B.dim() == 2 else B.mT.contiguous()  # column-major n x k per matrix
    Xc = torch.empty_like(Bc)
    ctx = topo.context()
    fn = _lib.lib().capital_cholinv_apply_r_batched_f64 if factor_r else _lib.lib().capital_cholinv_apply_rinv_batched_f64
    ctx.check(fn(ctx.handle, n, b, Fc.data_ptr(), trans, k, Bc.data_ptr(), Xc.data_ptr()))
    return Xc if B.dim() == 2 else Xc.mT.contiguous()


def apply_Rinv_batched(Rinv: torch.Tensor, B: torch.Tensor, topo) -> torch.Tensor:
    """X[b] = Rinv[b] @ B[b] = R[b]^-1 B[b] (capital_cholinv_apply_rinv_batched_f64, trans = 0): the back-transform of sygst_batched for
    itypes 1 and 2.  Rinv as for `solve_batched`; B: CUDA float64 (b, n) or (b, n, k).  Returns X with B's shape, with the bits of
    `apply_Rinv` on the same factor.  Enqueued on the current stream; deterministic."""
    return _apply_batched(Rinv, B, topo, 0, "apply_Rinv_batched", "Rinv", False)


def apply_RinvT_batched(Rinv: torch.Tensor, B: torch.Tensor, topo) -> torch.Tensor:
    """X[b] = Rinv[b].mT @ B[b] = R[b]^-T B[b] (trans = 1): whitening.  As apply_Rinv_batched otherwise."""
    return _apply_batched(Rinv, B, topo, 1, "apply_RinvT_batched", "Rinv", False)


def apply_R_batched(R: torch.Tensor, B: torch.Tensor, topo) -> torch.Tensor:
    """X[b] = R[b] @ B[b] with R from `factor_batched` (capital_cholinv_apply_r_batched_f64, trans = 0); only R's upper triangle in
    torch indexing is read.  As apply_Rinv_batched otherwise."""
    return _apply_batched(R, B, topo, 0, "apply_R_batched", "R", True)


def apply_RT_batched(R: torch.Tensor, B: torch.Tensor, topo) -> torch.Tensor:
    """X[b] = R[b].mT @ B[b] (trans = 1): the back-transform of sygst_batched for itype 3, and samples of covariance A[b] from white
    noise B[b].  As apply_R_batched otherwise."""
    return _apply_batched(R, B, topo, 1, "apply_RT_batched", "R", True)


def eigh_batched(A: torch.Tensor, B: torch.Tensor, topo, itype: int = 1):
    """Generalized symmetric-definite eigenproblems of many small pencils, with the conventions of scipy.linalg.eigh(a, b, type=itype):
      itype 1: A[b] x = lambda B[b] x,  itype 2: A[b] B[b] x = lambda x,  itype 3: B[b] A[b] x = lambda x.
    A, B: CUDA float64 (b, n, n), 1 <= n <= 512, symmetric, B positive definite; only their lower triangles in torch indexing are read.
    Returns (w, X, info): eigenvalues w (b, n) in ascending order, eigenvectors X (b, n, n) in the columns, normalised X^T B X = I for
    itypes 1 and 2 and X^T B^-1 X = I for itype 3, and factor_batched's info (b,).  A matrix with info != 0 gets NaN in w and X and
    leaves the others untouched; nothing raises for it.
    The composition: factor_batched(B), sygst_batched, torch.linalg.eigh on C (the eigensolver is torch's, not this library's), then
    apply_Rinv_batched (itypes 1, 2) or apply_RT_batched (itype 3).  torch.linalg.eigh synchronises with the host."""
    what = "eigh_batched"
    _check_batched(A, what, "A", (3,))
    _check_batched(B, what, "B", (3,))
    like = _square_batch(A, what, "A")
    _square_batch(B, what, "B", like)
    b, n = like
    _check_n(n, what)
    _check_itype(itype, what)
    _check_cuda(what, A, B)
    R, Rinv, info = factor_batched(B, topo)
    C = sygst_batched(A, R, Rinv, topo, itype)
    bad = info != 0
    # a failed factor's C is replaced by the identity on the device (no host synchronisation), so that eigh neither raises nor spends
    # its iterations on it; its eigenpairs are NaN below
    C = torch.where(bad.view(b, 1, 1), torch.eye(n, dtype=torch.float64, device=C.device), C)
    w, Y = torch.linalg.eigh(C)
    X = apply_Rinv_batched(Rinv, Y, topo) if itype in (1, 2) else apply_RT_batched(R, Y, topo)
    nan = float("nan")
    return w.masked_fill(bad.view(b, 1), nan), X.masked_fill(bad.view(b, 1, 1), nan), info
