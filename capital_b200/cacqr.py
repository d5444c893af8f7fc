"""qr::cacqr -- host-side mirror of the reference's CholeskyQR2 entry points (src/alg/qr/cacqr/cacqr.h:42-49).

    ci = cholinv.info(complete_inv, split, bc_mult_dim, 'U')
    args = cacqr.info(num_iter, ci)                 # 1 = CholeskyQR, 2 = CholeskyQR2 (cacqr.h:28-32), 3 = shifted CholeskyQR3
    cacqr.factor(A, args, topo)                     # cacqr.hpp:217-248 -> args.Q (rect), args.R (packed upper)
    Y = cacqr.apply_QT(B, args, topo)               # cacqr.h:55: Q^T B      (capital_cacqr_apply_qt_f64)
    C = cacqr.apply_Q(Z, args, topo)                # cacqr.h:52: Q Z        (capital_cacqr_apply_q_f64)
    X = cacqr.lstsq(args, B, topo)                  # argmin ||A X - B|| = R^-1 Q^T B   (capital_cacqr_lstsq_f64)
    Q, R, info = cacqr.factor_batched(A, topo, 2)   # many (b, m, n) matrices, n <= 512, one GPU (capital_cacqr_factor_batched_f64)
    X = cacqr.lstsq_batched(Q, R, B, topo)          # X[b] = R[b]^-1 Q[b]^T B[b]  (capital_cacqr_lstsq_batched_f64)

num_iter = 3 is shifted CholeskyQR3 (Fukaya et al., SIAM J. Sci. Comput. 42(1), 2020), an extension beyond the reference: a first
sweep on the shifted Gram matrix G + s I, s = 11 (m n + n (n + 1)) 2^-53 trace(G), then CholeskyQR2 on its Q; R = R3 R2 R1.  It
factors matrices with condition numbers up to about 1e12 (CholeskyQR2 breaks down past about 1e8), on every grid the factor runs
on, for one sweep more.  A numerically rank-deficient A raises CapitalError with CAPITAL_ERR_NOT_SPD.

apply_QT / apply_Q / lstsq run on one GPU and on the 1D row grid (topo.rect with c = 1).  B and C hold this rank's rows (the rows
of A.data: shape (rows_local,) or (rows_local, k)); Y, Z and X are the full n-row right-hand sides, the same on every rank.
"""
from __future__ import annotations
import ctypes as C
import torch
from . import _lib
from . import cholinv as _ci
from .matrix import matrix


class info:
    def __init__(self, num_iter: int, cholesky_inverse_args: _ci.info, serialize: bool = True):
        if int(num_iter) not in (1, 2, 3):
            raise ValueError(f"cacqr.info: num_iter must be 1 (CholeskyQR), 2 (CholeskyQR2) or 3 (shifted CholeskyQR3), got {num_iter}")
        self.num_iter = int(num_iter)
        self.cholesky_inverse_args = cholesky_inverse_args
        self.serialize = serialize
        self.Q = None
        self.R = None
        self.n = 0
        self.rows_local = 0
        self.m_global = 0
        self.n_global = 0


def factor(A: matrix, args: info, topo):
    ctx = topo.context()
    m, n = A.num_rows_global, A.num_columns_global
    dev = A.data.device
    pin = dev.type == "cpu"
    if args.Q is None or args.Q.numel() != A.data.numel() or args.Q.device != dev:
        args.Q = torch.empty_like(A.data, pin_memory=pin) if pin else torch.empty_like(A.data)
    lc = A.num_columns_local
    rcount = lc * (lc + 1) // 2 if args.serialize else lc * lc
    if args.R is None or args.R.numel() != rcount or args.R.device != dev:
        args.R = torch.empty(rcount, dtype=torch.float64, device=dev, pin_memory=pin)
    args.n = lc
    args.rows_local = A.num_rows_local
    args.m_global, args.n_global = m, n
    cargs = args.cholesky_inverse_args._c()
    ctx.check(_lib.lib().capital_cacqr_factor_f64(ctx.handle, A.data.data_ptr(), m, n, args.num_iter, C.byref(cargs),
                                                  _lib.UPPERTRI_PACKED if args.serialize else _lib.RECT,
                                                  args.Q.data_ptr(), args.R.data_ptr()))


def construct_Q(args: info, topo=None) -> torch.Tensor:
    return args.Q.view(args.n, args.rows_local).t()


def construct_R(args: info, topo=None) -> torch.Tensor:
    return _ci._expand(args.R, args.n, args.serialize)


def validate(A: matrix, args: info, topo):
    """(residual, orthogonality) of qr::validate (test/qr/validate.hpp:7-52)."""
    ctx = topo.context()
    r, o = C.c_double(), C.c_double()
    ctx.check(_lib.lib().capital_cacqr_residual_f64(ctx.handle, A.data.data_ptr(), A.num_rows_global, A.num_columns_global,
                                                    args.Q.data_ptr(), _lib.UPPERTRI_PACKED if args.serialize else _lib.RECT,
                                                    args.R.data_ptr(), C.byref(r), C.byref(o)))
    return float(r.value), float(o.value)


def _check(name: str, args: info, T, rows: int, what: str) -> int:
    """ValueError unless `args` holds factors and T is a float64 tensor of `rows` rows (1-D or 2-D); returns the column count."""
    if args.Q is None or args.R is None or args.m_global <= 0 or args.n_global <= 0:
        raise ValueError(f"cacqr.{name}: `args` holds no factors (run cacqr.factor first)")
    if not isinstance(T, torch.Tensor) or T.dtype != torch.float64:
        raise ValueError(f"cacqr.{name}: {what} must be a float64 tensor")
    if T.dim() not in (1, 2) or T.shape[0] != rows or T.numel() == 0:
        raise ValueError(f"cacqr.{name}: {what} must have shape ({rows},) or ({rows}, k), got {tuple(T.shape)}")
    if args.Q.numel() != args.rows_local * args.n:
        raise ValueError(f"cacqr.{name}: args.Q does not hold rows_local x n values")
    return 1 if T.dim() == 1 else T.shape[1]


def _colmajor(T: torch.Tensor) -> torch.Tensor:
    return T.contiguous() if T.dim() == 1 else T.t().contiguous()


def _result(Tc: torch.Tensor, dim: int) -> torch.Tensor:
    return Tc if dim == 1 else Tc.t().contiguous()


def apply_QT(B: torch.Tensor, args: info, topo) -> torch.Tensor:
    """Q^T B (capital_cacqr_apply_qt_f64).  B: this rank's rows, (rows_local,) or (rows_local, k), float64, on CUDA or the host.
    Returns Y with shape (n,) or (n, k) on B's device, bit-identical on every rank."""
    k = _check("apply_QT", args, B, args.rows_local, "B")
    Bc = _colmajor(B)
    Yc = torch.empty((args.n_global,) if B.dim() == 1 else (k, args.n_global), dtype=torch.float64, device=B.device)
    ctx = topo.context()
    ctx.check(_lib.lib().capital_cacqr_apply_qt_f64(ctx.handle, args.m_global, args.n_global, args.Q.data_ptr(), k, Bc.data_ptr(),
                                                    args.rows_local, Yc.data_ptr(), args.n_global))
    return _result(Yc, B.dim())


def apply_Q(Z: torch.Tensor, args: info, topo) -> torch.Tensor:
    """Q Z (capital_cacqr_apply_q_f64).  Z: (n,) or (n, k), float64, the same on every rank.  Returns this rank's rows of Q Z,
    (rows_local,) or (rows_local, k), on Z's device."""
    k = _check("apply_Q", args, Z, args.n_global, "Z")
    Zc = _colmajor(Z)
    Cc = torch.empty((args.rows_local,) if Z.dim() == 1 else (k, args.rows_local), dtype=torch.float64, device=Z.device)
    ctx = topo.context()
    ctx.check(_lib.lib().capital_cacqr_apply_q_f64(ctx.handle, args.m_global, args.n_global, args.Q.data_ptr(), k, Zc.data_ptr(),
                                                   args.n_global, Cc.data_ptr(), args.rows_local))
    return _result(Cc, Z.dim())


def lstsq(args: info, B: torch.Tensor, topo) -> torch.Tensor:
    """argmin_X ||A X - B||_F = R^-1 Q^T B from the factors of `factor(A, args, topo)` (capital_cacqr_lstsq_f64).  B: this rank's
    rows, (rows_local,) or (rows_local, k), float64, on CUDA or the host.  Returns X with shape (n,) or (n, k) on B's device,
    bit-identical on every rank."""
    k = _check("lstsq", args, B, args.rows_local, "B")
    n = args.n_global
    if args.R.numel() != (n * (n + 1) // 2 if args.serialize else n * n):
        raise ValueError("cacqr.lstsq: args.R does not hold an n x n factor")
    Bc = _colmajor(B)
    Xc = torch.empty((n,) if B.dim() == 1 else (k, n), dtype=torch.float64, device=B.device)
    ctx = topo.context()
    ctx.check(_lib.lib().capital_cacqr_lstsq_f64(ctx.handle, args.m_global, n, args.Q.data_ptr(),
                                                 _lib.UPPERTRI_PACKED if args.serialize else _lib.RECT, args.R.data_ptr(), k,
                                                 Bc.data_ptr(), args.rows_local, Xc.data_ptr(), n))
    return _result(Xc, B.dim())


_BATCHED_MAX_N = 512


def _check_batched(t, what: str, name: str, ranks):
    """ValueError unless t is a non-empty float64 tensor of one of the ranks in `ranks` (the device is checked by the caller, last)"""
    if not isinstance(t, torch.Tensor) or t.dtype != torch.float64:
        raise ValueError(f"cacqr.{what}: {name} must be a float64 tensor")
    if t.dim() not in ranks or t.numel() == 0:
        raise ValueError(f"cacqr.{what}: {name} has shape {tuple(t.shape)}")


def _colmajor_batch(T: torch.Tensor) -> torch.Tensor:
    """the (b, cols, rows) buffer whose matrices are T[b] column-major: T.mT itself when it is contiguous, else one copy"""
    Tt = T.mT
    return Tt if Tt.is_contiguous() else Tt.contiguous()


def factor_batched(A: torch.Tensor, topo, num_iter: int = 2):
    """QR of a batch of tall-skinny matrices at once (capital_cacqr_factor_batched_f64): A[b] = Q[b] @ R[b].  A: a CUDA float64
    tensor of shape (b, m, n) with 1 <= n <= 512 and m >= n; when A.mT is contiguous (A[b] column-major) it is read without a copy.
    num_iter: 1 = CholeskyQR, 2 = CholeskyQR2, 3 = shifted CholeskyQR3 (as in cacqr.info).  Returns (Q, R, info): Q of shape
    (b, m, n), R of shape (b, n, n), upper triangular with exact zeros below the diagonal (both .mT views of column-major buffers),
    and info, an int32 tensor of shape (b,): 0 where the factor succeeded, else the 1-based pivot of the first sweep whose Gram
    matrix was not positive definite (Q[b] and R[b] are then unspecified).  A failure does not raise: check info.  Enqueued on the
    current stream without a host synchronisation.  On a grid, each rank factors its own batch on its own GPU."""
    _check_batched(A, "factor_batched", "A", (3,))
    b, m, n = A.shape
    if int(num_iter) not in (1, 2, 3):
        raise ValueError(f"cacqr.factor_batched: num_iter must be 1, 2 or 3, got {num_iter}")
    if n > _BATCHED_MAX_N:
        raise ValueError(f"cacqr.factor_batched: n = {n} > {_BATCHED_MAX_N} (factor such matrices one by one with cacqr.factor)")
    if m < n:
        raise ValueError(f"cacqr.factor_batched: m = {m} < n = {n}")
    if not A.is_cuda:
        raise ValueError("cacqr.factor_batched: A must be a CUDA tensor")
    Ac = _colmajor_batch(A)
    Qc = torch.empty((b, n, m), dtype=torch.float64, device=A.device)
    Rc = torch.empty((b, n, n), dtype=torch.float64, device=A.device)
    info = torch.empty(b, dtype=torch.int32, device=A.device)
    ctx = topo.context()
    ctx.check(_lib.lib().capital_cacqr_factor_batched_f64(ctx.handle, m, n, b, int(num_iter), Ac.data_ptr(), Qc.data_ptr(),
                                                          Rc.data_ptr(), info.data_ptr()))
    return Qc.mT, Rc.mT, info


def lstsq_batched(Q: torch.Tensor, R: torch.Tensor, B: torch.Tensor, topo) -> torch.Tensor:
    """X[b] = R[b]^-1 Q[b]^T B[b] = argmin ||A[b] X - B[b]|| from the outputs of `factor_batched` (capital_cacqr_lstsq_batched_f64).
    Q: CUDA float64 (b, m, n); R: CUDA float64 (b, n, n), upper triangular (only that triangle is read); B: CUDA float64 (b, m) or
    (b, m, k).  Returns X of shape (b, n) or (b, n, k).  Enqueued on the current stream; deterministic."""
    _check_batched(Q, "lstsq_batched", "Q", (3,))
    _check_batched(R, "lstsq_batched", "R", (3,))
    _check_batched(B, "lstsq_batched", "B", (2, 3))
    b, m, n = Q.shape
    if R.shape != (b, n, n):
        raise ValueError(f"cacqr.lstsq_batched: R must have shape ({b}, {n}, {n}), got {tuple(R.shape)}")
    if n > _BATCHED_MAX_N:
        raise ValueError(f"cacqr.lstsq_batched: n = {n} > {_BATCHED_MAX_N}")
    if m < n:
        raise ValueError(f"cacqr.lstsq_batched: m = {m} < n = {n}")
    if B.shape[0] != b or B.shape[1] != m:
        raise ValueError(f"cacqr.lstsq_batched: B must have shape ({b}, {m}) or ({b}, {m}, k), got {tuple(B.shape)}")
    if not Q.is_cuda or not R.is_cuda or not B.is_cuda or len({Q.device, R.device, B.device}) != 1:
        raise ValueError("cacqr.lstsq_batched: Q, R and B must be CUDA tensors on the same device")
    k = 1 if B.dim() == 2 else B.shape[2]
    Qc, Rc = _colmajor_batch(Q), _colmajor_batch(R)
    Bc = B.contiguous() if B.dim() == 2 else _colmajor_batch(B)
    Xc = torch.empty((b, n) if B.dim() == 2 else (b, k, n), dtype=torch.float64, device=B.device)
    ctx = topo.context()
    ctx.check(_lib.lib().capital_cacqr_lstsq_batched_f64(ctx.handle, m, n, b, Qc.data_ptr(), Rc.data_ptr(), k, Bc.data_ptr(),
                                                         Xc.data_ptr()))
    return Xc if B.dim() == 2 else Xc.mT
