"""Batched symmetric eigensolver: the eigenvalues and eigenvectors of many small symmetric matrices in one call
(capital_syevj_batched_f64, parallel cyclic Jacobi on the GPU)."""
from __future__ import annotations
import torch
from . import _lib
from .cholinv import _BATCHED_MAX_N


def syevj_batched(A: torch.Tensor, topo):
    """A[b] = V[b] @ diag(w[b]) @ V[b].mT for many symmetric matrices (capital_syevj_batched_f64).  A: CUDA float64 (b, n, n),
    1 <= n <= 512, symmetric; only its lower triangle in torch indexing (A[b, i, j], i >= j) is read, as in cholinv.factor_batched.
    Returns (w, V, info): eigenvalues w (b, n) in ascending order, eigenvectors V (b, n, n) in the columns, and info (b,): 0 when the
    matrix converged, 1 when it did not within the sweep bound (w and V then hold the last iterate) or when it contains NaN or Inf
    (outputs unspecified).  Nothing raises for such a matrix, and the others keep their bits.  Every matrix gets the same bits
    whatever batch it is in.  For n > 64 the call synchronises with the host once per outer sweep; for n <= 64 it is enqueued on the
    current stream without one."""
    what = "syevj_batched"
    if not isinstance(A, torch.Tensor) or A.dtype != torch.float64:
        raise ValueError(f"eig.{what}: A must be a float64 tensor")
    if A.dim() != 3 or A.numel() == 0 or A.shape[1] != A.shape[2]:
        raise ValueError(f"eig.{what}: A must have shape (b, n, n), got {tuple(A.shape)}")
    b, n = A.shape[0], A.shape[1]
    if n > _BATCHED_MAX_N:
        raise ValueError(f"eig.{what}: n = {n} > {_BATCHED_MAX_N}")
    if not A.is_cuda:
        raise ValueError(f"eig.{what}: A must be a CUDA tensor")
    Ac = A.contiguous()  # row-major A[b] is column-major A[b]^T: the library's upper triangle is A[b]'s lower one
    w = torch.empty(b, n, dtype=torch.float64, device=A.device)
    Vc = torch.empty(b, n, n, dtype=torch.float64, device=A.device)
    info = torch.empty(b, dtype=torch.int32, device=A.device)
    ctx = topo.context()
    ctx.check(_lib.lib().capital_syevj_batched_f64(ctx.handle, n, b, Ac.data_ptr(), w.data_ptr(), Vc.data_ptr(), info.data_ptr()))
    return w, Vc.mT.contiguous(), info

