"""ctypes binding of the C ABI (include/capital_b200.h).  The shared library is built in-tree by
capital_b200/build.py; there is no fallback implementation: a missing library or device is an error."""
from __future__ import annotations
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("CAPITAL_B200_LIB") or os.path.join(_HERE, "libcapital_b200.so")  # (the env override lets tools/ bisect builds)

OK, ERR_INVALID, ERR_CUDA, ERR_NOT_SPD, ERR_COMM, ERR_UNSUPPORTED = range(6)
RECT, UPPERTRI_PACKED = 0, 1
GEMM_A_UPPER, GEMM_A_LOWER, GEMM_B_UPPER, GEMM_B_LOWER, GEMM_C_UPPER = 1, 2, 4, 8, 16

EXPORTS = [  # every symbol include/capital_b200.h declares
    "capital_grid_square", "capital_grid_rect", "capital_cholinv_bc_dimension", "capital_create",
    "capital_comm_unique_id", "capital_comm_init", "capital_comm_init_host", "capital_peer_wait_mode", "capital_set_peer_wait_mode", "capital_dist_trace_cholinv", "capital_dist_trace_cacqr", "capital_dist_trace_cholinv_inverse", "capital_dist_trace_cholinv_sygst", "capital_dist_trace_cholinv_sygst_ab", "capital_destroy", "capital_last_error", "capital_get_counters",
    "capital_reset_counters", "capital_synchronize", "capital_set_stream", "capital_release_workspace", "capital_last_factor_ms", "capital_profile_begin", "capital_profile_end", "capital_probe_dmma_f64", "capital_blas_gemm_tn_tf32", "capital_set_trailing_precision", "capital_tf32_stats", "capital_timeline_begin", "capital_timeline_end", "capital_set_overlap", "capital_distribute_symmetric_f64",
    "capital_distribute_random_f64", "capital_cholinv_factor_f64", "capital_cholinv_residual_f64", "capital_cholinv_solve_f64",
    "capital_cholinv_inverse_f64", "capital_cholinv_inverse_residual_f64", "capital_cholinv_sygst_f64", "capital_cholinv_apply_rinv_f64",
    "capital_cholinv_sygst_ab_f64", "capital_cholinv_apply_r_f64", "capital_cholinv_factor_batched_f64", "capital_cholinv_solve_batched_f64",
    "capital_cholinv_inverse_batched_f64", "capital_cholinv_sygst_batched_f64", "capital_cholinv_sygst_ab_batched_f64",
    "capital_cholinv_apply_rinv_batched_f64", "capital_cholinv_apply_r_batched_f64", "capital_syevj_batched_f64",
    "capital_cacqr_factor_f64", "capital_cacqr_residual_f64", "capital_cacqr_apply_qt_f64", "capital_cacqr_apply_q_f64",
    "capital_cacqr_lstsq_f64", "capital_cacqr_factor_batched_f64", "capital_cacqr_lstsq_batched_f64", "capital_summa_gemm_tn_f64", "capital_blas_gemm_tn_f64",
    "capital_lapack_potrf_trtri_f64",
]


class Grid(C.Structure):
    _fields_ = [(n, C.c_int) for n in ("size", "rank", "c", "d", "x", "y", "z", "layout", "num_chunks")]


class CholinvArgs(C.Structure):
    _fields_ = [("complete_inv", C.c_int64), ("split", C.c_int64), ("bc_mult_dim", C.c_int64), ("dir", C.c_char)]


class Counters(C.Structure):
    _fields_ = [("kernel_launches", C.c_int64), ("gemm_launches", C.c_int64), ("leaf_launches", C.c_int64),
                ("h2d_bytes", C.c_int64), ("d2h_bytes", C.c_int64), ("gemm_flops", C.c_double)]


ALLGATHER_FN = C.CFUNCTYPE(C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64)


class CapitalError(RuntimeError):
    def __init__(self, status: int, msg: str):
        super().__init__(f"capital_b200 status {status}: {msg}")
        self.status = status


_lib = None


def lib() -> C.CDLL:
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise ImportError(f"{LIB_PATH} is missing: run `python -m capital_b200.build` (there is no fallback path)")
    L = C.CDLL(LIB_PATH)
    vp, i64, dbl, ci = C.c_void_p, C.c_int64, C.c_double, C.c_int
    L.capital_grid_square.argtypes = [ci, ci, ci, ci, ci, C.POINTER(Grid)]
    L.capital_grid_rect.argtypes = [ci, ci, ci, ci, ci, C.POINTER(Grid)]
    L.capital_cholinv_bc_dimension.argtypes = [i64, ci, ci, i64]
    L.capital_cholinv_bc_dimension.restype = i64
    L.capital_create.argtypes = [C.POINTER(vp), C.POINTER(Grid), ci, vp]
    L.capital_comm_unique_id.argtypes = [vp]
    L.capital_comm_init.argtypes = [vp, vp]
    L.capital_comm_init_host.argtypes = [vp, ALLGATHER_FN, vp]
    L.capital_blas_gemm_tn_tf32.argtypes = [vp, i64, i64, i64, dbl, vp, i64, vp, i64, dbl, vp, i64, ci, ci]
    L.capital_set_trailing_precision.argtypes = [vp, ci]
    L.capital_tf32_stats.argtypes = [vp, C.POINTER(i64), C.POINTER(dbl)]
    L.capital_peer_wait_mode.argtypes = [vp]
    L.capital_peer_wait_mode.restype = C.c_int
    L.capital_set_peer_wait_mode.argtypes = [vp, ci]
    L.capital_dist_trace_cholinv.argtypes = [C.POINTER(Grid), i64, C.POINTER(CholinvArgs), C.POINTER(i64), i64, C.POINTER(i64)]
    L.capital_dist_trace_cacqr.argtypes = [C.POINTER(Grid), i64, i64, ci, C.POINTER(CholinvArgs), C.POINTER(i64), i64, C.POINTER(i64)]
    L.capital_destroy.argtypes = [vp]
    L.capital_destroy.restype = None
    L.capital_last_error.argtypes = [vp]
    L.capital_last_error.restype = C.c_char_p
    L.capital_get_counters.argtypes = [vp, C.POINTER(Counters)]
    L.capital_reset_counters.argtypes = [vp]
    L.capital_synchronize.argtypes = [vp]
    L.capital_set_stream.argtypes = [vp, vp]
    L.capital_release_workspace.argtypes = [vp]
    L.capital_last_factor_ms.argtypes = [vp, C.POINTER(C.c_float)]
    L.capital_profile_begin.argtypes = [vp]
    L.capital_set_overlap.argtypes = [vp, ci]
    L.capital_profile_end.argtypes = [vp, C.POINTER(dbl), C.POINTER(dbl), C.POINTER(i64)]
    L.capital_probe_dmma_f64.argtypes = [vp, C.POINTER(dbl), C.POINTER(dbl)]
    L.capital_timeline_begin.argtypes = [vp]
    L.capital_timeline_end.argtypes = [vp, C.POINTER(dbl), i64, C.POINTER(i64)]
    L.capital_distribute_symmetric_f64.argtypes = [vp, vp, i64, ci]
    L.capital_distribute_random_f64.argtypes = [vp, vp, i64, i64, i64]
    L.capital_cholinv_factor_f64.argtypes = [vp, vp, i64, C.POINTER(CholinvArgs), ci, vp, vp]
    L.capital_cholinv_residual_f64.argtypes = [vp, vp, i64, ci, vp, C.POINTER(dbl)]
    L.capital_cholinv_solve_f64.argtypes = [vp, i64, C.POINTER(CholinvArgs), ci, vp, vp, i64, vp, i64, vp, i64]
    L.capital_cholinv_inverse_f64.argtypes = [vp, i64, C.POINTER(CholinvArgs), ci, vp, vp, vp]
    L.capital_cholinv_inverse_residual_f64.argtypes = [vp, vp, i64, ci, vp, C.POINTER(dbl)]
    L.capital_dist_trace_cholinv_inverse.argtypes = [C.POINTER(Grid), i64, C.POINTER(CholinvArgs), C.POINTER(i64), i64, C.POINTER(i64)]
    L.capital_cholinv_sygst_f64.argtypes = [vp, i64, C.POINTER(CholinvArgs), ci, vp, vp, vp, vp]
    L.capital_cholinv_apply_rinv_f64.argtypes = [vp, i64, C.POINTER(CholinvArgs), ci, vp, vp, ci, i64, vp, i64, vp, i64]
    L.capital_dist_trace_cholinv_sygst.argtypes = [C.POINTER(Grid), i64, C.POINTER(CholinvArgs), C.POINTER(i64), i64, C.POINTER(i64)]
    L.capital_cholinv_sygst_ab_f64.argtypes = [vp, i64, C.POINTER(CholinvArgs), ci, vp, vp, vp]
    L.capital_cholinv_apply_r_f64.argtypes = [vp, i64, C.POINTER(CholinvArgs), ci, vp, ci, i64, vp, i64, vp, i64]
    L.capital_cholinv_factor_batched_f64.argtypes = [vp, i64, i64, vp, vp, vp, vp]
    L.capital_cholinv_solve_batched_f64.argtypes = [vp, i64, i64, vp, i64, vp, vp]
    L.capital_cholinv_inverse_batched_f64.argtypes = [vp, i64, i64, vp, vp]
    L.capital_cholinv_sygst_batched_f64.argtypes = [vp, i64, i64, vp, vp, vp]
    L.capital_cholinv_sygst_ab_batched_f64.argtypes = [vp, i64, i64, vp, vp, vp]
    L.capital_cholinv_apply_rinv_batched_f64.argtypes = [vp, i64, i64, vp, ci, i64, vp, vp]
    L.capital_cholinv_apply_r_batched_f64.argtypes = [vp, i64, i64, vp, ci, i64, vp, vp]
    L.capital_syevj_batched_f64.argtypes = [vp, i64, i64, vp, vp, vp, vp]
    L.capital_dist_trace_cholinv_sygst_ab.argtypes = [C.POINTER(Grid), i64, C.POINTER(CholinvArgs), C.POINTER(i64), i64, C.POINTER(i64)]
    L.capital_cacqr_factor_f64.argtypes = [vp, vp, i64, i64, ci, C.POINTER(CholinvArgs), ci, vp, vp]
    L.capital_cacqr_residual_f64.argtypes = [vp, vp, i64, i64, vp, ci, vp, C.POINTER(dbl), C.POINTER(dbl)]
    L.capital_cacqr_apply_qt_f64.argtypes = [vp, i64, i64, vp, i64, vp, i64, vp, i64]
    L.capital_cacqr_apply_q_f64.argtypes = [vp, i64, i64, vp, i64, vp, i64, vp, i64]
    L.capital_cacqr_lstsq_f64.argtypes = [vp, i64, i64, vp, ci, vp, i64, vp, i64, vp, i64]
    L.capital_cacqr_factor_batched_f64.argtypes = [vp, i64, i64, i64, ci, vp, vp, vp, vp]
    L.capital_cacqr_lstsq_batched_f64.argtypes = [vp, i64, i64, i64, vp, vp, i64, vp, vp]
    L.capital_summa_gemm_tn_f64.argtypes = [vp, i64, i64, i64, dbl, vp, vp, dbl, vp]
    L.capital_blas_gemm_tn_f64.argtypes = [vp, i64, i64, i64, dbl, vp, i64, vp, i64, dbl, vp, i64, ci]
    L.capital_lapack_potrf_trtri_f64.argtypes = [vp, i64, vp, i64, vp, i64, vp, i64]
    for name in EXPORTS:
        fn = getattr(L, name)
        if name not in ("capital_destroy", "capital_last_error", "capital_cholinv_bc_dimension"):
            fn.restype = ci
    _lib = L
    return L


class Context:
    """One context per process / GPU (capital_create ... capital_destroy)."""

    def __init__(self, grid: Grid, device: int = 0, stream: int | None = None):
        self.grid = grid
        self._h = C.c_void_p()
        st = lib().capital_create(C.byref(self._h), C.byref(grid), device, C.c_void_p(stream or 0))
        if st != OK:
            raise CapitalError(st, "capital_create failed (needs an sm_90 device; no CPU fallback exists)")

    def check(self, status: int):
        if status != OK:
            raise CapitalError(status, lib().capital_last_error(self._h).decode())

    @property
    def handle(self):
        return self._h

    def counters(self) -> Counters:
        c = Counters()
        self.check(lib().capital_get_counters(self._h, C.byref(c)))
        return c

    def reset_counters(self):
        self.check(lib().capital_reset_counters(self._h))

    def synchronize(self):
        self.check(lib().capital_synchronize(self._h))

    def set_stream(self, stream: int):
        self.check(lib().capital_set_stream(self._h, C.c_void_p(stream)))

    def set_trailing_precision(self, mode: int):
        """EXPERIMENTAL (BASELINE config 5): 0 = FP64 trailing updates (default), 1 = TF32 tensor cores, 3 = 3 x TF32 split operands."""
        self.check(lib().capital_set_trailing_precision(self._h, mode))

    def tf32_stats(self):
        n, f = C.c_int64(), C.c_double()
        self.check(lib().capital_tf32_stats(self._h, C.byref(n), C.byref(f)))
        return int(n.value), float(f.value)

    def peer_wait_mode(self) -> str:
        """how this rank's streams wait for a peer-written flag (capital_peer_wait_mode)"""
        return {-1: "none", 0: "memop", 1: "memop+flush", 2: "kernel"}[lib().capital_peer_wait_mode(self._h)]

    def set_peer_wait_mode(self, name: str):
        """'memop' | 'memop+flush' | 'kernel' -- between calls only"""
        self.check(lib().capital_set_peer_wait_mode(self._h, {"memop": 0, "memop+flush": 1, "kernel": 2}[name]))

    def release_workspace(self):
        """policy::cholinv::FlushIntermediates: free every work buffer (re-allocated by the next call)."""
        self.check(lib().capital_release_workspace(self._h))

    def last_factor_ms(self) -> float:
        ms = C.c_float()
        self.check(lib().capital_last_factor_ms(self._h, C.byref(ms)))
        return float(ms.value)

    def set_overlap(self, enabled: bool):
        self.check(lib().capital_set_overlap(self._h, int(enabled)))

    def profile_begin(self):
        self.check(lib().capital_profile_begin(self._h))

    def profile_end(self):
        """(summed duration in ms, algorithmic flops, launches) of the dominant kernel since profile_begin."""
        ms, fl, n = C.c_double(), C.c_double(), C.c_int64()
        self.check(lib().capital_profile_end(self._h, C.byref(ms), C.byref(fl), C.byref(n)))
        return float(ms.value), float(fl.value), int(n.value)

    def timeline_begin(self):
        self.check(lib().capital_timeline_begin(self._h))

    def timeline_end(self):
        """numpy array (launches x 8): stream id, kind, start ms, end ms, a, b, c, 0 -- see capital_timeline_end in the header."""
        import numpy as np
        n = C.c_int64()
        cap = 1 << 18
        buf = np.zeros((cap, 8), dtype=np.float64)
        self.check(lib().capital_timeline_end(self._h, buf.ctypes.data_as(C.POINTER(C.c_double)), cap, C.byref(n)))
        return buf[:min(cap, n.value)].copy()

    def probe_dmma(self):
        """(TFLOP/s, ms) of a register-resident DMMA.16x8x16 loop on every SM: the FP64 tensor-pipe ceiling of this device now."""
        tf, ms = C.c_double(), C.c_double()
        self.check(lib().capital_probe_dmma_f64(self._h, C.byref(tf), C.byref(ms)))
        return float(tf.value), float(ms.value)

    def close(self):
        if self._h:
            lib().capital_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
