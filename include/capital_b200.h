/* capital_b200 -- C ABI of the H100-native CholInv / CholeskyQR2 hot path.
 *
 * Drop-in boundary for the factorization entry points of tbennun/capital (a header-only C++14
 * template library; it has no FFI of its own, so each entry point below names the reference
 * template it replaces, paths relative to the reference root).  Plain pointers and sizes only;
 * no torch / C++ types.  All matrices are FP64, column-major, in the reference's element-cyclic
 * layout (src/matrix/matrix.hpp:6-19, src/matrix/structure.h:13,37-39):
 *   global (row gy, col gx) lives on process (x = gx mod d, y = gy mod d) at local (col gx/d, row gy/d);
 *   `rect` local block: element (col i, row j) at i*ld + j;  packed `uppertri`: (i, j<=i) at i(i+1)/2 + j.
 *
 * Pointers passed to the compute entry points may be device pointers (resident HBM, the fast
 * path) or host pointers (the library stages them through pinned buffers: this is the
 * "reference-facing" call a C++ caller of the reference would make).  There is NO CPU fallback:
 * every entry point fails with CAPITAL_ERR_CUDA when no sm_90 device is usable.
 */
#ifndef CAPITAL_B200_H
#define CAPITAL_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#if defined(__GNUC__)
#pragma GCC visibility push(default) /* the library is built with -fvisibility=hidden; only this ABI is exported */
#endif

typedef struct capital_ctx capital_ctx;

typedef enum {
  CAPITAL_OK = 0,
  CAPITAL_ERR_INVALID = 1,     /* bad argument (the reference would assert: cholinv.hpp:9,81) */
  CAPITAL_ERR_CUDA = 2,        /* CUDA runtime / driver failure, or no sm_90 device */
  CAPITAL_ERR_NOT_SPD = 3,     /* non-positive pivot in a base case (reference drops LAPACKE info: lapack/interface.hpp:39) */
  CAPITAL_ERR_COMM = 4,        /* NCCL failure */
  CAPITAL_ERR_UNSUPPORTED = 5  /* grid / policy combination outside the hot path */
} capital_status_t;

/* topo::square / topo::rect public members (src/util/topology.h:62-64,140-142). */
typedef struct {
  int size, rank;          /* world */
  int c, d;                /* replication depth, face edge (square: c x d x d; rect: c x d x c) */
  int x, y, z;             /* process column, process row, layer */
  int layout, num_chunks;  /* kept for signature parity; layout 0 only, num_chunks ignored on NVSwitch */
} capital_grid_t;

/* cholesky::cholinv<...>::info user members (src/alg/cholesky/cholinv/cholinv.h:25-30). */
typedef struct {
  int64_t complete_inv;  /* 0: skip the top-level Rinv12 block (cholinv.hpp:147) */
  int64_t split;         /* recursion split shift (>0; 1 = halves) */
  int64_t bc_mult_dim;   /* base-case depth factor (cholinv.hpp:15-18) */
  char dir;              /* must be 'U' (cholinv.hpp:9) */
} capital_cholinv_args_t;

/* serialize policy of the outputs: policy::cholinv::Serialize -> packed uppertri, NoSerialize -> rect. */
typedef enum { CAPITAL_RECT = 0, CAPITAL_UPPERTRI_PACKED = 1 } capital_structure_t;

/* counters for bench/tests: how many of OUR kernels were launched since the last reset */
typedef struct {
  int64_t kernel_launches;
  int64_t gemm_launches;
  int64_t leaf_launches;
  int64_t h2d_bytes, d2h_bytes;
  double gemm_flops;  /* flops executed by the tensor-core GEMM kernel (2*m*n*k over computed tiles) */
} capital_counters_t;

/* ---- grid helpers -------------------------------------------------------------------------- */
/* topo::square(comm, c, layout, num_chunks) rank -> (x,y,z) map, topology.h:67-95 (layout 0). */
capital_status_t capital_grid_square(int size, int rank, int c, int layout, int num_chunks, capital_grid_t* out);
/* topo::rect(comm, c, layout, num_chunks), topology.h:16-51. */
capital_status_t capital_grid_rect(int size, int rank, int c, int layout, int num_chunks, capital_grid_t* out);
/* base-case global dimension derived from bc_mult_dim, cholinv.hpp:15-18. */
int64_t capital_cholinv_bc_dimension(int64_t local_dim, int c, int d, int64_t bc_mult_dim);

/* ---- context ------------------------------------------------------------------------------- */
/* One context per process / GPU.  `stream` is a cudaStream_t (NULL = library-owned stream). */
capital_status_t capital_create(capital_ctx** ctx, const capital_grid_t* grid, int device, void* stream);
/* Multi-GPU: join the NCCL clique.  `nccl_unique_id` = 128 bytes of ncclUniqueId produced by
 * capital_comm_unique_id on rank 0 and broadcast by the caller (replaces MPI_Comm_split in
 * topology.h:84-94).  Not needed when grid.size == 1. */
capital_status_t capital_comm_unique_id(void* out128);
capital_status_t capital_comm_init(capital_ctx* ctx, const void* nccl_unique_id);
/* Same, bootstrapped through a caller-supplied host allgather instead of NCCL (MPI_Allgather in an MPI program:
 *   int ag(void* user, const void* send, void* recv, int64_t bytes) { return MPI_Allgather(send, bytes, MPI_BYTE, recv, bytes, MPI_BYTE, *(MPI_Comm*)user); }
 * ).  The library only exchanges small blobs (IPC handles) through it, at init and when its peer-visible arena has to grow;
 * matrix data never goes through it.  Must return 0 on success; recv holds size * bytes. */
typedef int (*capital_allgather_fn)(void* user, const void* send, void* recv, int64_t bytes_per_rank);
capital_status_t capital_comm_init_host(capital_ctx* ctx, capital_allgather_fn allgather, void* user);
/* How this rank's streams wait for a flag written by a peer GPU: 0 = stream memory-op wait, 1 = memory-op wait followed by a flush
 * of outstanding remote writes (CU_STREAM_WAIT_VALUE_FLUSH; the default where the device supports it), 2 = one-warp kernel spinning
 * on ld.acquire.sys, -1 = the context has not joined a clique.  Override: env CAPITAL_PEER_WAIT = memop | flush | kernel. */
int capital_peer_wait_mode(const capital_ctx* ctx);
/* Switch the wait flavour between calls (measurement: bench.py times both on the same box).  CAPITAL_ERR_UNSUPPORTED when the device
 * cannot do it (mode 1 without flush support). */
capital_status_t capital_set_peer_wait_mode(capital_ctx* ctx, int mode);
void capital_destroy(capital_ctx* ctx);
const char* capital_last_error(const capital_ctx* ctx);
capital_status_t capital_get_counters(const capital_ctx* ctx, capital_counters_t* out);
capital_status_t capital_reset_counters(capital_ctx* ctx);
capital_status_t capital_synchronize(capital_ctx* ctx);
/* Rebind the context to another caller stream (cudaStream_t): later calls are enqueued on it, ordered after everything already
 * enqueued on the previous stream.  The Python mirror calls it whenever torch's current stream changed. */
capital_status_t capital_set_stream(capital_ctx* ctx, void* stream);
/* policy::cholinv::FlushIntermediates (cholinv/policy.h:85-156): release every work buffer the context holds (the next factor call
 * re-allocates: SaveIntermediates semantics -- keep them between calls -- are the default, cholinv/policy.h:20-83). */
capital_status_t capital_release_workspace(capital_ctx* ctx);
/* time (ms) between two library-recorded CUDA events bracketing the last factor call, on its stream */
capital_status_t capital_last_factor_ms(const capital_ctx* ctx, float* ms);

/* Per-launch CUDA-event timing of the dominant kernel (the 128x128 DMMA GEMM) on the stream it is launched on:
 * begin arms it; end synchronizes and returns the summed launch durations, the algorithmic flops of those
 * launches (structure exploited) and their count.  Used by bench.py for the roofline line. */
capital_status_t capital_profile_begin(capital_ctx* ctx);
/* enabled = 0 runs the recursion on a single stream (no deferred-update overlap): isolates per-kernel durations. */
capital_status_t capital_set_overlap(capital_ctx* ctx, int enabled);
capital_status_t capital_profile_end(capital_ctx* ctx, double* kernel_ms, double* kernel_flops, int64_t* launches);
/* Timeline of the schedule (profiling aid; the image has no nsys): between begin and end every launch of the library is bracketed by
 * CUDA events on its own stream.  end synchronizes the device and writes 8 doubles per launch: stream id (0 caller, 1 critical chain,
 * 2..4 deferred (recursion depth 0..2), 5..9 push streams, 10 copy-in, 11 copy-out), kind (1 big GEMM, 2 small GEMM, 3 cluster base case, 4 leaf, 5 flag wait,
 * 6 flag signal, 7 peer DMA, 8 layout kernel), start ms, end ms, three kind-specific numbers (GEMM: m, n, k), 0. */
capital_status_t capital_timeline_begin(capital_ctx* ctx);
capital_status_t capital_timeline_end(capital_ctx* ctx, double* out, int64_t cap_records, int64_t* n_records);
/* FP64 tensor-pipe ceiling of this device right now: a register-resident DMMA.16x8x16 loop on every SM (~15 ms), CUDA-event timed.
 * The denominator of bench.py's roofline fraction. */
capital_status_t capital_probe_dmma_f64(capital_ctx* ctx, double* tflops, double* ms);

/* Test facility, no device needed: records the synchronisation-relevant operations (flag waits / signals, fused products, events,
 * peer DMA, arena windows read / written) that rank `grid->rank` would enqueue for two consecutive cholinv::factor calls, 8 int64
 * per record (kind, stream, a .. f); tests replay the traces of all ranks of a grid to prove the flag protocol cannot deadlock. */
capital_status_t capital_dist_trace_cholinv(const capital_grid_t* grid, int64_t n_global, const capital_cholinv_args_t* args,
                                            int64_t* out, int64_t cap_records, int64_t* n_records);
/* The same for two consecutive cacqr::factor calls on a rect grid with c == d > 1 (3D) or 1 < c < d (tunable; the trace includes the
 * cross-cube Gram all-reduce).  num_iter 1, 2 or 3 (3 also records the Gram shift's scalar sum: copies of the trace partials and their
 * flags, control words CTRL_SAR); other num_iter: CAPITAL_ERR_INVALID.  CAPITAL_ERR_UNSUPPORTED for the other grids. */
capital_status_t capital_dist_trace_cacqr(const capital_grid_t* grid, int64_t m_global, int64_t n_global, int num_iter,
                                          const capital_cholinv_args_t* ci_args, int64_t* out, int64_t cap_records, int64_t* n_records);
/* The same for two consecutive capital_cholinv_inverse_f64 calls (rect output) on a square grid. */
capital_status_t capital_dist_trace_cholinv_inverse(const capital_grid_t* grid, int64_t n_global, const capital_cholinv_args_t* args,
                                                    int64_t* out, int64_t cap_records, int64_t* n_records);
/* The same for two consecutive capital_cholinv_sygst_f64 calls (rect output) on a square grid. */
capital_status_t capital_dist_trace_cholinv_sygst(const capital_grid_t* grid, int64_t n_global, const capital_cholinv_args_t* args,
                                                  int64_t* out, int64_t cap_records, int64_t* n_records);
/* The same for two consecutive capital_cholinv_sygst_ab_f64 calls (rect output) on a square grid. */
capital_status_t capital_dist_trace_cholinv_sygst_ab(const capital_grid_t* grid, int64_t n_global, const capital_cholinv_args_t* args,
                                                     int64_t* out, int64_t cap_records, int64_t* n_records);

/* ---- generators (device kernels; bit-exact with the reference's drand48-based ones) ---------- */
/* matrix::distribute_symmetric(x, y, d, d, key, diagonallyDominant) -- structure.hpp:69-103. */
capital_status_t capital_distribute_symmetric_f64(capital_ctx* ctx, double* A_local, int64_t n_global,
                                                  int diagonally_dominant);
/* matrix::distribute_random(x, y, c, d, key) -- structure.hpp:106-129 (rows over d, columns over c). */
capital_status_t capital_distribute_random_f64(capital_ctx* ctx, double* A_local, int64_t m_global,
                                               int64_t n_global, int64_t key);

/* ---- CholInv ------------------------------------------------------------------------------- */
/* cholesky::cholinv<SP,IP,BP>::factor(A, args, topo) -- cholinv.hpp:6-28 (+ invoke :87-165, base
 * case policy.h:160-224 semantics: zeros on local-diagonal slots of ranks with y > x).
 * A_local: rect local block, ld = ceil(n/d), never modified.  R_local / Rinv_local: caller-owned,
 * packed upper (L(L+1)/2) or rect (L*L, lower part zero), identical on all c layers. */
capital_status_t capital_cholinv_factor_f64(capital_ctx* ctx, const double* A_local, int64_t n_global,
                                            const capital_cholinv_args_t* args, capital_structure_t out_structure,
                                            double* R_local, double* Rinv_local);
/* cholesky::validate<Alg>::residual -- test/cholesky/validate.hpp:7-49:
 * sqrt(sum_upper (R^T R - A)^2) / sqrt(sum_upper A^2), computed on the device(s). */
capital_status_t capital_cholinv_residual_f64(capital_ctx* ctx, const double* A_local, int64_t n_global,
                                              capital_structure_t structure, const double* R_local, double* residual);

/* cholesky::cholinv solve: A X = B with the outputs of capital_cholinv_factor_f64 (A = R^T R).  Collective on a grid: every rank calls
 * it with the same n_global, args (the ones given to the factor), structure and nrhs.  R_local / Rinv_local: this rank's local blocks
 * exactly as the factor wrote them (packed upper or rect).  B, X: the FULL n x nrhs right-hand side / solution, column-major,
 * ldb, ldx >= n, replicated: the same B on every rank in, bit-identical X on every rank out.  X may alias B (ldx == ldb).
 * R_local is read only when the top-level Rinv12 block was skipped (complete_inv = 0 and the top node splits); it may be NULL otherwise.
 * Rinv complete: X = Rinv (Rinv^T B).  Rinv12 skipped (split n1): Y1 = Rinv11^T B1, Y2 = Rinv22^T (B2 - R12^T Y1), X2 = Rinv22 Y2,
 * X1 = Rinv11 (Y1 - R12 X2).  The factor is read in place, one pass per product and panel of up to 32 right-hand sides; the result is
 * deterministic (same inputs, same bits).  Host or device pointers.  One GPU: enqueued on the context stream, synchronous only when X
 * is a host pointer.  Grid: synchronous; its all-reduce slots use the peer arena, so the next factor call re-clears the arena.
 * CAPITAL_ERR_UNSUPPORTED when d does not divide n on a grid. */
capital_status_t capital_cholinv_solve_f64(capital_ctx* ctx, int64_t n_global, const capital_cholinv_args_t* args,
                                           capital_structure_t structure, const double* R_local, const double* Rinv_local,
                                           int64_t nrhs, const double* B, int64_t ldb, double* X, int64_t ldx);
/* One half of the solve alone: trans = 0: X = R^-1 B (the back-transform x = R^-1 y of capital_cholinv_sygst_f64); trans = 1:
 * X = R^-T B (whitening).  Arguments, conventions and guarantees as capital_cholinv_solve_f64 (X may alias B).  Rinv complete: one pass
 * over the triangle per panel.  Rinv12 skipped: trans = 1 runs the solve's first three steps (Y1, B2 - R12^T Y1, Y2), trans = 0 its
 * last three (X2, Y1 - R12 X2, X1).  Each step is the solve's own, so apply_rinv(0) after apply_rinv(1) gives the solve's bits.  On a
 * grid it uses the solve's all-reduce slots: switching between solve and apply costs no arena clear. */
capital_status_t capital_cholinv_apply_rinv_f64(capital_ctx* ctx, int64_t n_global, const capital_cholinv_args_t* args,
                                                capital_structure_t structure, const double* R_local, const double* Rinv_local,
                                                int trans, int64_t nrhs, const double* B, int64_t ldb, double* X, int64_t ldx);
/* A product with the factor itself: trans = 0: X = R B; trans = 1: X = R^T B (the back-transform x = R^T y of
 * capital_cholinv_sygst_ab_f64 for B A x = lambda x; R^T xi draws samples of covariance B = R^T R from white noise xi).  Only R_local
 * is read, exactly as the factor wrote it; Rinv is not an argument.  Otherwise arguments, conventions and guarantees as
 * capital_cholinv_solve_f64: the full replicated B and X, X may alias B, bit-identical X on every rank, host or device pointers.  One
 * pass over R's triangle per panel of up to 32 right-hand sides.  On a grid it uses the solve's all-reduce slots: switching between
 * solve, apply_rinv and apply_r costs no arena clear. */
capital_status_t capital_cholinv_apply_r_f64(capital_ctx* ctx, int64_t n_global, const capital_cholinv_args_t* args,
                                             capital_structure_t structure, const double* R_local, int trans, int64_t nrhs,
                                             const double* B, int64_t ldb, double* X, int64_t ldx);

/* Batched CholInv on this context's GPU: `batch` independent SPD matrices of order n <= 512, each factored A_b = R_b^T R_b with
 * R_b^-1, in a few launches for the whole batch (one CTA per matrix for n <= 64, one thread-block cluster per matrix above).
 * A, R, Rinv: batch x n x n, column-major, matrix b at offset b n n.  Only the upper triangle of each A_b, the diagonal included, is
 * read; A is never written.  R_b and Rinv_b are written whole: upper triangular with exact zeros below the diagonal.  info[b] = 0 on
 * success, else the 1-based pivot that was not positive (the factor then continues with 1 in its place, and the other matrices are
 * unaffected); a non-SPD matrix is reported through info only, so the call returns CAPITAL_OK without waiting for the device.
 * Device pointers only (CAPITAL_ERR_INVALID otherwise); R and Rinv must not overlap A.  Enqueued on the context stream; never
 * communicates, so on a grid context each rank factors its own batch.  Intermediates take at most 2 GiB of device memory (kept
 * until capital_release_workspace): larger batches run in chunks.  n > 512: CAPITAL_ERR_UNSUPPORTED; n < 1, batch < 1 or a NULL
 * argument: CAPITAL_ERR_INVALID. */
capital_status_t capital_cholinv_factor_batched_f64(capital_ctx* ctx, int64_t n, int64_t batch, const double* A, double* R,
                                                    double* Rinv, int* info);
/* X_b = Rinv_b (Rinv_b^T B_b) = A_b^-1 B_b for the outputs of capital_cholinv_factor_batched_f64.  Rinv: batch x n x n as the factor
 * wrote it (only its upper triangles are read); B, X: batch x n x nrhs, column-major, matrix b at offset b n nrhs.  X may alias B.
 * Two passes over each Rinv_b per panel of up to 32 right-hand sides; deterministic.  Device pointers only; enqueued on the context
 * stream.  Errors as capital_cholinv_factor_batched_f64 (nrhs < 1: CAPITAL_ERR_INVALID). */
capital_status_t capital_cholinv_solve_batched_f64(capital_ctx* ctx, int64_t n, int64_t batch, const double* Rinv, int64_t nrhs,
                                                   const double* B, double* X);
/* The batched inverse, sygst and products with the factors: for each of `batch` matrices of order 1 <= n <= 512 the single-GPU call of
 * the same name (capital_cholinv_inverse_f64, _sygst_f64, _sygst_ab_f64, _apply_rinv_f64, _apply_r_f64), on the outputs of
 * capital_cholinv_factor_batched_f64, with that call's bits on the same factors.  All matrices column-major, matrix b at offset b n n
 * (b n nrhs for B and X).  R and Rinv are read as the batched factor wrote them, and only their upper triangles: whatever lies below
 * the diagonal changes no bit.  Of A only the upper triangle of each A_b, the diagonal included, is read (the triangle the batched
 * factor reads).  C and Ainv are written whole, exactly symmetric: the lower half is the upper half's mirror, bit for bit; they must
 * not overlap any input (CAPITAL_ERR_INVALID).  X may alias B.  Device pointers only; enqueued on the context stream with no host
 * synchronisation; never communicates, so on a grid context each rank works on its own batch.  Intermediates take at most 2 GiB of
 * device memory (kept until capital_release_workspace): larger batches run in chunks of at most 65535 matrices.  n > 512:
 * CAPITAL_ERR_UNSUPPORTED; n < 1, batch < 1, nrhs < 1, trans not 0 or 1, a NULL argument or a host pointer: CAPITAL_ERR_INVALID. */
/* Ainv_b = Rinv_b Rinv_b^T = A_b^-1 (LAPACK potri): one DMMA product of n^3 / 3 flops per matrix. */
capital_status_t capital_cholinv_inverse_batched_f64(capital_ctx* ctx, int64_t n, int64_t batch, const double* Rinv, double* Ainv);
/* itype 1: C_b = Rinv_b^T A_b Rinv_b (A x = lambda B x), n^3 flops per matrix. */
capital_status_t capital_cholinv_sygst_batched_f64(capital_ctx* ctx, int64_t n, int64_t batch, const double* Rinv, const double* A,
                                                   double* C);
/* itype 2 and 3: C_b = R_b A_b R_b^T (A B x = lambda x, B A x = lambda x), n^3 flops per matrix. */
capital_status_t capital_cholinv_sygst_ab_batched_f64(capital_ctx* ctx, int64_t n, int64_t batch, const double* R, const double* A,
                                                      double* C);
/* trans 0: X_b = Rinv_b B_b (the back-transform of itype 1 and 2); trans 1: X_b = Rinv_b^T B_b (whitening). */
capital_status_t capital_cholinv_apply_rinv_batched_f64(capital_ctx* ctx, int64_t n, int64_t batch, const double* Rinv, int trans,
                                                        int64_t nrhs, const double* B, double* X);
/* trans 0: X_b = R_b B_b; trans 1: X_b = R_b^T B_b (the back-transform of itype 3; samples of covariance A_b from white noise). */
capital_status_t capital_cholinv_apply_r_batched_f64(capital_ctx* ctx, int64_t n, int64_t batch, const double* R, int trans,
                                                     int64_t nrhs, const double* B, double* X);

/* Batched symmetric eigensolver on this context's GPU: A_b = V_b diag(w_b) V_b^T for `batch` symmetric matrices of order 1 <= n <= 512,
 * by parallel cyclic Jacobi (one CTA per matrix for n <= 64, block Jacobi on 64 x 64 DMMA tile products above).  A, V: batch x n x n,
 * column-major, matrix b at offset b n n; w: batch x n.  Only the upper triangle of each A_b, the diagonal included, is read (the
 * triangle capital_cholinv_factor_batched_f64 reads); the other may hold anything, NaN included.  w_b holds the eigenvalues in
 * ascending order and column j of V_b the eigenvector of w_b[j].  info[b] = 0 when A_b converged, 1 when it did not within the fixed
 * sweep bound (w_b and V_b then hold the last iterate); a matrix containing NaN or Inf gets info = 1 and unspecified outputs, and
 * never affects the others.  Each matrix gets the same bits whatever batch or chunk it is in, from run to run.
 * Host synchronisation: for n > 64 the call reads one device counter per outer sweep (and so returns when the work is done) to stop
 * once every matrix has converged; that is its only synchronisation.  For n <= 64 it is enqueued on the context stream with none.
 * Device pointers only; w, V and info must not overlap each other or A.  Intermediates (n > 64) take at most 2 GiB of device memory
 * (kept until capital_release_workspace): larger batches run in chunks of at most 65535 matrices.  n > 512: CAPITAL_ERR_UNSUPPORTED;
 * n < 1, batch < 1, a NULL argument, a host pointer or overlapping outputs: CAPITAL_ERR_INVALID. */
capital_status_t capital_syevj_batched_f64(capital_ctx* ctx, int64_t n, int64_t batch, const double* A, double* w, double* V,
                                           int* info);

/* cholesky::cholinv inverse: A^-1 = Rinv Rinv^T from the outputs of capital_cholinv_factor_f64 (LAPACK potri).  Collective on a grid:
 * every rank calls it with the same n_global, args (the ones given to the factor) and structure.  R_local / Rinv_local: this rank's
 * local blocks exactly as the factor wrote them; R_local is read only when the top-level Rinv12 block was skipped (complete_inv = 0
 * and the top node splits), where that block is rebuilt first with the factor's own two products; it may be NULL otherwise.
 * Ainv_local: the rank's L x L local block (L = n / d) in `structure`: packed = the upper triangle, column-packed like R (zeros on the
 * local-diagonal slots of ranks with y > x); rect = the full symmetric block, exactly symmetric (the lower half is the upper half's
 * mirror, not a second computation).  Identical on the c layers; deterministic.  One DMMA product of n^3 / 3 flops.  Ainv must not
 * overlap R or Rinv.  Host or device pointers.  One GPU: enqueued on the context stream, synchronous only when Ainv is a host
 * pointer; the only device memory is the factor's own workspace.  Grid: synchronous; the product uses the peer arena, so the next
 * factor call re-clears it.  CAPITAL_ERR_UNSUPPORTED when d does not divide n on a grid. */
capital_status_t capital_cholinv_inverse_f64(capital_ctx* ctx, int64_t n_global, const capital_cholinv_args_t* args,
                                             capital_structure_t structure, const double* R_local, const double* Rinv_local,
                                             double* Ainv_local);
/* Generalized symmetric-definite eigenproblem A x = lambda B x, reduced to standard form with the outputs of
 * capital_cholinv_factor_f64 for B = R^T R (LAPACK dsygst, itype 1, upper): C = R^-T A R^-1, so that C y = lambda y and x = R^-1 y
 * (capital_cholinv_apply_rinv_f64 with trans = 0).  Collective on a grid, with the arguments of the factor of B.  A_local: the rank's
 * L x L rect block of the symmetric A (as the generator writes it); only its GLOBAL lower triangle, the diagonal included, is read.
 * R_local / Rinv_local as for capital_cholinv_inverse_f64 (R only for a skipped top-level Rinv12, rebuilt first; NULL otherwise).
 * C_local: the rank's L x L block in `structure`, written exactly as the inverse writes A^-1: packed upper (zeros on the
 * local-diagonal slots of ranks with y > x) or the full rect block, exactly symmetric.  Identical on the c layers; deterministic.
 * n^3 DMMA flops (LAPACK's split A = U + U^T): V = U R^-1, then C = R^-T V + V^T R^-1, upper tiles only.  C must not overlap A, R
 * or Rinv.  Host or device pointers.  One GPU: enqueued on the context stream, synchronous only when C is a host pointer; with device
 * pointers the only device memory is the factor's own four L x L workspaces.  Grid: synchronous; the products use the peer arena, so
 * the next factor call re-clears it.  CAPITAL_ERR_UNSUPPORTED when d does not divide n on a grid. */
capital_status_t capital_cholinv_sygst_f64(capital_ctx* ctx, int64_t n_global, const capital_cholinv_args_t* args,
                                           capital_structure_t structure, const double* R_local, const double* Rinv_local,
                                           const double* A_local, double* C_local);
/* The other two generalized symmetric-definite eigenproblems, A B x = lambda x (LAPACK itype 2) and B A x = lambda x (itype 3), both
 * reduced to standard form with the outputs of capital_cholinv_factor_f64 for B = R^T R (LAPACK dsygst, itype 2 / 3, upper):
 * C = R A R^T, so that C y = lambda y and x = R^-1 y for itype 2 (capital_cholinv_apply_rinv_f64, trans = 0) or x = R^T y for itype 3
 * (capital_cholinv_apply_r_f64, trans = 1).  Arguments and output as capital_cholinv_sygst_f64, except that only R is read (always
 * complete, so complete_inv changes nothing) and Rinv is not an argument.  n^3 DMMA flops by the same split A = U + U^T: W = R U,
 * then C = W R^T + R W^T, upper tiles only.  C must not overlap A or R.  CAPITAL_ERR_UNSUPPORTED when d does not divide n on a grid. */
capital_status_t capital_cholinv_sygst_ab_f64(capital_ctx* ctx, int64_t n_global, const capital_cholinv_args_t* args,
                                              capital_structure_t structure, const double* R_local, const double* A_local,
                                              double* C_local);
/* inverse::validate -- test/inverse/validate.hpp:7-34: ||A Ainv - I||_F / ||I||_F over the whole matrix, computed on the device(s),
 * the diagonal taken by GLOBAL index.  A_local: the full symmetric rect local block (as the generator writes it); Ainv_local: as
 * capital_cholinv_inverse_f64 wrote it in `structure`. */
capital_status_t capital_cholinv_inverse_residual_f64(capital_ctx* ctx, const double* A_local, int64_t n_global,
                                                      capital_structure_t structure, const double* Ainv_local, double* residual);

/* ---- CholeskyQR2 --------------------------------------------------------------------------- */
/* qr::cacqr<SP,IP>::factor(A, args, topo) -- cacqr.hpp:217-248, on a topo::rect grid c x d x c.  num_iter: 1 = CQR, 2 = CQR2,
 *  3 = shifted CholeskyQR3 (an extension beyond the reference; Fukaya et al., SIAM J. Sci. Comput. 42(1), 2020): the first sweep
 *  factors G + s I, s = 11 (m n + n (n + 1)) 2^-53 trace(G), then CQR2 runs on its Q; R = R3 R2 R1.  It factors A with condition
 *  numbers up to about 1e12 (CQR2 breaks down past about 1e8), on every grid below, with the same outputs.  A numerically rank
 *  deficient A returns CAPITAL_ERR_NOT_SPD (the sweep after the shifted one breaks down).  Other num_iter: CAPITAL_ERR_INVALID.
 *  1D (c == 1, d == size): invoke_1d :172-193, sweep_1d :5-29, Gram allreduce policy.h:78-85.  A_local: (m/d) x n rect, Q_local same
 *    shape; R_local: n x n packed upper (or rect), replicated on every rank.
 *  3D (c == d) and tunable (1 < c < d, c | d, at most 16 ranks; sweep_tune :122-170): A_local and Q_local (m/d) x (n/c);
 *    R_local: the (n/c) x (n/c) cyclic block of R on the rank's square grid -- the whole grid for c == d, its cube of c^3
 *    consecutive ranks on the tunable grid (square coordinates (x, y mod c, z)) -- packed upper, with zeros on the local diagonal
 *    where that y > x; replicated on the c layers and, on the tunable grid, in every cube.  complete_inv = 0 applies the complete
 *    inverse instead of the reference's block `solve` (:44-73): the same Q.  Other grids: CAPITAL_ERR_UNSUPPORTED. */
capital_status_t capital_cacqr_factor_f64(capital_ctx* ctx, const double* A_local, int64_t m_global, int64_t n_global,
                                          int num_iter, const capital_cholinv_args_t* ci_args,
                                          capital_structure_t r_structure, double* Q_local, double* R_local);
/* qr::validate<Alg>::residual / orthogonality -- test/qr/validate.hpp:7-52. */
capital_status_t capital_cacqr_residual_f64(capital_ctx* ctx, const double* A_local, int64_t m_global, int64_t n_global,
                                            const double* Q_local, capital_structure_t r_structure,
                                            const double* R_local, double* residual, double* orthogonality);
/* qr::cacqr apply_QT / apply_Q (cacqr.h:52,55) and least squares, from the outputs of capital_cacqr_factor_f64 on one GPU or the 1D
 * row grid (c == 1, d == size); other grids: CAPITAL_ERR_UNSUPPORTED.  Collective on the grid: every rank calls with the same
 * m_global, n_global, nrhs (and r_structure).  Q_local, R_local: exactly as the factor wrote them -- Q_local lr x n with
 * lr = ceil(m/d) and leading dimension lr; R_local packed upper or rect, replicated.  B_local / C_local: lr x nrhs, column-major,
 * ldb / ldc >= lr, holding the rows this rank's A_local holds (global row gy at local row gy / d on rank gy mod d).  Where d does
 * not divide m, the pad rows of Q are zero, so finite pad rows of B contribute nothing.  Y, Z, X: full n x nrhs, column-major,
 * ldy / ldz / ldx >= n.  Right-hand sides go in panels of 32; each product reads Q once per panel, in place.  Only the rows of an
 * output are written (rows n .. ldx, lr .. ldc stay untouched).  Host or device pointers.  Results are deterministic.  One GPU:
 * enqueued on the context stream, synchronous only for a host output.  Grid: apply_QT and lstsq are synchronous; their all-reduce
 * slots use the peer arena, so the next factor call re-clears the arena.  CAPITAL_ERR_INVALID: a NULL pointer, nrhs < 1, m < n, a
 * leading dimension too small or a bad structure. */
/* Y = Q^T B.  Y: full n x nrhs, replicated, bit-identical on every rank. */
capital_status_t capital_cacqr_apply_qt_f64(capital_ctx* ctx, int64_t m_global, int64_t n_global, const double* Q_local,
                                            int64_t nrhs, const double* B_local, int64_t ldb, double* Y, int64_t ldy);
/* C_local = Q_local Z.  Z: full n x nrhs, the same on every rank.  No communication. */
capital_status_t capital_cacqr_apply_q_f64(capital_ctx* ctx, int64_t m_global, int64_t n_global, const double* Q_local,
                                           int64_t nrhs, const double* Z, int64_t ldz, double* C_local, int64_t ldc);
/* X = argmin ||A X - B||_F = R^-1 (Q^T B): apply_QT, then triangular substitution with R (blocked, R read in place, entries below
 * the diagonal never read).  X: full n x nrhs, replicated, bit-identical on every rank. */
capital_status_t capital_cacqr_lstsq_f64(capital_ctx* ctx, int64_t m_global, int64_t n_global, const double* Q_local,
                                         capital_structure_t r_structure, const double* R_local, int64_t nrhs,
                                         const double* B_local, int64_t ldb, double* X, int64_t ldx);

/* Batched CholeskyQR on this context's GPU: `batch` independent m x n matrices (1 <= n <= 512, m >= n), each factored A_b = Q_b R_b in
 * a few launches for the whole batch.  num_iter as in cacqr::factor: 1 = CholeskyQR, 2 = CholeskyQR2, 3 = shifted CholeskyQR3.
 * A, Q: batch x m x n, column-major, matrix b at offset b m n; R: batch x n x n, written whole (upper triangular, exact zeros below
 * the diagonal).  info[b] = 0 on success, else the 1-based pivot of the first sweep whose Gram matrix was not positive definite (that
 * sweep continues with 1 in its place; Q_b and R_b are then unspecified, and the other matrices are unaffected).  Where the single
 * path's base case is one kernel (n <= 64 or n a multiple of 64), Q_b and R_b have the bits of capital_cacqr_factor_f64 on A_b alone
 * on one GPU.  Device pointers only; Q must not overlap A.  Enqueued on the context stream without a host synchronisation; never
 * communicates, so on a grid context each rank factors its own batch.  Intermediates take at most 2 GiB of device memory (more only
 * when one matrix needs more): larger batches run in chunks.  n > 512: CAPITAL_ERR_UNSUPPORTED; m < n, n < 1, batch < 1, num_iter not
 * 1, 2 or 3, a NULL argument or a host pointer: CAPITAL_ERR_INVALID. */
capital_status_t capital_cacqr_factor_batched_f64(capital_ctx* ctx, int64_t m, int64_t n, int64_t batch, int num_iter, const double* A,
                                                  double* Q, double* R, int* info);
/* X_b = R_b^-1 (Q_b^T B_b) = argmin ||A_b X_b - B_b||_F from the outputs of capital_cacqr_factor_batched_f64.  B: batch x m x nrhs,
 * X: batch x n x nrhs, column-major, matrix b at offsets b m nrhs and b n nrhs.  Each X_b has the bits of capital_cacqr_lstsq_f64 on
 * Q_b, R_b (rect) and B_b.  Device pointers only; X must not overlap B.  Enqueued on the context stream; deterministic.  Errors as
 * the factor (nrhs < 1: CAPITAL_ERR_INVALID). */
capital_status_t capital_cacqr_lstsq_batched_f64(capital_ctx* ctx, int64_t m, int64_t n, int64_t batch, const double* Q, const double* R,
                                                 int64_t nrhs, const double* B, double* X);

/* ---- SUMMA ------------------------------------------------------------------------------------ */
/* matmult::summa::invoke(A, B, C, topo, gemm{Trans, NoTrans, alpha, beta}) -- summa.hpp:6-44 in the T*N form the validators
 * and syrk_internal use (test/cholesky/validate.hpp:35, summa.hpp:143-145):  C = alpha * A^T B + beta * C  with A (k x m),
 * B (k x n), C (m x n) all element-cyclic over the d x d face (local blocks k/d x m/d, k/d x n/d, m/d x n/d, column-major,
 * replicated over the c layers; d must divide m, n, k).  Host or device pointers. */
capital_status_t capital_summa_gemm_tn_f64(capital_ctx* ctx, int64_t m_global, int64_t n_global, int64_t k_global, double alpha,
                                           const double* A_local, const double* B_local, double beta, double* C_local);

/* ---- leaf-engine seam (the reference's designated swap point, blas/engine.h:7-8) ------------- */
/* blas::engine::_gemm (blas/interface.hpp:43-59) restricted to the T*N form the hot path executes
 * (summa.hpp:143-145): C[m x n] = alpha * A^T B + beta * C, A is k x m, B is k x n, all column-major
 * DEVICE pointers.  `flags` = OR of CAPITAL_GEMM_* below (structure hints that skip zero tiles). */
enum {
  CAPITAL_GEMM_A_UPPER = 1,  /* A[k,i] == 0 for k > i   (trmm Left/Upper/Trans, summa.hpp:64) */
  CAPITAL_GEMM_A_LOWER = 2,  /* A[k,i] == 0 for k < i */
  CAPITAL_GEMM_B_UPPER = 4,  /* B[k,j] == 0 for k > j */
  CAPITAL_GEMM_B_LOWER = 8,  /* B[k,j] == 0 for k < j */
  CAPITAL_GEMM_C_UPPER = 16  /* only tiles touching i <= j are computed/stored (syrk 'U') */
};
capital_status_t capital_blas_gemm_tn_f64(capital_ctx* ctx, int64_t m, int64_t n, int64_t k, double alpha,
                                          const double* A, int64_t lda, const double* B, int64_t ldb,
                                          double beta, double* C, int64_t ldc, int flags);
/* EXPERIMENTAL, OFF BY DEFAULT -- BASELINE config 5 ("FP32/TF32 Cholesky, mixed-precision trailing update with FP64 panel").
 * The reference has no float BLAS path (src/blas/interface.hpp:43-97 is double only): this is an extension of the blas::engine seam,
 * not a replacement of a reference entry point.  capital_blas_gemm_tn_tf32: the product of capital_blas_gemm_tn_f64 (FP64 operands
 * and result, only the CAPITAL_GEMM_C_UPPER flag) computed on the TF32 tensor cores (wgmma.mma_async .tf32, FP32 accumulators in registers);
 * passes = 1: operands rounded to TF32 (relative error ~ 5e-4 per product), passes = 3: operands split hi + lo (FP32-class).
 * capital_set_trailing_precision(ctx, 0 | 1 | 3): cholinv::factor runs its trailing updates A22 -= R12^T R12 (cholinv.hpp:131-134,
 * summa::syrk) in that mode; base cases, R12, the inverse and every other product stay FP64.  Single GPU and c = 1 grids.
 * capital_tf32_stats: launches / flops of the TF32 kernel since capital_create. */
capital_status_t capital_blas_gemm_tn_tf32(capital_ctx* ctx, int64_t m, int64_t n, int64_t k, double alpha, const double* A, int64_t lda,
                                           const double* B, int64_t ldb, double beta, double* C, int64_t ldc, int flags, int passes);
capital_status_t capital_set_trailing_precision(capital_ctx* ctx, int mode);
capital_status_t capital_tf32_stats(const capital_ctx* ctx, int64_t* launches, double* flops);

/* lapack::engine::_potrf('U') + _trtri('U','N') fused (lapack/interface.hpp:30-58; called back to
 * back at cholinv/policy.h:199-201): A (n x n, upper read) -> R, Rinv upper (lower zeroed). DEVICE pointers. */
capital_status_t capital_lapack_potrf_trtri_f64(capital_ctx* ctx, int64_t n, const double* A, int64_t lda,
                                                double* R, int64_t ldr, double* Rinv, int64_t ldri);

#if defined(__GNUC__)
#pragma GCC visibility pop
#endif
#ifdef __cplusplus
}
#endif
#endif /* CAPITAL_B200_H */
