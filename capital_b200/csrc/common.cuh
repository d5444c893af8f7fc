// capital_b200 -- shared declarations for the CUDA translation units (sm_90a only).
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <string>
#include <vector>
#include <map>
#include "../../include/capital_b200.h"

#define CAP_CUDA(call)                                                                                    \
  do {                                                                                                     \
    cudaError_t e__ = (call);                                                                              \
    if (e__ != cudaSuccess) {                                                                              \
      ctx->set_error(std::string(#call) + ": " + cudaGetErrorString(e__) + " (" + __FILE__ + ":" +         \
                     std::to_string(__LINE__) + ")");                                                      \
      return CAPITAL_ERR_CUDA;                                                                             \
    }                                                                                                      \
  } while (0)

#define CAP_TRY(call)                                  \
  do {                                                 \
    capital_status_t s__ = (call);                     \
    if (s__ != CAPITAL_OK) return s__;                 \
  } while (0)

typedef CUresult (*cuTensorMapEncodeTiled_fn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                              const cuuint64_t*, const cuuint32_t*, const cuuint32_t*,
                                              CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion,
                                              CUtensorMapFloatOOBfill);

struct DeviceBuf {
  void* p = nullptr;
  size_t bytes = 0;
};

struct capital_ctx {
  capital_grid_t grid{};
  int device = 0;
  int num_sms = 132;
  cudaStream_t stream = nullptr;   // main stream (caller's or owned)
  cudaStream_t side = nullptr;     // low-priority stream: deferred ("far") trailing updates, T^T products; lives in a green context
  void* green = nullptr;           // (CUgreenCtx) SM partition of the deferred stream, see make_green_side_stream (api.cu)
  cudaStream_t side_deep[2] = {nullptr, nullptr};  // deferred streams of recursion depths 1 and 2 (multi-GPU schedule; on one GPU they carry
                                                   // the bands and the T^T products, cholinv_local.cu), same partition, rising priority
  cudaStream_t hi = nullptr;       // high-priority stream: the critical chain of the recursion
  cudaStream_t copy_in = nullptr, copy_out = nullptr;  // H2D / D2H streams of the host-pointer path
  std::vector<cudaEvent_t> dep_pool;  // dependency events (timing disabled), recycled per factor call
  size_t dep_used = 0;
  std::vector<cudaEvent_t> io_pool;   // events of the host-pointer streaming path
  size_t io_used = 0;
  bool own_stream = false;
  cudaEvent_t ev_start = nullptr, ev_stop = nullptr, ev_fork = nullptr;
  cuTensorMapEncodeTiled_fn encode = nullptr;
  capital_counters_t counters{};
  std::string err;
  int* d_info = nullptr;           // device flag: first non-SPD pivot (0 = ok)
  double* d_scalars = nullptr;     // device scratch for reductions (16 doubles)
  std::map<std::string, DeviceBuf> pool;  // named, grow-only workspace (the reference's `info` tables, cholinv.h:35-40)
  // multi-GPU: peer layer (peer.cuh) -- IPC-mapped arenas and flags; NCCL (dlopen'ed) only bootstraps the handle exchange
  void* comm_world = nullptr;          // ncclComm_t, when capital_comm_init was used
  void* peer = nullptr;                // Peer*
  std::vector<cudaEvent_t> comm_pool;  // dependency events of the distributed schedules, recycled per call
  size_t comm_used = 0;
  std::string arena_signature;         // which layout the peer arena currently holds (a new layout starts from zeros)

  // per-launch timing of the dominant kernel (gemm_tn 128x128), off by default
  struct ProfRec { cudaEvent_t e0, e1; double flops; };
  bool profiling = false;
  int64_t far_min = 2048;   // trailing updates at least this large are split into near (critical) / far (deferred)   [env CAPITAL_FAR_MIN]
  int64_t side_min = 1024;  // nodes whose left part is at least this large defer T^T to the low-priority stream      [env CAPITAL_SIDE_MIN]
  int64_t band_min = 4096;  // nodes whose left part is at least this large issue the leading bands of R12 / Rinv12 early [env CAPITAL_BAND_MIN]
  bool no_overlap = false;  // debug / measurement: run the recursion on one stream
  bool poison_workspace = false;  // debug / tests: fill every (re)allocated workspace with 0xFF bytes (NaN)  [env CAPITAL_POISON_WORKSPACE=1]
  // EXPERIMENTAL, off by default (capital_set_trailing_precision): trailing updates A22 -= R12^T R12 on the TF32 tensor cores
  // (gemm_tf32.cu); 0 = FP64 DMMA, 1 = TF32, 3 = 3 x TF32 with split operands.  Products with k below tf32_min_k stay FP64.
  int trailing_mode = 0;
  bool tf32_ready = false;  // the TF32 kernel's attributes are set at its first use, never by the default FP64 path
  int64_t tf32_min_k = 256;
  int64_t tf32_launches = 0;
  double tf32_flops = 0.0;
  std::vector<cudaEvent_t> prof_pool;
  size_t prof_used = 0;
  std::vector<ProfRec> prof_recs;
  capital_status_t prof_event(cudaEvent_t* out) {
    if (prof_used == prof_pool.size()) {
      cudaEvent_t e;
      if (cudaEventCreate(&e) != cudaSuccess) { err = "cudaEventCreate failed"; return CAPITAL_ERR_CUDA; }
      prof_pool.push_back(e);
    }
    *out = prof_pool[prof_used++];
    return CAPITAL_OK;
  }

  // timeline (debug / profiling): CUDA events around every launch of the schedule, read back by capital_timeline_end
  struct TlRec { cudaEvent_t e0, e1; int sid, kind; double a, b, c; };
  bool timeline = false;
  std::vector<TlRec> tl;
  std::vector<cudaEvent_t> tl_pool;
  size_t tl_used = 0;
  int stream_id(cudaStream_t st) const;  // 0 caller, 1 chain, 2-4 deferred (depth 0-2), 5-9 push streams, 10 copy-in, 11 copy-out
  int tl_begin(cudaStream_t st, int kind, double a = 0, double b = 0, double c = 0);
  void tl_end(cudaStream_t st, int idx);

  void set_error(const std::string& s) { err = s; }
  capital_status_t workspace(const std::string& name, size_t bytes, void** out);
};

// ---- gemm_tn.cu -------------------------------------------------------------------------------
capital_status_t gemm_tn_init(capital_ctx* ctx);  // per-device kernel attributes
capital_status_t leaf_init(capital_ctx* ctx);
capital_status_t gemm_probe_dmma(capital_ctx* ctx, double* tflops, double* ms);

// Multi-GPU form of the product (dist.cu).  (1) The contraction may run over several operand CLASSES -- the k-slices owned by
// different process rows (summa.hpp:185-193), resident in local mirrors -- inside one launch, accumulators staying in
// registers.  (2) The first half of the reference's depth reduction (MPI_Allreduce over the c layers, summa.hpp:236) is fused
// into the epilogue over peer-mapped memory: every stored value also goes, over NVLink, into buffers of the other layers.
//   mode 1 (k split over layers, c == d): C is this layer's PARTIAL-product buffer and Cpeer[i] the receive buffer that the i-th
//          other layer keeps for this layer: when the kernel has retired on every layer (one flag handshake), each layer holds all
//          c partials and adds them up in layer order with one streaming pass (dist.cu: reduce_partials) -- identical bits in
//          every replica, no collective call, no in-kernel waiting.
//   mode 2 (n split, d == 1): layer tn mod c computes tile column tn with the full k range and stores the FINAL values into its own
//          C and into the C replica of every other layer (Cpeer[i]).
constexpr int GEMM_NCLS_MAX = 2;
constexpr int GEMM_XPEERS_MAX = 3;
struct GemmXDev {
  int mode, c, z;
  double* Cpeer[GEMM_XPEERS_MAX];  // same window as C inside the i-th OTHER layer's buffer
};
struct GemmOperands {
  int ncls = 1;
  const double* A[GEMM_NCLS_MAX] = {nullptr, nullptr};
  const double* B[GEMM_NCLS_MAX] = {nullptr, nullptr};
  int64_t lda = 0, ldb = 0;
};
capital_status_t gemm_tn_x(capital_ctx* ctx, cudaStream_t st, int64_t m, int64_t n, int64_t k, double alpha, const GemmOperands& ops,
                           double beta, double* C, int64_t ldc, int flags, int noff, const GemmXDev* x, int moff = 0);
capital_status_t gemm_tn(capital_ctx* ctx, cudaStream_t st, int64_t m, int64_t n, int64_t k, double alpha, const double* A,
                         int64_t lda, const double* B, int64_t ldb, double beta, double* C, int64_t ldc, int flags);

capital_status_t gemm_tn_off(capital_ctx* ctx, cudaStream_t st, int64_t m, int64_t n, int64_t k, double alpha, const double* A,
                             int64_t lda, const double* B, int64_t ldb, double beta, double* C, int64_t ldc, int flags, int noff, int moff = 0);
capital_status_t gemm_tn_splitk(capital_ctx* ctx, cudaStream_t st, int64_t m, int64_t n, int64_t k, double alpha, const double* A,
                                int64_t lda, const double* B, int64_t ldb, double* C, int64_t ldc, int flags);
capital_status_t gemm_tn_t(capital_ctx* ctx, cudaStream_t st, int64_t m, int64_t n, int64_t k, double alpha, const double* A, int64_t lda,
                           const double* B, int64_t ldb, double* C, int64_t ldc, double* Ct, int64_t ldct, int flags);
// split-k chunk count of gemm_tn_splitk for this shape (and whether it runs 128 x 128 tiles)
int64_t gemm_splitk_chunks(const capital_ctx* ctx, int64_t m, int64_t n, int64_t k, int flags, bool* big);
// A batch of products of one shape: matrix b reads A + b sa and B + b sb (16-byte aligned bases, even lda, ldb, sa, sb) and writes
// C + b sc, Ct + b sct (gemm_tn_batched, gemm_tn.cu).  ncls = 2 adds a second operand class (A1, B1: the same lda, ldb, sa, sb),
// summed after class 0 in the same launch as gemm_tn_x does; beta != 0 adds beta C_b (read at C + b sc).
struct GemmBatchOps {
  int64_t batch = 1;
  const double* A = nullptr;
  int64_t lda = 0, sa = 0;
  const double* B = nullptr;
  int64_t ldb = 0, sb = 0;
  int64_t sc = 0, sct = 0;
  int ncls = 1;
  const double* A1 = nullptr;
  const double* B1 = nullptr;
  double beta = 0.0;
};
capital_status_t gemm_tn_batched(capital_ctx* ctx, cudaStream_t st, int64_t m, int64_t n, int64_t k, double alpha, const GemmBatchOps& b,
                                 double* C, int64_t ldc, double* Ct, int64_t ldct, int flags, bool gram);

// ---- gemm_tf32.cu (experimental mixed-precision trailing update, BASELINE config 5) ----------------------------
capital_status_t gemm_tf32_init(capital_ctx* ctx);
capital_status_t gemm_tn_tf32(capital_ctx* ctx, cudaStream_t st, int64_t m, int64_t n, int64_t k, double alpha, const double* A, int64_t lda,
                              const double* B, int64_t ldb, double beta, double* C, int64_t ldc, int flags, int passes);
capital_status_t gemm_tn_tf32_x(capital_ctx* ctx, cudaStream_t st, int64_t m, int64_t n, int64_t k, double alpha, const GemmOperands& ops,
                                double beta, double* C, int64_t ldc, int flags, int noff, int passes);
// the trailing update of one node: FP64 DMMA by default, TF32 when the context asks for it and the contraction is long enough
static inline bool trailing_uses_tf32(const capital_ctx* ctx, int64_t k) { return ctx->trailing_mode != 0 && k >= ctx->tf32_min_k; }

// ---- layout.cu --------------------------------------------------------------------------------
capital_status_t transpose_block(capital_ctx* ctx, cudaStream_t st, int64_t rows, int64_t cols, const double* src,
                                 int64_t lds, double* dst, int64_t ldd, double scale);
capital_status_t copy_block(capital_ctx* ctx, cudaStream_t st, int64_t rows, int64_t cols, const double* src, int64_t lds,
                            double* dst, int64_t ldd);
capital_status_t zero_block(capital_ctx* ctx, cudaStream_t st, int64_t rows, int64_t cols, double* dst, int64_t ldd);
capital_status_t zero_band(capital_ctx* ctx, cudaStream_t st, int64_t n, double* a, int64_t ld);
// columns [col_begin, col_end) of the upper triangle of src into the packed triangle; with skip_top > 0, rows [0, skip_top) of the
// columns from skip_top on are neither read nor written (the top-level block of Rinv that complete_inv = 0 skips: zero_packed_top)
capital_status_t pack_upper(capital_ctx* ctx, cudaStream_t st, int64_t n, const double* src, int64_t lds, double* packed,
                            int zero_diag, int64_t col_begin = 0, int64_t col_end = -1, int64_t skip_top = 0);
// zeros into rows [0, top) of the packed columns [top, n)
capital_status_t zero_packed_top(capital_ctx* ctx, cudaStream_t st, int64_t n, double* packed, int64_t top);
capital_status_t unpack_upper(capital_ctx* ctx, cudaStream_t st, int64_t n, const double* packed, double* dst, int64_t ldd);
capital_status_t triu_copy(capital_ctx* ctx, cudaStream_t st, int64_t n, const double* src, int64_t lds, double* dst,
                           int64_t ldd, int zero_diag);
// n x n local block of a symmetric matrix from its computed upper half U: out = U on and above the global diagonal (local (r, c) is
// global (y + d r, x + d c)), below it the mirror S, read transposed (s_trans: S(c, r), on one GPU S = U) or as it is
capital_status_t sym_merge(capital_ctx* ctx, cudaStream_t st, int64_t n, const double* U, int64_t ldu, const double* S, int64_t lds,
                           bool s_trans, double* out, int64_t ldo, int x, int y, int d);
// n x n local block of U^T, U = triu(A) with its diagonal halved (sygst's A = U + U^T): the global lower triangle of the symmetric A
// (local (r, c) is global (y + d r, x + d c)) with its diagonal times 1/2, zeros above it.  The global upper triangle is never read.
capital_status_t tril_half_copy(capital_ctx* ctx, cudaStream_t st, int64_t n, const double* src, int64_t lds, double* dst, int64_t ldd,
                                int x, int y, int d);
// Batched factor (n <= BASECASE_MAX): W_b, nb x nb (nb a multiple of 32), from the upper triangle of A_b (n x n contiguous, mirrored below
// the diagonal; the lower triangle is never read), the identity in the pad; and back: dst_b (ld ldd, stride sd) = triu of the leading
// n x n block of src_b (ld lds, stride ss), exact zeros below the diagonal.
capital_status_t sym_pad_batched(capital_ctx* ctx, cudaStream_t st, int64_t n, int64_t nb, int64_t batch, const double* A, double* W);
capital_status_t triu_out_batched(capital_ctx* ctx, cudaStream_t st, int64_t n, int64_t batch, const double* src, int64_t lds, int64_t ss,
                                  double* dst, int64_t ldd, int64_t sd);
// Batched inverse / sygst (matrix b at src + b ss, dst + b sd, <= 65535 matrices): tril_half_copy's operand U_b^T (diagonal halved,
// zeros above), read from A_b's UPPER triangle; sym_merge on one GPU (out_b from the upper triangle of U_b and its mirror; <= 65535 matrices); and a plain copy
// of rows x cols blocks (the right-hand-side panels of the batched products).
capital_status_t tril_half_batched(capital_ctx* ctx, cudaStream_t st, int64_t n, int64_t batch, const double* src, int64_t lds, int64_t ss,
                                   double* dst, int64_t ldd, int64_t sd);
capital_status_t sym_merge_batched(capital_ctx* ctx, cudaStream_t st, int64_t n, int64_t batch, const double* U, int64_t ldu, int64_t su,
                                   double* out, int64_t ldo, int64_t so);
capital_status_t copy_batched(capital_ctx* ctx, cudaStream_t st, int64_t rows, int64_t cols, int64_t batch, const double* src, int64_t lds,
                              int64_t ss, double* dst, int64_t ldd, int64_t sd);
capital_status_t gen_symmetric(capital_ctx* ctx, cudaStream_t st, double* A, int64_t ld, int64_t lrows, int64_t lcols,
                               int64_t n_global, int x, int y, int d, int diag_dom);
capital_status_t gen_random(capital_ctx* ctx, cudaStream_t st, double* A, int64_t ld, int64_t lrows, int64_t lcols,
                            int64_t pad_rows, int64_t pad_cols, int64_t key);
// sum of squares over the (global-)upper part (or everything) of a local block; accumulates into out[0]
capital_status_t sumsq_block(capital_ctx* ctx, cudaStream_t st, int64_t rows, int64_t cols, const double* a, int64_t ld,
                             int upper_mode, int x, int y, int d, double* out);
capital_status_t sub_identity_local(capital_ctx* ctx, cudaStream_t st, int64_t n, double* a, int64_t ld);
// Gram shift of shifted CholeskyQR3: G(i, i) += coef * trace, the trace summed in a fixed order by one CTA (no atomics), so that
// every holder of a bit-identical replica of G derives the same shift bits.  gram_shift: the trace of this n x n block.  On a grid
// the two halves run apart: gram_diag_partial stores the local diagonal's sum to *out, gram_shift_by adds coef * (parts[0] + ...
// + parts[nparts - 1]), summed in index order, to the local diagonal (parts may have been written by peer GPUs' copy engines).
capital_status_t gram_shift(capital_ctx* ctx, cudaStream_t st, int64_t n, double* G, int64_t ld, double coef);
capital_status_t gram_diag_partial(capital_ctx* ctx, cudaStream_t st, int64_t n, const double* G, int64_t ld, double* out);
capital_status_t gram_shift_by(capital_ctx* ctx, cudaStream_t st, int64_t n, double* G, int64_t ld, const double* parts, int nparts,
                               double coef);
// Batches (<= 65535 matrices, matrix b at src + b ss, dst + b sd): gram_shift with one CTA per matrix, in gram_shift's summation order;
// and transpose_block (scale 1) of every matrix.
capital_status_t gram_shift_batched(capital_ctx* ctx, cudaStream_t st, int64_t n, int64_t batch, double* G, int64_t ld, int64_t sg,
                                    double coef);
capital_status_t transpose_batched(capital_ctx* ctx, cudaStream_t st, int64_t rows, int64_t cols, int64_t batch, const double* src,
                                   int64_t lds, int64_t ss, double* dst, int64_t ldd, int64_t sd);

// ---- leaf.cu ----------------------------------------------------------------------------------
// potrf('U') + trtri('U','N') of one nb x nb block (nb <= LEAF_MAX) in shared memory.
constexpr int LEAF_MAX = 64;
constexpr int BASECASE_MAX = 512;  // largest block handled by the one-launch cluster kernel (multiple of 64)
// A batch of independent blocks in one launch: matrix b at W + b s.w, R + b s.r, ... with its own info[b], on clusters of cw CTAs
// (2, 4 or 8; the cluster kernel only).  Without one (nullptr): a single block, ctx->d_info, width 8.  A failing pivot k of the block
// is recorded as pivot_base + k + 1: the recursion passes the block's diagonal offset, so that info numbers the column of the whole matrix.
struct BatchStrides { long long w = 0, r = 0, ri = 0, rit = 0; };
struct LeafBatch {
  int64_t batch;  // leaf: <= INT32_MAX; cluster kernel: <= 65535 (grid y)
  BatchStrides s;
  int* info;
  int cw;
};
capital_status_t basecase_cholinv(capital_ctx* ctx, cudaStream_t st, int nb, double* W, int64_t ldw, double* R, int64_t ldr,
                                  double* Ri, int64_t ldri, double* RiT, int64_t ldrit, const LeafBatch* bt = nullptr,
                                  int pivot_base = 0);
capital_status_t leaf_cholinv(capital_ctx* ctx, cudaStream_t st, int nb, const double* W, int64_t ldw, double* R, int64_t ldr,
                              double* Ri, int64_t ldri, double* RiT, int64_t ldrit, const LeafBatch* bt = nullptr, int pivot_base = 0);
// Cluster width of the batched cluster kernel for nb = 64 T: no phase of the kernel has work for more CTAs than tiles of a block row,
// and an idle CTA still holds its SM's shared memory.  CAPITAL_BATCHED_CW=8 forces the single-matrix width (measurement).
static inline int batched_cluster_width(int64_t nb) {
  const char* e = getenv("CAPITAL_BATCHED_CW");
  if (e && atoi(e) == 8) return 8;
  const int64_t T = nb / 64;
  return T <= 2 ? 2 : T <= 4 ? 4 : 8;
}

// Device memory the batched calls hold for intermediates, whatever the batch: larger batches run in chunks.
constexpr size_t BATCHED_WORKSPACE_CAP = size_t(2) << 30;

// ---- syevj.cu ---------------------------------------------------------------------------------
// Batched symmetric eigensolver (capital_syevj_batched_f64), arguments already checked: n <= BASECASE_MAX, device pointers.
capital_status_t syevj_init(capital_ctx* ctx);  // per-device kernel attributes
// matrices per chunk: at most 65535, and for n > 64 as many as fit BATCHED_WORKSPACE_CAP
int64_t syevj_chunk(int64_t n, int64_t batch);
capital_status_t syevj_batched(capital_ctx* ctx, cudaStream_t st, int64_t n, int64_t batch, const double* A, double* w, double* V,
                               int* info);

// ---- cholinv.cu -------------------------------------------------------------------------------
// local (single-GPU) recursive CholInv on dense n x n blocks; W is destroyed (Schur complements).
// Optional callbacks of the top-level call (cholinv::factor on one GPU): `need_cols` makes the chain's stream `st` wait until
// columns [0, col_end) of W have arrived; `left_done` fires after each left child on the right spine (depth <= 3), when columns
// [0, col_end) of R are final, and those of Rinv too at depth 0.
struct CholinvHooks {
  void* user;
  capital_status_t (*need_cols)(void* user, cudaStream_t st, int64_t col_end);
  capital_status_t (*left_done)(void* user, cudaStream_t st, int64_t col_end, int depth);
  // optional.  `wait_cols`: as need_cols, for a stream other than the chain (the leading band of an R12 product).
  // `cols_waited` (host input): how many leading columns the chain already waited for -- while it is short of a
  // node's extent, the node's R12 product is issued in column chunks, each behind the arrival of its own columns only.
  // `right_done`: the top-level right child has returned, all of R is final.  `inv_cols`: the top-level inverse block is issued in
  // column chunks; columns [0, col_end) of Rinv are final.
  int64_t (*cols_waited)(void* user);
  capital_status_t (*right_done)(void* user, cudaStream_t st);
  capital_status_t (*inv_cols)(void* user, cudaStream_t st, int64_t col_end);
  capital_status_t (*wait_cols)(void* user, cudaStream_t st, int64_t col_end);
  // `r_final`: the last base case (bottom of the right spine) has been issued on `st`, all of R is final after it.
  capital_status_t (*r_final)(void* user, cudaStream_t st);
};
// allow_side = false keeps everything on `st` (the distributed base case runs on the critical chain and must not queue behind
// the deferred stream's GEMMs).
capital_status_t cholinv_local(capital_ctx* ctx, cudaStream_t st, int64_t n, double* W, int64_t ldw, double* R, int64_t ldr,
                               double* Ri, int64_t ldri, double* RiT, int64_t ldrit, bool complete_top, int64_t bc, int split,
                               const CholinvHooks* hooks = nullptr, bool allow_side = true);

// ---- solve.cu ---------------------------------------------------------------------------------
// C = beta Cin + alpha op(U[r0:r1, c0:c1]) P for one panel of nrhs <= SOLVE_W right-hand sides (op = T when `trans`).  U: upper
// triangular, packed (ldu == 0, column i at i(i+1)/2) or rect (ld ldu); entries below the diagonal are never read.  Panel rows are
// addressed by the factor index: P(k, w) at P[k pinc + w ldp], C(o, w) at C[o cinc + w ldc], Cin(o, w) at Cin[o cinc + w ldcin]
// (Cin may be null, or C itself).  pinc / cinc > 1 gather / scatter the cyclic rows of a grid rank from a full-length vector.
constexpr int SOLVE_W = 32;
struct TriApply {
  const double* U;
  int64_t ldu;
  bool trans;
  int64_t r0, r1, c0, c1;
  int64_t nrhs;
  double alpha;
  const double* P;
  int64_t pinc, ldp;
  double beta;
  const double* Cin;
  int64_t ldcin;
  double* C;
  int64_t cinc, ldc;
  bool full = false;  // a rect window read whole (no j <= i mask, no triangular k ranges): Q^T P and Q P for a tall rect Q (ldu > 0)
  // a batch of independent problems (<= 65535, grid z): matrix b reads U + b su, P + b sp, Cin + b scin and writes C + b sc
  int64_t batch = 1, su = 0, sp = 0, scin = 0, sc = 0;
};
capital_status_t tri_apply(capital_ctx* ctx, cudaStream_t st, const TriApply& a);
// Y <- U[0:n, 0:n]^-1 Y in place for one panel of nrhs <= SOLVE_W right-hand sides (Y(k, w) at Y[k + w ldy]); U upper triangular,
// packed (ldu == 0) or rect, entries below the diagonal never read.  Deterministic.
capital_status_t tri_solve(capital_ctx* ctx, cudaStream_t st, const double* U, int64_t ldu, int64_t n, int64_t nrhs, double* Y,
                           int64_t ldy);
// tri_solve on a batch of <= 65535 independent problems: U + b su (rect), Y + b sy; each gets tri_solve's bits
capital_status_t tri_solve_batched(capital_ctx* ctx, cudaStream_t st, const double* U, int64_t ldu, int64_t su, int64_t n, int64_t nrhs,
                                   double* Y, int64_t ldy, int64_t sy, int64_t batch);
// Out = S + Cin (Cin may be null) on a rows x w column-major panel
capital_status_t panel_add(capital_ctx* ctx, cudaStream_t st, int64_t rows, int64_t w, const double* S, int64_t lds, const double* Cin,
                           int64_t ldcin, double* Out, int64_t ldo);

static inline int64_t round_up(int64_t a, int64_t b) { return (a + b - 1) / b * b; }
// Does cholinv::invoke split a node of (global = local, single GPU) size n, or is it the reference's base case (potrf + trtri of the
// whole block, cholinv.hpp:93)?  Decides whether complete_inv == 0 skips an inverse block at all: a top-level base case always
// returns the full inverse.
static inline bool cholinv_node_splits(int64_t n, int64_t bc, int split) { return n > bc && (n >> split) >= split && (n >> split) > 0; }
static inline int64_t ceil_div(int64_t a, int64_t b) { return (a + b - 1) / b; }
