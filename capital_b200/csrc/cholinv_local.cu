// Single-device recursive CholInv on a dense block (the schedule of cholinv::invoke, cholinv.hpp:87-165, with
// every product expressed as C = alpha A^T B + beta C so that one DMMA kernel serves all four of them).
//
// Buffers (all column-major, same leading dimension allowed):
//   W   : in  -- SPD block, upper triangle read; destroyed (Schur complements; the dead lower-left blocks are
//               reused as the scratch for T^T, which replaces the reference's rect_table temporaries, cholinv.h:37-38)
//   R   : out -- upper factor, A = R^T R
//   Ri  : out -- R^{-1} (upper);   RiT : out -- (R^{-1})^T (lower), kept so that "Left/Upper/NoTrans" and
//               "Right/Upper/NoTrans" trmm (cholinv.hpp:150-154) are both A^T B products with K-contiguous operands.
// Ri and RiT must be zero on entry (the triangular products read whole diagonal tiles).
//
// Two streams.  The reference's recursion is strictly sequential; here the chain that the next diagonal block
// depends on (base cases, R12, and the part of the trailing update the right child's left subtree reads -- "near")
// runs on a high-priority stream, while work nobody waits for yet (the rest of the trailing update -- "far" -- and
// T^T of the inverse combine) is queued on low-priority streams and joined by events exactly where it is consumed.
// The latency-bound bottom of the recursion then overlaps with DMMA-bound work instead of idling 140 SMs.  Deferred work that is
// wanted sooner must not queue behind work that is wanted later, so the deferred streams are split by when their work is needed:
// the top-level node's far update (~10 ms, needed by the right half's R12) on the lowest-priority stream, the far updates of every
// other node (needed within a subtree) on a higher-priority one, and the T^T products (needed as soon as a right child returns)
// on the highest.
//
// Bands.  Two products of a node wait on the chain for a whole child although their leading part depends on half of it only:
// rows [0, r) of R12 = Rinv11^T A12 read Rinv11[0:r, 0:r], the inverse of the left child's own left child, and columns [0, c) of
// Rinv12 = -(T^T)^T Rinv22 read Rinv22[0:c, 0:c], that of the right child's left child.  These leading bands are issued from inside
// the child, on a deferred stream of their own, as soon as that grandchild has returned; they then run beside the base cases of
// the child's right half, and the chain issues only the rest of the product (same tiles, same k ranges: identical results).
#include "common.cuh"

namespace {

int64_t split_point(int64_t n) {
  // halves (split = 1), rounded so that leaves stay LEAF_MAX-aligned
  int64_t s1 = n >> 1;
  if (n > 2 * LEAF_MAX) s1 = round_up(s1, LEAF_MAX);
  else s1 = round_up(s1, 2);  // even split points keep every window 16-byte aligned for TMA
  if (s1 >= n) s1 = n >> 1;
  return s1;
}

constexpr int64_t IN_CHUNK = 2048;  // columns per launch of an R12 product issued while A is still arriving from the host

struct Rec {
  capital_ctx* ctx;
  cudaStream_t M;     // critical chain
  cudaStream_t S, D;  // deferred far updates and bands of the top-level node / of every other node (nullptr: one stream)
  cudaStream_t T;     // T^T products
  bool bands;         // leading bands of R12 / Rinv12 are issued early
  double *W, *R, *Ri, *RiT;
  int64_t ldw, ldr, ldri, ldrit;
  int64_t bc;
  int split;
  const CholinvHooks* hooks;
  int64_t far_min;  // trailing updates smaller than this are not split
  int64_t band_min;   // nodes whose left part is smaller than this issue their products whole
  int64_t total;      // size of the top-level block
  bool base_aligned;  // all four buffers 16-byte aligned with even leading dimensions (cluster kernel uses 16-byte accesses)
  // A node's T^T reads the RiT of its left child only, so the RiT21 blocks of the right spine (o + n == total) are read by nobody
  // when the top node skips its Rinv12 (complete_inv = 0): they are not written then.
  bool spine_rit;
};

bool writes_rit21(const Rec& r, int64_t o, int64_t n) { return r.spine_rit || o + n != r.total; }

// Levels above the base case (n > bc) split by the reference's rule s1 = n >> split (cholinv.hpp:92,107); it fixes
// which Rinv block stays zero when complete_inv == 0.  Below it -- the reference's potrf/trtri base case
// (cholinv.hpp:93-104) -- the recursion continues with 64-aligned halves down to the cluster / leaf kernels.
// Returns 0 when the block is handled by a single kernel.
int64_t choose_split(const Rec& r, int64_t o, int64_t n, bool complete) {
  if (cholinv_node_splits(n, r.bc, r.split) && (n > LEAF_MAX || !complete)) return n >> r.split;
  if (n <= LEAF_MAX) return 0;
  if (n <= BASECASE_MAX && n % 64 == 0 && complete && r.base_aligned && (o & 1) == 0) return 0;
  return split_point(n);
}

capital_status_t new_event(capital_ctx* ctx, cudaEvent_t* e) {
  if (ctx->dep_used == ctx->dep_pool.size()) {
    cudaEvent_t ev;
    CAP_CUDA(cudaEventCreateWithFlags(&ev, cudaEventDisableTiming));
    ctx->dep_pool.push_back(ev);
  }
  *e = ctx->dep_pool[ctx->dep_used++];
  return CAPITAL_OK;
}

// The leading band of one of a node's products, handed to the child whose first half it depends on.
struct Band {
  bool r12;          // true: rows [0, edge) of R12 (left child); false: columns [0, edge) of Rinv12 and their rows of RiT21 (right child)
  int64_t o, s1, s2;  // the node
  cudaEvent_t wait;   // what the operands wait for besides the chain: the node's `pending` (R12) / its T^T (Rinv12), or nullptr
  cudaStream_t st;    // the node's deferred far-update stream
  int64_t edge = 0;   // set when issued
  cudaEvent_t done = nullptr;
};

// Issue band b on its stream behind everything the chain has issued so far; `split` is the split point of the child that
// issues it (its left child has just returned), rounded down to whole 128-wide tiles so that every tile keeps its k range.
capital_status_t issue_band(Rec& r, Band& b, int64_t split) {
  capital_ctx* ctx = r.ctx;
  const int64_t edge = split / 128 * 128;
  if (edge == 0) return CAPITAL_OK;
  cudaEvent_t e;
  CAP_TRY(new_event(ctx, &e));
  CAP_CUDA(cudaEventRecord(e, r.M));
  CAP_CUDA(cudaStreamWaitEvent(b.st, e, 0));
  if (b.wait) CAP_CUDA(cudaStreamWaitEvent(b.st, b.wait, 0));
  const int64_t o = b.o, s1 = b.s1, s2 = b.s2;
  const int64_t ldw = r.ldw, ldr = r.ldr, ldri = r.ldri, ldrit = r.ldrit;
  double* Ri = r.Ri + o * ldri + o;
  if (b.r12) {
    // R12[0:edge, :] = Rinv11[0:edge, 0:edge]^T A12[0:edge, :], once A12 has arrived
    if (r.hooks && r.hooks->wait_cols) CAP_TRY(r.hooks->wait_cols(r.hooks->user, b.st, o + s1 + s2));
    CAP_TRY(gemm_tn(ctx, b.st, edge, s2, edge, 1.0, Ri, ldri, r.W + (o + s1) * ldw + o, ldw, 0.0, r.R + (o + s1) * ldr + o, ldr,
                    CAPITAL_GEMM_A_UPPER));
  } else {
    // Rinv12[:, 0:edge] = -(T^T)^T Rinv22[0:edge, 0:edge]
    double* Ri12 = Ri + s1 * ldri;
    CAP_TRY(gemm_tn(ctx, b.st, s1, edge, edge, -1.0, r.W + o * ldw + o + s1, ldw, Ri12 + s1, ldri, 0.0, Ri12, ldri, CAPITAL_GEMM_B_UPPER));
    if (writes_rit21(r, o, s1 + s2)) CAP_TRY(transpose_block(ctx, b.st, s1, edge, Ri12, ldri, r.RiT + o * ldrit + o + s1, ldrit, 1.0));
  }
  CAP_TRY(new_event(ctx, &b.done));
  CAP_CUDA(cudaEventRecord(b.done, b.st));
  b.edge = edge;
  return CAPITAL_OK;
}

// o: offset of the node inside the buffers (diagonal position); pending / pending22: events the node's first use of A12 / A22 has to
// wait for (the two parts of the parent's deferred "far" update, recorded in this order on the deferred stream), or nullptr; up: the
// parent's band this node issues once its left child has returned, or nullptr.
capital_status_t rec(Rec& r, int64_t o, int64_t n, bool complete, cudaEvent_t pending, cudaEvent_t pending22, int depth, Band* up) {
  capital_ctx* ctx = r.ctx;
  double* W = r.W + o * r.ldw + o;
  double* R = r.R + o * r.ldr + o;
  double* Ri = r.Ri + o * r.ldri + o;
  double* RiT = r.RiT + o * r.ldrit + o;
  const int64_t ldw = r.ldw, ldr = r.ldr, ldri = r.ldri, ldrit = r.ldrit;
  const int64_t s1 = choose_split(r, o, n, complete);
  if (s1 == 0) {
    if (r.hooks && r.hooks->need_cols) CAP_TRY(r.hooks->need_cols(r.hooks->user, r.M, o + n));
    if (pending22) CAP_CUDA(cudaStreamWaitEvent(r.M, pending22, 0));
    // info numbers the pivot as a column of the whole matrix: the leaf adds this node's diagonal offset
    if (n <= LEAF_MAX) CAP_TRY(leaf_cholinv(ctx, r.M, (int)n, W, ldw, R, ldr, Ri, ldri, RiT, ldrit, nullptr, (int)o));
    else CAP_TRY(basecase_cholinv(ctx, r.M, (int)n, W, ldw, R, ldr, Ri, ldri, RiT, ldrit, nullptr, (int)o));
    if (o + n == r.total && r.hooks && r.hooks->r_final) CAP_TRY(r.hooks->r_final(r.hooks->user, r.M));
    return CAPITAL_OK;
  }
  const int64_t s2 = n - s1;
  double* W12 = W + s1 * ldw;
  double* W21 = W + s1;  // dead lower-left block: scratch for T^T (s2 x s1)
  double* W22 = W + s1 * ldw + s1;
  double* R12 = R + s1 * ldr;
  double* Ri12 = Ri + s1 * ldri;
  double* Ri22 = Ri + s1 * ldri + s1;
  double* RiT21 = RiT + s1;

  cudaStream_t F = depth == 0 ? r.S : r.D;  // this node's deferred far updates and bands
  const bool bands = r.bands && s1 >= r.band_min;
  Band b12{true, o, s1, s2, pending, F};
  CAP_TRY(rec(r, o, s1, true, nullptr, nullptr, depth + 1, bands ? &b12 : nullptr));
  if (up) CAP_TRY(issue_band(r, *up, s1));
  // right spine only (o + n == total size): everything left of column o + s1 is final for R
  if (depth <= 3 && o + n == r.total && r.hooks && r.hooks->left_done) CAP_TRY(r.hooks->left_done(r.hooks->user, r.M, o + s1, depth));
  // "trsm" via the inverse (cholinv.hpp:116-122): R12 = Rinv11^T A12
  const bool inflight = r.hooks && r.hooks->need_cols && r.hooks->cols_waited && r.hooks->cols_waited(r.hooks->user) < o + n;
  if (inflight && s2 >= 2 * IN_CHUNK) {
    // A is still arriving from the host (left spine of the recursion): issue the product by column chunks, each waiting for its own
    // columns only, so that the tensor pipe starts on A12 while the copy engine is still delivering its right part
    if (pending) CAP_CUDA(cudaStreamWaitEvent(r.M, pending, 0));
    for (int64_t c0 = 0; c0 < s2;) {
      const int64_t nc = (s2 - c0 < IN_CHUNK + IN_CHUNK / 2) ? s2 - c0 : IN_CHUNK;
      CAP_TRY(r.hooks->need_cols(r.hooks->user, r.M, o + s1 + c0 + nc));
      CAP_TRY(gemm_tn(ctx, r.M, s1, nc, s1, 1.0, Ri, ldri, W12 + c0 * ldw, ldw, 0.0, R12 + c0 * ldr, ldr, CAPITAL_GEMM_A_UPPER));
      c0 += nc;
    }
  } else {
    if (r.hooks && r.hooks->need_cols) CAP_TRY(r.hooks->need_cols(r.hooks->user, r.M, o + n));
    if (pending) CAP_CUDA(cudaStreamWaitEvent(r.M, pending, 0));  // the first part of the parent's deferred update covers W12
    // rows [0, e) are the band already issued from inside the left child
    const int64_t e = b12.edge;
    CAP_TRY(gemm_tn_off(ctx, r.M, s1 - e, s2, s1, 1.0, Ri + e * ldri, ldri, W12, ldw, 0.0, R12 + e, ldr, CAPITAL_GEMM_A_UPPER, 0, (int)e));
    if (b12.done) CAP_CUDA(cudaStreamWaitEvent(r.M, b12.done, 0));
  }
  // the trailing update accumulates into W22: the whole of the parent's deferred update has to be in
  if (pending22) CAP_CUDA(cudaStreamWaitEvent(r.M, pending22, 0));
  cudaEvent_t e_r12 = nullptr, e_tt = nullptr, e_far12 = nullptr, e_far = nullptr;
  const bool use_side = r.S != nullptr && s1 >= r.ctx->side_min;
  if (use_side) {
    CAP_TRY(new_event(ctx, &e_r12));
    CAP_CUDA(cudaEventRecord(e_r12, r.M));
    CAP_CUDA(cudaStreamWaitEvent(F, e_r12, 0));
    if (complete) CAP_CUDA(cudaStreamWaitEvent(r.T, e_r12, 0));
  }
  cudaStream_t tS = use_side ? r.T : r.M;
  // trailing update (cholinv.hpp:131-134): A22 -= R12^T R12, upper tiles only.
  // near = what the right child's left subtree reads (leading h x h block), far = everything else.
  const int64_t h = choose_split(r, o + s1, s2, true);
  // experimental mixed precision (BASELINE config 5): this product, and only this one, may run on the TF32 tensor cores
  const int tf = trailing_uses_tf32(ctx, s1) ? ctx->trailing_mode : 0;
  if (use_side && h > 0 && s2 >= r.far_min) {
    if (tf) {
      CAP_TRY(gemm_tn_tf32(ctx, r.M, h, h, s1, -1.0, R12, ldr, R12, ldr, 1.0, W22, ldw, CAPITAL_GEMM_C_UPPER, tf));
      CAP_TRY(gemm_tn_tf32(ctx, F, h, s2 - h, s1, -1.0, R12, ldr, R12 + h * ldr, ldr, 1.0, W22 + h * ldw, ldw, 0, tf));
      CAP_TRY(new_event(ctx, &e_far12));
      CAP_CUDA(cudaEventRecord(e_far12, F));
      CAP_TRY(gemm_tn_tf32(ctx, F, s2 - h, s2 - h, s1, -1.0, R12 + h * ldr, ldr, R12 + h * ldr, ldr, 1.0, W22 + h * ldw + h, ldw,
                           CAPITAL_GEMM_C_UPPER, tf));
    } else {
      CAP_TRY(gemm_tn(ctx, r.M, h, h, s1, -1.0, R12, ldr, R12, ldr, 1.0, W22, ldw, CAPITAL_GEMM_C_UPPER));
      CAP_TRY(gemm_tn(ctx, F, h, s2 - h, s1, -1.0, R12, ldr, R12 + h * ldr, ldr, 1.0, W22 + h * ldw, ldw, 0));
      CAP_TRY(new_event(ctx, &e_far12));  // the right child's R12 needs only this part
      CAP_CUDA(cudaEventRecord(e_far12, F));
      CAP_TRY(gemm_tn(ctx, F, s2 - h, s2 - h, s1, -1.0, R12 + h * ldr, ldr, R12 + h * ldr, ldr, 1.0, W22 + h * ldw + h, ldw,
                      CAPITAL_GEMM_C_UPPER));
    }
    CAP_TRY(new_event(ctx, &e_far));
    CAP_CUDA(cudaEventRecord(e_far, F));
  } else if (tf) {
    CAP_TRY(gemm_tn_tf32(ctx, r.M, s2, s2, s1, -1.0, R12, ldr, R12, ldr, 1.0, W22, ldw, CAPITAL_GEMM_C_UPPER, tf));
  } else {
    CAP_TRY(gemm_tn(ctx, r.M, s2, s2, s1, -1.0, R12, ldr, R12, ldr, 1.0, W22, ldw, CAPITAL_GEMM_C_UPPER));
  }
  if (complete) {
    // inverse combine, first half (cholinv.hpp:151): T^T = R12^T Rinv11^T  (B = RiT11, lower triangular) -- nobody needs
    // it before the right child is done, so it is deferred; on a stream of its own, since on the far updates' stream the T^T of a
    // small node would wait behind the far update of an ancestor that nobody needs for milliseconds.
    CAP_TRY(gemm_tn(ctx, tS, s2, s1, s1, 1.0, R12, ldr, RiT, ldrit, 0.0, W21, ldw, CAPITAL_GEMM_B_LOWER));
    if (use_side) {
      CAP_TRY(new_event(ctx, &e_tt));
      CAP_CUDA(cudaEventRecord(e_tt, r.T));
    }
  }
  const int64_t ct = s2 / 128;  // whole 128-column tiles of the block
  const bool inv_chunks = depth == 0 && r.hooks && r.hooks->inv_cols && ct >= 32;
  Band bi{false, o, s1, s2, e_tt, F};
  CAP_TRY(rec(r, o + s1, s2, true, e_far12, e_far, depth + 1, (bands && complete && !inv_chunks) ? &bi : nullptr));
  if (depth == 0 && r.hooks && r.hooks->right_done) CAP_TRY(r.hooks->right_done(r.hooks->user, r.M));
  if (complete) {
    if (e_tt) CAP_CUDA(cudaStreamWaitEvent(r.M, e_tt, 0));
    //   Rinv12 = -(T^T)^T Rinv22  (B = Ri22, upper triangular)   (cholinv.hpp:152-155)
    if (inv_chunks) {
      // last product of the factorization, and the host is waiting for its result: four column chunks (the k extent grows with the
      // column, so the leading half is cheap), each handed to the copy-out stream as soon as it is done; only the D2H of the last,
      // narrow chunk stays exposed.  Chunk edges are multiples of the 128-column tile: every tile computes exactly what it computes
      // in the single launch.
      const int64_t e3 = ct - ct * 3 / 32, e2 = e3 - ct * 5 / 32, e1 = e2 - ct / 4;
      const int64_t edge[5] = {0, e1 * 128, e2 * 128, e3 * 128, s2};
      for (int i = 0; i < 4; i++) {
        const int64_t c0 = edge[i], c1 = edge[i + 1];
        if (c1 <= c0) continue;
        CAP_TRY(gemm_tn_off(ctx, r.M, s1, c1 - c0, c1, -1.0, W21, ldw, Ri22 + c0 * ldri, ldri, 0.0, Ri12 + c0 * ldri, ldri,
                            CAPITAL_GEMM_B_UPPER, (int)c0));
        CAP_TRY(r.hooks->inv_cols(r.hooks->user, r.M, o + s1 + c1));
      }
    } else {
      // columns [0, c) are the band already issued from inside the right child
      const int64_t c = bi.edge;
      CAP_TRY(gemm_tn_off(ctx, r.M, s1, s2 - c, s2, -1.0, W21, ldw, Ri22 + c * ldri, ldri, 0.0, Ri12 + c * ldri, ldri, CAPITAL_GEMM_B_UPPER,
                          (int)c));
    }
    if (writes_rit21(r, o, n)) CAP_TRY(transpose_block(ctx, r.M, s1, s2 - bi.edge, Ri12 + bi.edge * ldri, ldri, RiT21 + bi.edge, ldrit, 1.0));
    if (bi.done) CAP_CUDA(cudaStreamWaitEvent(r.M, bi.done, 0));
  }
  return CAPITAL_OK;
}

}  // namespace

capital_status_t cholinv_local(capital_ctx* ctx, cudaStream_t st, int64_t n, double* W, int64_t ldw, double* R, int64_t ldr, double* Ri,
                               int64_t ldri, double* RiT, int64_t ldrit, bool complete_top, int64_t bc, int split,
                               const CholinvHooks* hooks, bool allow_side) {
  // `st` is the caller-visible stream; the recursion runs on the context's high-priority stream, fenced by events.
  cudaStream_t M = (ctx->hi && allow_side) ? ctx->hi : st;
  cudaStream_t S = (allow_side && ctx->hi && ctx->side && n >= 1024 && !ctx->no_overlap) ? ctx->side : nullptr;
  cudaStream_t D = S ? ctx->side_deep[0] : nullptr, T = S ? ctx->side_deep[1] : nullptr;
  // no bands while A arrives from the host: there the R12 products follow the arrival of their columns instead
  const bool bands = S && !(hooks && hooks->cols_waited);
  ctx->dep_used = 0;
  cudaEvent_t e_in = nullptr, e_out = nullptr, e_s = nullptr;
  if (M != st) {
    CAP_TRY(new_event(ctx, &e_in));
    CAP_CUDA(cudaEventRecord(e_in, st));
    CAP_CUDA(cudaStreamWaitEvent(M, e_in, 0));
    if (S) CAP_CUDA(cudaStreamWaitEvent(S, e_in, 0));
  }
  const bool aligned = ((((uintptr_t)W | (uintptr_t)R | (uintptr_t)Ri | (uintptr_t)RiT) & 15) == 0) && !((ldw | ldr | ldri | ldrit) & 1);
  Rec r{ctx, M, S, D, T, bands, W, R, Ri, RiT, ldw, ldr, ldri, ldrit, bc, split, hooks, ctx->far_min, ctx->band_min, n, aligned};
  // a top-level node the reference treats as its base case (n <= bc, cholinv.hpp:93-104) gets the FULL inverse whatever complete_inv
  // says; the skip of cholinv.hpp:147 only exists where the top node really splits at n >> split
  if (!cholinv_node_splits(n, bc, split)) complete_top = true;
  r.spine_rit = complete_top;
  CAP_TRY(rec(r, 0, n, complete_top, nullptr, nullptr, 0, nullptr));
  if (M != st) {
    if (S) {  // join the deferred streams (all their work has been consumed through events, this is just the fence)
      for (cudaStream_t d : {S, D, T}) {
        CAP_TRY(new_event(ctx, &e_s));
        CAP_CUDA(cudaEventRecord(e_s, d));
        CAP_CUDA(cudaStreamWaitEvent(M, e_s, 0));
      }
    }
    CAP_TRY(new_event(ctx, &e_out));
    CAP_CUDA(cudaEventRecord(e_out, M));
    CAP_CUDA(cudaStreamWaitEvent(st, e_out, 0));
  }
  return CAPITAL_OK;
}
