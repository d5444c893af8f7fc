// C ABI (include/capital_b200.h): context, grid helpers, generators, validators and the factor entry points.
// Host orchestration only -- every flop and every byte of layout work runs in the kernels of gemm_tn.cu,
// leaf.cu and layout.cu.  There is no CPU fallback: without a usable sm_90 device capital_create fails.
#include "common.cuh"
#include "dist.cuh"
#include "peer.cuh"
#include <math.h>
#include <stdlib.h>
#include <algorithm>

capital_status_t capital_ctx::workspace(const std::string& name, size_t bytes, void** out) {
  capital_ctx* ctx = this;
  DeviceBuf& b = pool[name];
  if (b.bytes < bytes) {
    if (b.p) CAP_CUDA(cudaFree(b.p));
    b.p = nullptr; b.bytes = 0;
    CAP_CUDA(cudaMalloc(&b.p, bytes));
    b.bytes = bytes;
    if (poison_workspace) {  // NaN in every double (and float): a read of a value nobody wrote shows up in the result
      CAP_CUDA(cudaMemsetAsync(b.p, 0xFF, bytes, cudaStreamLegacy));
      CAP_CUDA(cudaStreamSynchronize(cudaStreamLegacy));  // the context's streams are non-blocking: they do not wait for it
    }
  }
  *out = b.p;
  return CAPITAL_OK;
}

int capital_ctx::stream_id(cudaStream_t st) const {
  if (st == hi) return 1;
  if (st == side) return 2;
  if (st == side_deep[0]) return 3;
  if (st == side_deep[1]) return 4;
  if (peer) {
    const Peer* P = (const Peer*)peer;
    for (int q = 0; q < PEER_Q; q++) if (st == P->push[q]) return 5 + q;
  }
  if (st == copy_in) return 10;
  if (st == copy_out) return 11;
  return 0;
}
int capital_ctx::tl_begin(cudaStream_t st, int kind, double a, double b, double c) {
  if (!timeline) return -1;
  while (tl_pool.size() < tl_used + 2) {
    cudaEvent_t e;
    if (cudaEventCreate(&e) != cudaSuccess) return -1;
    tl_pool.push_back(e);
  }
  TlRec r{tl_pool[tl_used], tl_pool[tl_used + 1], stream_id(st), kind, a, b, c};
  tl_used += 2;
  cudaEventRecord(r.e0, st);
  tl.push_back(r);
  return (int)tl.size() - 1;
}
void capital_ctx::tl_end(cudaStream_t st, int idx) {
  if (idx >= 0) cudaEventRecord(tl[idx].e1, st);
}

bool cap_is_device_ptr(const void* p) {
  cudaPointerAttributes at;
  if (cudaPointerGetAttributes(&at, p) != cudaSuccess) { cudaGetLastError(); return false; }
  return at.type == cudaMemoryTypeDevice || at.type == cudaMemoryTypeManaged;
}

// Bring `count` doubles to the device (no-op for device pointers).
capital_status_t cap_stage_in(capital_ctx* ctx, const double* src, size_t count, const char* name, const double** out) {
  if (cap_is_device_ptr(src)) { *out = src; return CAPITAL_OK; }
  void* d;
  CAP_TRY(ctx->workspace(name, count * 8, &d));
  CAP_CUDA(cudaMemcpyAsync(d, src, count * 8, cudaMemcpyHostToDevice, ctx->stream));
  ctx->counters.h2d_bytes += (int64_t)count * 8;
  *out = (const double*)d;
  return CAPITAL_OK;
}
// Device output target for a caller pointer: the pointer itself if on device, else a workspace to be copied back.
capital_status_t cap_stage_out_begin(capital_ctx* ctx, double* dst, size_t count, const char* name, double** dev) {
  if (cap_is_device_ptr(dst)) { *dev = dst; return CAPITAL_OK; }
  void* d;
  CAP_TRY(ctx->workspace(name, count * 8, &d));
  *dev = (double*)d;
  return CAPITAL_OK;
}
capital_status_t cap_stage_out_end(capital_ctx* ctx, double* dst, size_t count, const double* dev) {
  if (dev == dst) return CAPITAL_OK;
  CAP_CUDA(cudaMemcpyAsync(dst, dev, count * 8, cudaMemcpyDeviceToHost, ctx->stream));
  ctx->counters.d2h_bytes += (int64_t)count * 8;
  return CAPITAL_OK;
}

capital_status_t cap_check_info(capital_ctx* ctx) {
  int info = 0;
  CAP_CUDA(cudaMemcpyAsync(&info, ctx->d_info, sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
  CAP_CUDA(cudaStreamSynchronize(ctx->stream));
  if (info == -3) {
    ctx->set_error("the experimental TF32 trailing-update kernel gave up on an mbarrier wait (gemm_tf32.cu watchdog): results are invalid");
    return CAPITAL_ERR_CUDA;
  }
  if (info < 0) {
    ctx->set_error("a wait on a peer GPU timed out (a rank of the grid died, or the ranks did not make the same sequence of calls)");
    return CAPITAL_ERR_COMM;
  }
  if (info != 0) {
    ctx->set_error("matrix is not positive definite: non-positive pivot " + std::to_string(info) +
                   " (a column of the matrix on one GPU; on a grid, of the base-case block that failed)");
    return CAPITAL_ERR_NOT_SPD;
  }
  return CAPITAL_OK;
}

// ---- column streaming of cholinv::factor (single GPU): A in, R and Rinv out --------------------------------------
namespace {
struct HostIO {
  capital_ctx* ctx = nullptr;
  int64_t L = 0, ld = 0;
  double *Rm = nullptr, *Ri = nullptr, *dR = nullptr, *dRinv = nullptr, *hR = nullptr, *hRinv = nullptr;
  bool packed = true;
  std::vector<std::pair<int64_t, cudaEvent_t>> chunks;  // (col_end, arrived)
  int64_t waited = 0;
  int64_t cols_out = 0, rinv_cols_out = 0;
  bool rinv_streams = false;  // Rinv columns right of the top split are final as soon as R's are (complete_inv == 0)
  int64_t rinv_top = 0;       // complete_inv == 0, packed: rows [0, rinv_top) of Rinv's columns from rinv_top on are the skipped block,
                              // zeroed in the output once at the start; the packs leave them alone
  cudaEvent_t e_out = nullptr;
};
capital_status_t io_event(capital_ctx* ctx, cudaEvent_t* e) {
  if (ctx->io_used == ctx->io_pool.size()) {
    cudaEvent_t ev;
    CAP_CUDA(cudaEventCreateWithFlags(&ev, cudaEventDisableTiming));
    ctx->io_pool.push_back(ev);
  }
  *e = ctx->io_pool[ctx->io_used++];
  return CAPITAL_OK;
}
// make st wait for the first chunk that covers columns [0, col_end); returns that chunk's end
capital_status_t hostio_wait_chunk(HostIO* io, cudaStream_t st, int64_t col_end, int64_t* waited) {
  capital_ctx* ctx = io->ctx;
  for (auto& ch : io->chunks)
    if (ch.first >= col_end) {
      CAP_CUDA(cudaStreamWaitEvent(st, ch.second, 0));
      *waited = ch.first;
      return CAPITAL_OK;
    }
  return CAPITAL_OK;
}
capital_status_t hostio_need_cols(void* user, cudaStream_t st, int64_t col_end) {
  HostIO* io = (HostIO*)user;
  if (col_end <= io->waited) return CAPITAL_OK;
  return hostio_wait_chunk(io, st, col_end, &io->waited);
}
capital_status_t hostio_wait_cols(void* user, cudaStream_t st, int64_t col_end) {
  int64_t waited = 0;
  return hostio_wait_chunk((HostIO*)user, st, col_end, &waited);
}
// columns [cols_out, col_end) of R are final (and of Rinv too when the top-level inverse block is skipped, complete_inv == 0:
// then Rinv's columns right of the top split only hold the right child's own inverse): pack them -- a contiguous range of
// the packed triangle -- and start their D2H while the rest of the factorization runs.
capital_status_t hostio_left_done(void* user, cudaStream_t st, int64_t col_end, int depth) {
  HostIO* io = (HostIO*)user;
  capital_ctx* ctx = io->ctx;
  const int64_t c0 = io->cols_out;
  if (col_end <= c0) return CAPITAL_OK;
  // Rinv: left of the top split always; the next range only when the top-level inverse block is skipped (deeper ranges still
  // miss the off-diagonal inverse blocks of the right-spine ancestors, computed after their right children)
  const bool rinv_too = depth == 0 || (depth == 1 && io->rinv_streams && io->rinv_cols_out == c0);
  const size_t off = (size_t)c0 * (c0 + 1) / 2, cnt = (size_t)col_end * (col_end + 1) / 2 - off;
  // packing is HBM-bound filler work: it goes to a low-priority stream of its own (joined through e_out after the recursion), not
  // to the chain, nor in front of the deferred far updates (the top-level one would wait for it).  Host callers keep it on the chain:
  // the D2H of the range should start right away.
  cudaStream_t ps = (!ctx->no_overlap && !io->hR && !io->hRinv) ? ctx->copy_out : st;
  cudaEvent_t e;
  if (ps != st) {
    CAP_TRY(io_event(ctx, &e));
    CAP_CUDA(cudaEventRecord(e, st));
    CAP_CUDA(cudaStreamWaitEvent(ps, e, 0));
  }
  CAP_TRY(pack_upper(ctx, ps, io->L, io->Rm, io->ld, io->dR, 0, c0, col_end));
  if (rinv_too) CAP_TRY(pack_upper(ctx, ps, io->L, io->Ri, io->ld, io->dRinv, 0, c0, col_end, io->rinv_top));
  io->cols_out = col_end;
  if (rinv_too) io->rinv_cols_out = col_end;
  if (!io->hR && !io->hRinv) {  // device outputs: nothing to copy out
    if (ps != st) {
      CAP_TRY(io_event(ctx, &io->e_out));
      CAP_CUDA(cudaEventRecord(io->e_out, ps));
    }
    return CAPITAL_OK;
  }
  CAP_TRY(io_event(ctx, &e));
  CAP_CUDA(cudaEventRecord(e, ps));
  CAP_CUDA(cudaStreamWaitEvent(ctx->copy_out, e, 0));
  if (io->hR) { CAP_CUDA(cudaMemcpyAsync(io->hR + off, io->dR + off, cnt * 8, cudaMemcpyDeviceToHost, ctx->copy_out)); ctx->counters.d2h_bytes += (int64_t)cnt * 8; }
  if (io->hRinv && rinv_too) { CAP_CUDA(cudaMemcpyAsync(io->hRinv + off, io->dRinv + off, cnt * 8, cudaMemcpyDeviceToHost, ctx->copy_out)); ctx->counters.d2h_bytes += (int64_t)cnt * 8; }
  CAP_TRY(io_event(ctx, &io->e_out));
  CAP_CUDA(cudaEventRecord(io->e_out, ctx->copy_out));
  return CAPITAL_OK;
}
int64_t hostio_cols_waited(void* user) { return ((HostIO*)user)->waited; }
// all of R is final (the last base case has been issued on st): its columns not packed yet are packed, and copied out, on the copy-out
// stream while the chain still computes the inverse blocks of the right spine
capital_status_t hostio_r_final(void* user, cudaStream_t st) {
  HostIO* io = (HostIO*)user;
  capital_ctx* ctx = io->ctx;
  const int64_t c0 = io->cols_out;
  if (c0 >= io->L || ctx->no_overlap) return CAPITAL_OK;
  cudaEvent_t e;
  CAP_TRY(io_event(ctx, &e));
  CAP_CUDA(cudaEventRecord(e, st));
  CAP_CUDA(cudaStreamWaitEvent(ctx->copy_out, e, 0));
  CAP_TRY(pack_upper(ctx, ctx->copy_out, io->L, io->Rm, io->ld, io->dR, 0, c0, io->L));
  io->cols_out = io->L;
  if (io->hR) {
    const size_t off = (size_t)c0 * (c0 + 1) / 2, cnt = (size_t)io->L * (io->L + 1) / 2 - off;
    CAP_CUDA(cudaMemcpyAsync(io->hR + off, io->dR + off, cnt * 8, cudaMemcpyDeviceToHost, ctx->copy_out));
    ctx->counters.d2h_bytes += (int64_t)cnt * 8;
  }
  CAP_TRY(io_event(ctx, &io->e_out));
  CAP_CUDA(cudaEventRecord(io->e_out, ctx->copy_out));
  return CAPITAL_OK;
}
// pack columns [done, col_end) of R (or Rinv) on the chain and queue their D2H on the copy-out stream (host outputs only)
capital_status_t hostio_emit(HostIO* io, cudaStream_t st, bool r_part, int64_t col_end) {
  capital_ctx* ctx = io->ctx;
  int64_t& done = r_part ? io->cols_out : io->rinv_cols_out;
  const int64_t c0 = done;
  if (col_end <= c0) return CAPITAL_OK;
  const double* src = r_part ? io->Rm : io->Ri;
  double* dev = r_part ? io->dR : io->dRinv;
  double* host = r_part ? io->hR : io->hRinv;
  const size_t off = (size_t)c0 * (c0 + 1) / 2, cnt = (size_t)col_end * (col_end + 1) / 2 - off;
  CAP_TRY(pack_upper(ctx, st, io->L, src, io->ld, dev, 0, c0, col_end, r_part ? 0 : io->rinv_top));
  done = col_end;
  if (!host) return CAPITAL_OK;
  cudaEvent_t e;
  CAP_TRY(io_event(ctx, &e));
  CAP_CUDA(cudaEventRecord(e, st));
  CAP_CUDA(cudaStreamWaitEvent(ctx->copy_out, e, 0));
  CAP_CUDA(cudaMemcpyAsync(host + off, dev + off, cnt * 8, cudaMemcpyDeviceToHost, ctx->copy_out));
  ctx->counters.d2h_bytes += (int64_t)cnt * 8;
  CAP_TRY(io_event(ctx, &io->e_out));
  CAP_CUDA(cudaEventRecord(io->e_out, ctx->copy_out));
  return CAPITAL_OK;
}
// the top-level right child is done: R is final everywhere (and so is Rinv when the top-level inverse block is skipped); its last
// columns leave while the top-level inverse block is still being computed
capital_status_t hostio_right_done(void* user, cudaStream_t st) {
  HostIO* io = (HostIO*)user;
  CAP_TRY(hostio_emit(io, st, true, io->L));
  if (io->rinv_streams) CAP_TRY(hostio_emit(io, st, false, io->L));
  return CAPITAL_OK;
}
capital_status_t hostio_inv_cols(void* user, cudaStream_t st, int64_t col_end) { return hostio_emit((HostIO*)user, st, false, col_end); }
}  // namespace

extern "C" {

capital_status_t capital_grid_square(int size, int rank, int c, int layout, int num_chunks, capital_grid_t* out) {
  if (!out || size <= 0 || rank < 0 || rank >= size || c <= 0 || layout != 0) return CAPITAL_ERR_INVALID;
  capital_grid_t g{};
  g.size = size; g.rank = rank; g.c = c; g.layout = layout; g.num_chunks = num_chunks;
  g.d = (int)nearbyint(ceil(sqrt((double)(size / c))));  // topology.h:77
  g.z = rank % c;
  g.y = rank / (g.d * c);
  g.x = (rank % (g.d * c)) / c;
  if ((int64_t)g.c * g.d * g.d != size) return CAPITAL_ERR_INVALID;
  *out = g;
  return CAPITAL_OK;
}
capital_status_t capital_grid_rect(int size, int rank, int c, int layout, int num_chunks, capital_grid_t* out) {
  if (!out || size <= 0 || rank < 0 || rank >= size || c <= 0 || layout != 0) return CAPITAL_ERR_INVALID;
  if (size % (c * c)) return CAPITAL_ERR_INVALID;
  capital_grid_t g{};
  g.size = size; g.rank = rank; g.c = c; g.layout = layout; g.num_chunks = num_chunks;
  g.d = size / (c * c);  // topology.h:46
  g.z = rank % c;
  g.y = rank / (c * c);
  g.x = (rank % (c * c)) / c;
  *out = g;
  return CAPITAL_OK;
}
int64_t capital_cholinv_bc_dimension(int64_t local_dim, int c, int d, int64_t bc_mult_dim) {
  int64_t bc = (int64_t)c * d;  // cholinv.hpp:15-18
  if (bc_mult_dim < 0) { for (int64_t i = 0; i < -bc_mult_dim; i++) bc *= 2; }
  else { for (int64_t i = 0; i < bc_mult_dim; i++) bc /= 2; }
  if (bc < 1) bc = 1;
  if (bc > local_dim) bc = local_dim;
  return (int64_t)d * (local_dim / bc);
}

// The deferred stream gets its own SM partition (a CUDA green context): all SMs but `reserve` of them.  Deferred GEMM tiles hold an
// SM for up to ~1 ms and a running CTA cannot be preempted, so without a partition the latency-critical kernels of the chain
// (8-CTA cluster base case, small products) wait that long for SMs although their stream has the higher priority (tools/probe_greenctx.cu
// measures this).
// The chain's streams stay in the primary context and may use every SM.
static bool make_green_side_stream(capital_ctx* ctx, int reserve, int prio) {
  typedef CUresult (*fn_devget)(CUdevice*, int);
  typedef CUresult (*fn_getres)(CUdevice, CUdevResource*, CUdevResourceType);
  typedef CUresult (*fn_split)(CUdevResource*, unsigned int*, const CUdevResource*, CUdevResource*, unsigned int, unsigned int);
  typedef CUresult (*fn_desc)(CUdevResourceDesc*, CUdevResource*, unsigned int);
  typedef CUresult (*fn_gcreate)(CUgreenCtx*, CUdevResourceDesc, CUdevice, unsigned int);
  typedef CUresult (*fn_gstream)(CUstream*, CUgreenCtx, unsigned int, int);
  void *p1 = nullptr, *p2 = nullptr, *p3 = nullptr, *p4 = nullptr, *p5 = nullptr, *p6 = nullptr;
  cudaDriverEntryPointQueryResult q;
  if (cudaGetDriverEntryPoint("cuDeviceGet", &p1, cudaEnableDefault, &q) != cudaSuccess || !p1) return false;
  if (cudaGetDriverEntryPoint("cuDeviceGetDevResource", &p2, cudaEnableDefault, &q) != cudaSuccess || !p2) return false;
  if (cudaGetDriverEntryPoint("cuDevSmResourceSplitByCount", &p3, cudaEnableDefault, &q) != cudaSuccess || !p3) return false;
  if (cudaGetDriverEntryPoint("cuDevResourceGenerateDesc", &p4, cudaEnableDefault, &q) != cudaSuccess || !p4) return false;
  if (cudaGetDriverEntryPoint("cuGreenCtxCreate", &p5, cudaEnableDefault, &q) != cudaSuccess || !p5) return false;
  if (cudaGetDriverEntryPoint("cuGreenCtxStreamCreate", &p6, cudaEnableDefault, &q) != cudaSuccess || !p6) return false;
  CUdevice dev;
  if (((fn_devget)p1)(&dev, ctx->device) != CUDA_SUCCESS) return false;
  CUdevResource all, rem;
  if (((fn_getres)p2)(dev, &all, CU_DEV_RESOURCE_TYPE_SM) != CUDA_SUCCESS) return false;
  unsigned nb = 0;
  if (((fn_split)p3)(nullptr, &nb, &all, nullptr, 0, 8) != CUDA_SUCCESS || nb < 2) return false;
  std::vector<CUdevResource> groups(nb);
  if (((fn_split)p3)(groups.data(), &nb, &all, &rem, 0, 8) != CUDA_SUCCESS) return false;
  unsigned skip = 0, got = 0;
  while (skip < nb - 1 && (int)got < reserve) got += groups[skip++].sm.smCount;
  std::vector<CUdevResource> far(groups.begin() + skip, groups.begin() + nb);
  if (rem.sm.smCount) far.push_back(rem);
  CUdevResourceDesc desc;
  if (((fn_desc)p4)(&desc, far.data(), (unsigned)far.size()) != CUDA_SUCCESS) return false;
  CUgreenCtx g;
  if (((fn_gcreate)p5)(&g, desc, dev, CU_GREEN_CTX_DEFAULT_STREAM) != CUDA_SUCCESS) return false;
  CUstream gs, gd[2];
  if (((fn_gstream)p6)(&gs, g, CU_STREAM_NON_BLOCKING, prio) != CUDA_SUCCESS) return false;
  for (int i = 0; i < 2; i++)
    if (((fn_gstream)p6)(&gd[i], g, CU_STREAM_NON_BLOCKING, prio - 1 - i) != CUDA_SUCCESS) return false;
  ctx->side = (cudaStream_t)gs;
  ctx->side_deep[0] = (cudaStream_t)gd[0];
  ctx->side_deep[1] = (cudaStream_t)gd[1];
  ctx->green = (void*)g;
  return true;
}

capital_status_t capital_create(capital_ctx** out, const capital_grid_t* grid, int device, void* stream) {
  if (!out || !grid) return CAPITAL_ERR_INVALID;
  *out = nullptr;
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev <= 0 || device < 0 || device >= ndev) return CAPITAL_ERR_CUDA;
  cudaDeviceProp prop;
  if (cudaGetDeviceProperties(&prop, device) != cudaSuccess) return CAPITAL_ERR_CUDA;
  if (prop.major != 9) return CAPITAL_ERR_CUDA;  // sm_90a binary only: no fallback path exists
  if (cudaSetDevice(device) != cudaSuccess) return CAPITAL_ERR_CUDA;
  capital_ctx* ctx = new capital_ctx();
  ctx->grid = *grid;
  ctx->device = device;
  ctx->num_sms = prop.multiProcessorCount;
  if (stream) { ctx->stream = (cudaStream_t)stream; ctx->own_stream = false; }
  else {
    if (cudaStreamCreateWithFlags(&ctx->stream, cudaStreamNonBlocking) != cudaSuccess) { delete ctx; return CAPITAL_ERR_CUDA; }
    ctx->own_stream = true;
  }
  int prio_lo = 0, prio_hi = 0;
  cudaDeviceGetStreamPriorityRange(&prio_lo, &prio_hi);  // lo = numerically greatest = lowest priority
  int reserve = 8;  // SMs kept free of deferred work [env CAPITAL_GREEN_SMS; 0 = plain low-priority stream]
  if (const char* e = getenv("CAPITAL_GREEN_SMS")) reserve = atoi(e);
  bool ok = true;
  if (reserve <= 0 || !make_green_side_stream(ctx, reserve, prio_lo)) {
    ok = cudaStreamCreateWithPriority(&ctx->side, cudaStreamNonBlocking, prio_lo) == cudaSuccess;
    for (int i = 0; i < 2; i++) ok = ok && cudaStreamCreateWithPriority(&ctx->side_deep[i], cudaStreamNonBlocking, prio_lo - 1 - i) == cudaSuccess;
  }
  ok = ok && cudaStreamCreateWithPriority(&ctx->hi, cudaStreamNonBlocking, prio_hi) == cudaSuccess;
  ok = ok && cudaStreamCreateWithFlags(&ctx->copy_in, cudaStreamNonBlocking) == cudaSuccess;
  ok = ok && cudaStreamCreateWithFlags(&ctx->copy_out, cudaStreamNonBlocking) == cudaSuccess;
  ok = ok && cudaEventCreate(&ctx->ev_start) == cudaSuccess && cudaEventCreate(&ctx->ev_stop) == cudaSuccess;
  ok = ok && cudaEventCreateWithFlags(&ctx->ev_fork, cudaEventDisableTiming) == cudaSuccess;
  ok = ok && cudaMalloc(&ctx->d_info, sizeof(int)) == cudaSuccess && cudaMalloc(&ctx->d_scalars, 16 * sizeof(double)) == cudaSuccess;
  ok = ok && cudaMemset(ctx->d_info, 0, sizeof(int)) == cudaSuccess;
  cudaDriverEntryPointQueryResult qres;
  void* fn = nullptr;
  ok = ok && cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres) == cudaSuccess && fn != nullptr;
  if (!ok) { capital_destroy(ctx); return CAPITAL_ERR_CUDA; }
  ctx->encode = (cuTensorMapEncodeTiled_fn)fn;
  if (gemm_tn_init(ctx) != CAPITAL_OK || leaf_init(ctx) != CAPITAL_OK || syevj_init(ctx) != CAPITAL_OK) { capital_destroy(ctx); return CAPITAL_ERR_CUDA; }
  if (const char* e = getenv("CAPITAL_TF32_MIN_K")) ctx->tf32_min_k = atoll(e);
  if (const char* e = getenv("CAPITAL_FAR_MIN")) ctx->far_min = atoll(e);
  if (const char* e = getenv("CAPITAL_SIDE_MIN")) ctx->side_min = atoll(e);
  if (const char* e = getenv("CAPITAL_BAND_MIN")) ctx->band_min = atoll(e);
  if (const char* e = getenv("CAPITAL_POISON_WORKSPACE")) ctx->poison_workspace = atoi(e) != 0;
  *out = ctx;
  return CAPITAL_OK;
}

void capital_destroy(capital_ctx* ctx) {
  if (!ctx) return;
  cudaSetDevice(ctx->device);
  if (ctx->stream) cudaStreamSynchronize(ctx->stream);
  dist_destroy(ctx);
  for (auto& kv : ctx->pool) if (kv.second.p) cudaFree(kv.second.p);
  if (ctx->d_info) cudaFree(ctx->d_info);
  if (ctx->d_scalars) cudaFree(ctx->d_scalars);
  if (ctx->ev_start) cudaEventDestroy(ctx->ev_start);
  if (ctx->ev_stop) cudaEventDestroy(ctx->ev_stop);
  if (ctx->ev_fork) cudaEventDestroy(ctx->ev_fork);
  for (cudaEvent_t e : ctx->prof_pool) cudaEventDestroy(e);
  for (cudaEvent_t e : ctx->tl_pool) cudaEventDestroy(e);
  if (ctx->side) cudaStreamDestroy(ctx->side);
  for (int i = 0; i < 2; i++) if (ctx->side_deep[i]) cudaStreamDestroy(ctx->side_deep[i]);
  if (ctx->green) {
    typedef CUresult (*fn_gdestroy)(CUgreenCtx);
    void* pd = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuGreenCtxDestroy", &pd, cudaEnableDefault, &q) == cudaSuccess && pd) ((fn_gdestroy)pd)((CUgreenCtx)ctx->green);
  }
  if (ctx->hi) cudaStreamDestroy(ctx->hi);
  if (ctx->copy_in) cudaStreamDestroy(ctx->copy_in);
  if (ctx->copy_out) cudaStreamDestroy(ctx->copy_out);
  for (cudaEvent_t e : ctx->dep_pool) cudaEventDestroy(e);
  for (cudaEvent_t e : ctx->io_pool) cudaEventDestroy(e);
  if (ctx->own_stream && ctx->stream) cudaStreamDestroy(ctx->stream);
  delete ctx;
}

const char* capital_last_error(const capital_ctx* ctx) { return ctx ? ctx->err.c_str() : "null context"; }
capital_status_t capital_get_counters(const capital_ctx* ctx, capital_counters_t* out) {
  if (!ctx || !out) return CAPITAL_ERR_INVALID;
  *out = ctx->counters;
  return CAPITAL_OK;
}
capital_status_t capital_reset_counters(capital_ctx* ctx) {
  if (!ctx) return CAPITAL_ERR_INVALID;
  ctx->counters = capital_counters_t{};
  return CAPITAL_OK;
}
capital_status_t capital_synchronize(capital_ctx* ctx) {
  if (!ctx) return CAPITAL_ERR_INVALID;
  CAP_CUDA(cudaStreamSynchronize(ctx->stream));
  return CAPITAL_OK;
}
capital_status_t capital_set_stream(capital_ctx* ctx, void* stream) {
  if (!ctx || !stream) return CAPITAL_ERR_INVALID;
  CAP_CUDA(cudaSetDevice(ctx->device));
  cudaStream_t ns = (cudaStream_t)stream;
  if (ns == ctx->stream) return CAPITAL_OK;
  // order the new stream after the work already enqueued on the old one (workspaces are shared between calls)
  CAP_CUDA(cudaEventRecord(ctx->ev_fork, ctx->stream));
  CAP_CUDA(cudaStreamWaitEvent(ns, ctx->ev_fork, 0));
  if (ctx->own_stream) { CAP_CUDA(cudaStreamSynchronize(ctx->stream)); CAP_CUDA(cudaStreamDestroy(ctx->stream)); ctx->own_stream = false; }
  ctx->stream = ns;
  return CAPITAL_OK;
}
capital_status_t capital_release_workspace(capital_ctx* ctx) {
  if (!ctx) return CAPITAL_ERR_INVALID;
  CAP_CUDA(cudaSetDevice(ctx->device));
  CAP_CUDA(cudaDeviceSynchronize());  // side / copy streams may still reference the buffers
  CAP_TRY(dist_release_peer_maps(ctx));
  for (auto& kv : ctx->pool) if (kv.second.p) CAP_CUDA(cudaFree(kv.second.p));
  ctx->pool.clear();
  return CAPITAL_OK;
}
capital_status_t capital_last_factor_ms(const capital_ctx* ctx_, float* ms) {
  capital_ctx* ctx = const_cast<capital_ctx*>(ctx_);
  if (!ctx || !ms) return CAPITAL_ERR_INVALID;
  CAP_CUDA(cudaEventElapsedTime(ms, ctx->ev_start, ctx->ev_stop));
  return CAPITAL_OK;
}

capital_status_t capital_timeline_begin(capital_ctx* ctx) {
  if (!ctx) return CAPITAL_ERR_INVALID;
  ctx->timeline = true; ctx->tl.clear(); ctx->tl_used = 0;
  return CAPITAL_OK;
}
capital_status_t capital_timeline_end(capital_ctx* ctx, double* out, int64_t cap_records, int64_t* n_records) {
  if (!ctx || !n_records) return CAPITAL_ERR_INVALID;
  ctx->timeline = false;
  CAP_CUDA(cudaSetDevice(ctx->device));
  CAP_CUDA(cudaDeviceSynchronize());
  *n_records = (int64_t)ctx->tl.size();
  if (out && !ctx->tl.empty()) {
    // time origin: the earliest start
    cudaEvent_t base = ctx->tl[0].e0;
    for (auto& r : ctx->tl) {
      float d = 0;
      if (cudaEventElapsedTime(&d, base, r.e0) == cudaSuccess && d < 0) base = r.e0;
    }
    for (int64_t i = 0; i < *n_records && i < cap_records; i++) {
      const auto& r = ctx->tl[i];
      float t0 = 0, t1 = 0;
      CAP_CUDA(cudaEventElapsedTime(&t0, base, r.e0));
      CAP_CUDA(cudaEventElapsedTime(&t1, base, r.e1));
      double* o = out + i * 8;
      o[0] = r.sid; o[1] = r.kind; o[2] = t0; o[3] = t1; o[4] = r.a; o[5] = r.b; o[6] = r.c; o[7] = 0;
    }
  }
  return CAPITAL_OK;
}
capital_status_t capital_probe_dmma_f64(capital_ctx* ctx, double* tflops, double* ms) {
  if (!ctx || !tflops || !ms) return CAPITAL_ERR_INVALID;
  CAP_CUDA(cudaSetDevice(ctx->device));
  return gemm_probe_dmma(ctx, tflops, ms);
}
capital_status_t capital_set_overlap(capital_ctx* ctx, int enabled) {
  if (!ctx) return CAPITAL_ERR_INVALID;
  ctx->no_overlap = !enabled;
  return CAPITAL_OK;
}
capital_status_t capital_profile_begin(capital_ctx* ctx) {
  if (!ctx) return CAPITAL_ERR_INVALID;
  ctx->profiling = true; ctx->prof_used = 0; ctx->prof_recs.clear();
  return CAPITAL_OK;
}
capital_status_t capital_profile_end(capital_ctx* ctx, double* kernel_ms, double* kernel_flops, int64_t* launches) {
  if (!ctx || !kernel_ms || !kernel_flops || !launches) return CAPITAL_ERR_INVALID;
  ctx->profiling = false;
  CAP_CUDA(cudaStreamSynchronize(ctx->stream));
  double ms = 0, fl = 0;
  for (auto& r : ctx->prof_recs) {
    float t = 0;
    CAP_CUDA(cudaEventElapsedTime(&t, r.e0, r.e1));
    ms += t; fl += r.flops;
  }
  *kernel_ms = ms; *kernel_flops = fl; *launches = (int64_t)ctx->prof_recs.size();
  ctx->prof_recs.clear(); ctx->prof_used = 0;
  return CAPITAL_OK;
}

// ---- generators -------------------------------------------------------------------------------
capital_status_t capital_distribute_symmetric_f64(capital_ctx* ctx, double* A_local, int64_t n, int diag_dom) {
  if (!ctx || !A_local || n <= 0) return CAPITAL_ERR_INVALID;
  CAP_CUDA(cudaSetDevice(ctx->device));
  const int d = ctx->grid.d;
  const int64_t L = ceil_div(n, d);
  double* dev;
  CAP_TRY(cap_stage_out_begin(ctx, A_local, (size_t)L * L, "gen_out", &dev));
  CAP_TRY(gen_symmetric(ctx, ctx->stream, dev, L, L, L, n, ctx->grid.x, ctx->grid.y, d, diag_dom));
  CAP_TRY(cap_stage_out_end(ctx, A_local, (size_t)L * L, dev));
  CAP_CUDA(cudaStreamSynchronize(ctx->stream));
  return CAPITAL_OK;
}
capital_status_t capital_distribute_random_f64(capital_ctx* ctx, double* A_local, int64_t m, int64_t n, int64_t key) {
  if (!ctx || !A_local || n <= 0 || m <= 0) return CAPITAL_ERR_INVALID;
  CAP_CUDA(cudaSetDevice(ctx->device));
  const int c = ctx->grid.c, d = ctx->grid.d, x = ctx->grid.x, y = ctx->grid.y;
  const int64_t lr = ceil_div(m, d), lc = ceil_div(n, c);
  // structure.hpp:110-111: the stream is consumed over the un-padded local extent only
  const int64_t pad_c = ((n % c != 0) && ((lc - 1) * c + x >= n)) ? lc - 1 : lc;
  const int64_t pad_r = ((m % d != 0) && ((lr - 1) * d + y >= m)) ? lr - 1 : lr;
  double* dev;
  CAP_TRY(cap_stage_out_begin(ctx, A_local, (size_t)lr * lc, "gen_out", &dev));
  CAP_TRY(gen_random(ctx, ctx->stream, dev, lr, lr, lc, pad_r, pad_c, key));
  CAP_TRY(cap_stage_out_end(ctx, A_local, (size_t)lr * lc, dev));
  CAP_CUDA(cudaStreamSynchronize(ctx->stream));
  return CAPITAL_OK;
}

// ---- CholInv ----------------------------------------------------------------------------------
capital_status_t capital_cholinv_factor_f64(capital_ctx* ctx, const double* A_local, int64_t n, const capital_cholinv_args_t* args,
                                            capital_structure_t ostruct, double* R_local, double* Rinv_local) {
  if (!ctx) return CAPITAL_ERR_INVALID;
  if (!A_local || !args || !R_local || !Rinv_local || n <= 0 || args->split <= 0 || args->dir != 'U') {
    ctx->set_error("cholinv::factor: invalid arguments (split > 0 and dir == 'U' are required, cholinv.hpp:9)");
    return CAPITAL_ERR_INVALID;
  }
  CAP_CUDA(cudaSetDevice(ctx->device));
  const capital_grid_t& g = ctx->grid;
  if (g.size > 1) return dist_cholinv_factor(ctx, A_local, n, args, ostruct, R_local, Rinv_local);

  const int64_t L = n, ld = round_up(L, 16);
  const size_t out_count = ostruct == CAPITAL_UPPERTRI_PACKED ? (size_t)L * (L + 1) / 2 : (size_t)L * L;
  cudaStream_t st = ctx->stream;
  ctx->io_used = 0;
  CAP_CUDA(cudaEventRecord(ctx->ev_start, st));
  double *W, *Rm, *Ri, *RiT, *dR, *dRinv;
  CAP_TRY(ctx->workspace("W", (size_t)ld * L * 8, (void**)&W));
  CAP_TRY(ctx->workspace("Rm", (size_t)ld * L * 8, (void**)&Rm));
  CAP_TRY(ctx->workspace("Ri", (size_t)ld * L * 8, (void**)&Ri));
  CAP_TRY(ctx->workspace("RiT", (size_t)ld * L * 8, (void**)&RiT));
  CAP_TRY(cap_stage_out_begin(ctx, R_local, out_count, "R_out", &dR));
  CAP_TRY(cap_stage_out_begin(ctx, Rinv_local, out_count, "Rinv_out", &dRinv));
  CAP_CUDA(cudaMemsetAsync(ctx->d_info, 0, sizeof(int), st));
  const int64_t bc = capital_cholinv_bc_dimension(L, g.c, g.d, args->bc_mult_dim);
  // the top-level block of Rinv that complete_inv = 0 skips (cholinv.hpp:147) -- it only exists when the top node splits (same
  // predicate as cholinv_local: a top-level base case returns the full inverse).  Nothing in the factorization reads it: the packed
  // output gets its zeros without reading the workspace (zero_packed_top below), the rect output exposes the whole buffer and clears it.
  const bool skipped = args->complete_inv == 0 && cholinv_node_splits(L, bc, (int)args->split);
  if (ostruct == CAPITAL_RECT) CAP_CUDA(cudaMemsetAsync(Ri, 0, (size_t)ld * L * 8, st));
  else CAP_TRY(zero_band(ctx, st, L, Ri, ld));
  CAP_TRY(zero_band(ctx, st, L, RiT, ld));
  if (ostruct == CAPITAL_RECT) CAP_CUDA(cudaMemsetAsync(Rm, 0, (size_t)ld * L * 8, st));

  // A streams into W by column chunks on the copy-in stream while the recursion already works on the leading columns (it consumes
  // W left to right): the chain waits for each chunk where it first reads its columns, so the first base case starts after the
  // first, narrow chunk instead of after the whole copy.  Device input is copied too (the caller's A is not destroyed).
  // The finished left half of R / Rinv is packed (and, for host outputs, copied out) while the right half computes.
  HostIO io;
  io.ctx = ctx; io.L = L; io.ld = ld; io.Rm = Rm; io.Ri = Ri; io.dR = dR; io.dRinv = dRinv;
  io.hR = (dR != R_local) ? R_local : nullptr; io.hRinv = (dRinv != Rinv_local) ? Rinv_local : nullptr;
  io.packed = ostruct == CAPITAL_UPPERTRI_PACKED;
  io.rinv_streams = skipped;
  io.rinv_top = skipped && io.packed ? L >> args->split : 0;
  CholinvHooks hooks{&io, hostio_need_cols, nullptr};
  hooks.wait_cols = hostio_wait_cols;
  const bool host_in = !cap_is_device_ptr(A_local);
  cudaEvent_t e_zero = nullptr;
  {
    cudaEvent_t e0;
    CAP_TRY(io_event(ctx, &e0));
    CAP_CUDA(cudaEventRecord(e0, st));  // W and the outputs must be free (previous users on st) before the copies land
    CAP_CUDA(cudaStreamWaitEvent(ctx->copy_in, e0, 0));
    if (io.rinv_top) {
      // the zeros of the skipped Rinv block depend on nothing: they are written beside the first base cases, off the chain and out
      // of the final pack (the copy-out stream's packs and copies of finished columns queue behind them)
      CAP_CUDA(cudaStreamWaitEvent(ctx->copy_out, e0, 0));
      CAP_TRY(zero_packed_top(ctx, ctx->copy_out, L, dRinv, io.rinv_top));
      CAP_TRY(io_event(ctx, &e_zero));
      CAP_CUDA(cudaEventRecord(e_zero, ctx->copy_out));
    }
    const int64_t chunk = round_up(ceil_div(L, 16), 64);
    for (int64_t c0 = 0; c0 < L;) {
      // the first base case reads only its own columns: a narrow first chunk lets it start almost at once
      const int64_t nc = std::min(c0 == 0 ? std::min<int64_t>(chunk, 512) : chunk, L - c0);
      // only the upper triangle of A is read (serialize<uppertri>(A -> R), cholinv.hpp:13): rows [0, c0 + nc) of this chunk.  The
      // strictly lower blocks of W are the scratch for T^T, written before they are read.
      const int64_t rows = c0 + nc;
      const int tli = ctx->tl_begin(ctx->copy_in, 8, 2, (double)rows, (double)nc);
      CAP_CUDA(cudaMemcpy2DAsync(W + c0 * ld, (size_t)ld * 8, A_local + c0 * L, (size_t)L * 8, (size_t)rows * 8, (size_t)nc,
                                 host_in ? cudaMemcpyHostToDevice : cudaMemcpyDeviceToDevice, ctx->copy_in));
      ctx->tl_end(ctx->copy_in, tli);
      if (host_in) ctx->counters.h2d_bytes += rows * nc * 8;
      cudaEvent_t e;
      CAP_TRY(io_event(ctx, &e));
      CAP_CUDA(cudaEventRecord(e, ctx->copy_in));
      io.chunks.push_back({c0 + nc, e});
      c0 += nc;
    }
  }
  if (io.packed && L >= 2048) {  // finished column ranges are packed (and copied out) early
    hooks.left_done = hostio_left_done;
    hooks.r_final = hostio_r_final;
  }
  // Host input arrives at PCIe speed: R12 products are issued by column chunks that follow it (and there are no bands).  Device input
  // has arrived long before any R12: the products are issued whole, with their leading bands.
  if (host_in) hooks.cols_waited = hostio_cols_waited;
  if (hooks.left_done && (io.hR || io.hRinv)) {  // host outputs: the tail of R and the top-level inverse block stream out too
    hooks.right_done = hostio_right_done;
    if (io.hRinv) hooks.inv_cols = hostio_inv_cols;
  }
  CAP_TRY(cholinv_local(ctx, st, L, W, ld, Rm, ld, Ri, ld, RiT, ld, args->complete_inv != 0, bc, (int)args->split, &hooks));
  if (ostruct == CAPITAL_UPPERTRI_PACKED) {
    if (e_zero) CAP_CUDA(cudaStreamWaitEvent(st, e_zero, 0));
    {  // columns [0, c0) are already packed (and on their way to the host)
      const int64_t c0 = io.cols_out;
      const size_t off = (size_t)c0 * (c0 + 1) / 2, cnt = out_count - off;
      CAP_TRY(pack_upper(ctx, st, L, Rm, ld, dR, 0, c0, L));
      if (io.hR && cnt) { CAP_CUDA(cudaMemcpyAsync(io.hR + off, dR + off, cnt * 8, cudaMemcpyDeviceToHost, st)); ctx->counters.d2h_bytes += (int64_t)cnt * 8; }
    }
    {
      const int64_t c0 = io.rinv_cols_out;
      const size_t off = (size_t)c0 * (c0 + 1) / 2, cnt = out_count - off;
      CAP_TRY(pack_upper(ctx, st, L, Ri, ld, dRinv, 0, c0, L, io.rinv_top));
      if (io.hRinv && cnt) { CAP_CUDA(cudaMemcpyAsync(io.hRinv + off, dRinv + off, cnt * 8, cudaMemcpyDeviceToHost, st)); ctx->counters.d2h_bytes += (int64_t)cnt * 8; }
    }
    if (io.e_out) CAP_CUDA(cudaStreamWaitEvent(st, io.e_out, 0));  // the early D2H of the left half
  } else {
    CAP_TRY(triu_copy(ctx, st, L, Rm, ld, dR, L, 0));
    CAP_TRY(triu_copy(ctx, st, L, Ri, ld, dRinv, L, 0));
    CAP_TRY(cap_stage_out_end(ctx, R_local, out_count, dR));
    CAP_TRY(cap_stage_out_end(ctx, Rinv_local, out_count, dRinv));
  }
  CAP_CUDA(cudaEventRecord(ctx->ev_stop, st));
  return cap_check_info(ctx);
}

capital_status_t capital_cholinv_residual_f64(capital_ctx* ctx, const double* A_local, int64_t n, capital_structure_t structure,
                                              const double* R_local, double* residual) {
  if (!ctx || !A_local || !R_local || !residual || n <= 0) return CAPITAL_ERR_INVALID;
  CAP_CUDA(cudaSetDevice(ctx->device));
  const capital_grid_t& g = ctx->grid;
  if (g.size > 1) return dist_cholinv_residual(ctx, A_local, n, structure, R_local, residual);
  const int64_t L = n, ld = round_up(L, 16);
  cudaStream_t st = ctx->stream;
  const size_t r_count = structure == CAPITAL_UPPERTRI_PACKED ? (size_t)L * (L + 1) / 2 : (size_t)L * L;
  const double *dA, *dRin;
  CAP_TRY(cap_stage_in(ctx, A_local, (size_t)L * L, "A_in", &dA));
  CAP_TRY(cap_stage_in(ctx, R_local, r_count, "R_in", &dRin));
  double *E, *Rr;
  CAP_TRY(ctx->workspace("W", (size_t)ld * L * 8, (void**)&E));
  CAP_TRY(ctx->workspace("Rm", (size_t)ld * L * 8, (void**)&Rr));
  if (structure == CAPITAL_UPPERTRI_PACKED) CAP_TRY(unpack_upper(ctx, st, L, dRin, Rr, ld));
  else CAP_TRY(triu_copy(ctx, st, L, dRin, L, Rr, ld, 0));  // util::remove_triangle, validate.hpp:11
  CAP_TRY(copy_block(ctx, st, L, L, dA, L, E, ld));
  CAP_CUDA(cudaMemsetAsync(ctx->d_scalars, 0, 2 * sizeof(double), st));
  CAP_TRY(sumsq_block(ctx, st, L, L, E, ld, 1, 0, 0, 1, ctx->d_scalars + 1));  // control: sum_upper A^2
  // E = R^T R - A on the upper tiles (validate.hpp:35 with gemm(T,N,1,-1))
  CAP_TRY(gemm_tn(ctx, st, L, L, L, 1.0, Rr, ld, Rr, ld, -1.0, E, ld,
                  CAPITAL_GEMM_A_UPPER | CAPITAL_GEMM_B_UPPER | CAPITAL_GEMM_C_UPPER));
  CAP_TRY(sumsq_block(ctx, st, L, L, E, ld, 1, 0, 0, 1, ctx->d_scalars));
  double h[2];
  CAP_CUDA(cudaMemcpyAsync(h, ctx->d_scalars, 2 * sizeof(double), cudaMemcpyDeviceToHost, st));
  CAP_CUDA(cudaStreamSynchronize(st));
  *residual = sqrt(h[0]) / sqrt(h[1]);  // util.hpp:51
  return CAPITAL_OK;
}

// A X = B from the factor's outputs (mode SOLVE_FULL), or one of its two halves alone (SOLVE_RINVT: X = Rinv^T B, SOLVE_RINV: X = Rinv B).
// Rinv complete: X = Rinv (Rinv^T B), two passes over the triangle per panel.  Top-level Rinv12 skipped (complete_inv = 0 and the top
// node splits at s1): the block formula with R12 (the reference's cacqr::solve, cacqr.hpp:44-73)
//   Y1 = Rinv11^T B1,  Y2 = Rinv22^T (B2 - R12^T Y1),  X2 = Rinv22 Y2,  X1 = Rinv11 (Y1 - R12 X2),
// whose first three steps are Y = R^-T B and whose last three are X = R^-1 Y.  A half alone runs exactly the solve's steps of that half,
// through the same panel intermediate T, so applying both halves in turn gives the solve's bits.  SOLVE_R / SOLVE_RT (X = R B, X = R^T B)
// read only R: one pass over its triangle per panel, B copied into T first.
static capital_status_t cholinv_solve_mode(capital_ctx* ctx, int64_t n, const capital_cholinv_args_t* args, capital_structure_t structure,
                                           const double* R_local, const double* Rinv_local, int64_t nrhs, const double* B, int64_t ldb,
                                           double* X, int64_t ldx, int mode, const char* what) {
  const bool apply_r = mode == SOLVE_R || mode == SOLVE_RT;
  if (!args || (apply_r ? !R_local : !Rinv_local) || !B || !X || n <= 0 || nrhs < 1 || ldb < n || ldx < n || args->split <= 0 ||
      args->dir != 'U' || (structure != CAPITAL_RECT && structure != CAPITAL_UPPERTRI_PACKED)) {
    ctx->set_error(std::string("cholinv::") + what + ": invalid arguments (" + (apply_r ? "R" : "Rinv") +
                   ", B, X non-null, nrhs >= 1, ldb, ldx >= n, split > 0 and dir == 'U')");
    return CAPITAL_ERR_INVALID;
  }
  CAP_CUDA(cudaSetDevice(ctx->device));
  const capital_grid_t& g = ctx->grid;
  if (g.size > 1) return dist_cholinv_solve(ctx, n, args, structure, R_local, Rinv_local, nrhs, B, ldb, X, ldx, mode);
  const int64_t L = n;
  const int64_t bc = capital_cholinv_bc_dimension(L, g.c, g.d, args->bc_mult_dim);
  const bool skipped = !apply_r && args->complete_inv == 0 && cholinv_node_splits(L, bc, (int)args->split);
  if (skipped && !R_local) {
    ctx->set_error(std::string("cholinv::") + what + ": the top-level Rinv12 block was skipped (complete_inv = 0), R is needed");
    return CAPITAL_ERR_INVALID;
  }
  const int64_t s1 = L >> args->split;
  const bool packed = structure == CAPITAL_UPPERTRI_PACKED;
  const size_t f_count = packed ? (size_t)L * (L + 1) / 2 : (size_t)L * L;
  const int64_t ldu = packed ? 0 : L;
  cudaStream_t st = ctx->stream;
  const double *dRi = nullptr, *dR = nullptr, *dB;
  if (!apply_r) CAP_TRY(cap_stage_in(ctx, Rinv_local, f_count, "solve_Rinv", &dRi));
  if (skipped || apply_r) CAP_TRY(cap_stage_in(ctx, R_local, f_count, "solve_R", &dR));
  CAP_TRY(cap_stage_in(ctx, B, (size_t)ldb * (nrhs - 1) + n, "solve_B", &dB));
  const bool x_host = !cap_is_device_ptr(X);
  double* dX = X;
  if (x_host) CAP_TRY(ctx->workspace("solve_X", (size_t)ldx * nrhs * 8, (void**)&dX));
  double *T, *T2;  // panel intermediates, L x SOLVE_W
  CAP_TRY(ctx->workspace("solve_T", (size_t)L * SOLVE_W * 8, (void**)&T));
  CAP_TRY(ctx->workspace("solve_T2", (size_t)L * SOLVE_W * 8, (void**)&T2));
  // first half: T = R^-T Bp
  auto half_t = [&](const double* Bp, int64_t w) -> capital_status_t {
    //                 U    ldu  trans r0  r1  c0  c1  nrhs alpha P  pinc ldp   beta Cin     ldcin C   cinc ldc
    if (!skipped) return tri_apply(ctx, st, {dRi, ldu, true, 0, L, 0, L, w, 1.0, Bp, 1, ldb, 0.0, nullptr, 0, T, 1, L});  // Y = Rinv^T B
    CAP_TRY(tri_apply(ctx, st, {dRi, ldu, true, 0, s1, 0, s1, w, 1.0, Bp, 1, ldb, 0.0, nullptr, 0, T, 1, L}));   // T1 = Y1
    CAP_TRY(tri_apply(ctx, st, {dR, ldu, true, 0, s1, s1, L, w, -1.0, T, 1, L, 1.0, Bp, ldb, T2, 1, L}));       // T2_2 = B2 - R12^T Y1
    return tri_apply(ctx, st, {dRi, ldu, true, s1, L, s1, L, w, 1.0, T2, 1, L, 0.0, nullptr, 0, T, 1, L});      // T2 = Y2
  };
  // second half: Xp = R^-1 T
  auto half_n = [&](double* Xp, int64_t w) -> capital_status_t {
    if (!skipped) return tri_apply(ctx, st, {dRi, ldu, false, 0, L, 0, L, w, 1.0, T, 1, L, 0.0, nullptr, 0, Xp, 1, ldx});  // X = Rinv Y
    CAP_TRY(tri_apply(ctx, st, {dRi, ldu, false, s1, L, s1, L, w, 1.0, T, 1, L, 0.0, nullptr, 0, Xp, 1, ldx})); // X2
    CAP_TRY(tri_apply(ctx, st, {dR, ldu, false, 0, s1, s1, L, w, -1.0, Xp, 1, ldx, 1.0, T, L, T2, 1, L}));      // T2_1 = Y1 - R12 X2
    return tri_apply(ctx, st, {dRi, ldu, false, 0, s1, 0, s1, w, 1.0, T2, 1, L, 0.0, nullptr, 0, Xp, 1, ldx});  // X1
  };
  // a half alone goes through T as well (B is copied in, or the result copied out), so X may alias B
  for (int64_t p0 = 0; p0 < nrhs; p0 += SOLVE_W) {
    const int64_t w = std::min<int64_t>(SOLVE_W, nrhs - p0);
    const double* Bp = dB + p0 * ldb;
    double* Xp = dX + p0 * ldx;
    if (apply_r) {
      CAP_TRY(panel_add(ctx, st, L, w, Bp, ldb, nullptr, 0, T, L));
      CAP_TRY(tri_apply(ctx, st, {dR, ldu, mode == SOLVE_RT, 0, L, 0, L, w, 1.0, T, 1, L, 0.0, nullptr, 0, Xp, 1, ldx}));  // R B, R^T B
      continue;
    }
    if (mode != SOLVE_RINV) CAP_TRY(half_t(Bp, w));
    else CAP_TRY(panel_add(ctx, st, L, w, Bp, ldb, nullptr, 0, T, L));
    if (mode != SOLVE_RINVT) CAP_TRY(half_n(Xp, w));
    else CAP_TRY(panel_add(ctx, st, L, w, T, L, nullptr, 0, Xp, ldx));
  }
  if (x_host) {  // only the n rows of each column travel: the caller's rows n .. ldx stay untouched
    CAP_CUDA(cudaMemcpy2DAsync(X, (size_t)ldx * 8, dX, (size_t)ldx * 8, (size_t)n * 8, (size_t)nrhs, cudaMemcpyDeviceToHost, st));
    ctx->counters.d2h_bytes += n * nrhs * 8;
    CAP_CUDA(cudaStreamSynchronize(st));
  }
  return CAPITAL_OK;
}

capital_status_t capital_cholinv_solve_f64(capital_ctx* ctx, int64_t n, const capital_cholinv_args_t* args, capital_structure_t structure,
                                           const double* R_local, const double* Rinv_local, int64_t nrhs, const double* B, int64_t ldb,
                                           double* X, int64_t ldx) {
  if (!ctx) return CAPITAL_ERR_INVALID;
  return cholinv_solve_mode(ctx, n, args, structure, R_local, Rinv_local, nrhs, B, ldb, X, ldx, SOLVE_FULL, "solve");
}

// X = R^-1 B (trans = 0: the back-transform of sygst) or X = R^-T B (trans = 1: whitening), each one half of the solve.
capital_status_t capital_cholinv_apply_rinv_f64(capital_ctx* ctx, int64_t n, const capital_cholinv_args_t* args, capital_structure_t structure,
                                                const double* R_local, const double* Rinv_local, int trans, int64_t nrhs, const double* B,
                                                int64_t ldb, double* X, int64_t ldx) {
  if (!ctx) return CAPITAL_ERR_INVALID;
  if (trans != 0 && trans != 1) {
    ctx->set_error("cholinv::apply_rinv: trans must be 0 (X = R^-1 B) or 1 (X = R^-T B)");
    return CAPITAL_ERR_INVALID;
  }
  return cholinv_solve_mode(ctx, n, args, structure, R_local, Rinv_local, nrhs, B, ldb, X, ldx, trans ? SOLVE_RINVT : SOLVE_RINV,
                            "apply_rinv");
}

// X = R B (trans = 0) or X = R^T B (trans = 1, the back-transform of sygst_ab for itype 3) with the factor's R.
capital_status_t capital_cholinv_apply_r_f64(capital_ctx* ctx, int64_t n, const capital_cholinv_args_t* args, capital_structure_t structure,
                                             const double* R_local, int trans, int64_t nrhs, const double* B, int64_t ldb, double* X,
                                             int64_t ldx) {
  if (!ctx) return CAPITAL_ERR_INVALID;
  if (trans != 0 && trans != 1) {
    ctx->set_error("cholinv::apply_r: trans must be 0 (X = R B) or 1 (X = R^T B)");
    return CAPITAL_ERR_INVALID;
  }
  return cholinv_solve_mode(ctx, n, args, structure, R_local, nullptr, nrhs, B, ldb, X, ldx, trans ? SOLVE_RT : SOLVE_R, "apply_r");
}

// ---- batched CholInv: many independent n x n matrices, n <= BASECASE_MAX, on this context's GPU ------------------------------------

static bool all_device(std::initializer_list<const void*> ptrs) {
  for (const void* p : ptrs)
    if (!cap_is_device_ptr(p)) return false;
  return true;
}

capital_status_t capital_cholinv_factor_batched_f64(capital_ctx* ctx, int64_t n, int64_t batch, const double* A, double* R, double* Rinv,
                                                    int* info) {
  if (!ctx) return CAPITAL_ERR_INVALID;
  if (!A || !R || !Rinv || !info || n < 1 || batch < 1) {
    ctx->set_error("cholinv::factor_batched: invalid arguments (A, R, Rinv, info non-null, n >= 1, batch >= 1)");
    return CAPITAL_ERR_INVALID;
  }
  if (n > BASECASE_MAX) {
    ctx->set_error("cholinv::factor_batched: n > 512 is not supported (factor each matrix with capital_cholinv_factor_f64)");
    return CAPITAL_ERR_UNSUPPORTED;
  }
  CAP_CUDA(cudaSetDevice(ctx->device));
  if (!all_device({A, R, Rinv, info})) {
    ctx->set_error("cholinv::factor_batched: A, R, Rinv and info must be device pointers");
    return CAPITAL_ERR_INVALID;
  }
  cudaStream_t st = ctx->stream;
  const int64_t nn = n * n;
  CAP_CUDA(cudaMemsetAsync(info, 0, (size_t)batch * sizeof(int), st));
  if (n <= LEAF_MAX) {  // one CTA per matrix, straight from A's upper triangle into the outputs: no workspace
    for (int64_t b0 = 0; b0 < batch; b0 += INT32_MAX) {
      const LeafBatch bt{std::min<int64_t>(INT32_MAX, batch - b0), {nn, nn, nn, 0}, info + b0, 0};
      CAP_TRY(leaf_cholinv(ctx, st, (int)n, A + b0 * nn, n, R + b0 * nn, n, Rinv + b0 * nn, n, nullptr, 0, &bt));
    }
    return CAPITAL_OK;
  }
  // the cluster kernel on nb = roundup(n, 64), identity pad; R and Rinv straight into the outputs when no pad is needed and they are
  // 16-byte aligned (the kernel's 16-byte accesses; n is even then, so every matrix of the batch is aligned too)
  const int64_t nb = round_up(n, 64), mm = nb * nb;
  const bool direct = nb == n && (((uintptr_t)R | (uintptr_t)Rinv) & 15) == 0;
  const int64_t chunk = std::min<int64_t>({batch, 65535, (int64_t)(BATCHED_WORKSPACE_CAP / ((direct ? 2 : 4) * mm * 8))});
  double *W, *RiT, *Rw = nullptr, *Riw = nullptr;
  CAP_TRY(ctx->workspace("batched_W", (size_t)(chunk * mm) * 8, (void**)&W));
  CAP_TRY(ctx->workspace("batched_RiT", (size_t)(chunk * mm) * 8, (void**)&RiT));
  if (!direct) {
    CAP_TRY(ctx->workspace("batched_R", (size_t)(chunk * mm) * 8, (void**)&Rw));
    CAP_TRY(ctx->workspace("batched_Ri", (size_t)(chunk * mm) * 8, (void**)&Riw));
  }
  const int cw = batched_cluster_width(nb);
  for (int64_t b0 = 0; b0 < batch; b0 += chunk) {
    const int64_t cnt = std::min(chunk, batch - b0);
    CAP_TRY(sym_pad_batched(ctx, st, n, nb, cnt, A + b0 * nn, W));
    if (direct) {
      CAP_CUDA(cudaMemsetAsync(Rinv + b0 * nn, 0, (size_t)(cnt * nn) * 8, st));  // the kernel never writes Rinv's lower blocks
      const LeafBatch bt{cnt, {mm, nn, nn, mm}, info + b0, cw};
      CAP_TRY(basecase_cholinv(ctx, st, (int)nb, W, nb, R + b0 * nn, n, Rinv + b0 * nn, n, RiT, nb, &bt));
    } else {
      const LeafBatch bt{cnt, {mm, mm, mm, mm}, info + b0, cw};
      CAP_TRY(basecase_cholinv(ctx, st, (int)nb, W, nb, Rw, nb, Riw, nb, RiT, nb, &bt));
      CAP_TRY(triu_out_batched(ctx, st, n, cnt, Rw, nb, mm, R + b0 * nn, n, nn));
      CAP_TRY(triu_out_batched(ctx, st, n, cnt, Riw, nb, mm, Rinv + b0 * nn, n, nn));
    }
  }
  return CAPITAL_OK;
}

capital_status_t capital_cholinv_solve_batched_f64(capital_ctx* ctx, int64_t n, int64_t batch, const double* Rinv, int64_t nrhs,
                                                   const double* B, double* X) {
  if (!ctx) return CAPITAL_ERR_INVALID;
  if (!Rinv || !B || !X || n < 1 || batch < 1 || nrhs < 1) {
    ctx->set_error("cholinv::solve_batched: invalid arguments (Rinv, B, X non-null, n >= 1, batch >= 1, nrhs >= 1)");
    return CAPITAL_ERR_INVALID;
  }
  if (n > BASECASE_MAX) {
    ctx->set_error("cholinv::solve_batched: n > 512 is not supported");
    return CAPITAL_ERR_UNSUPPORTED;
  }
  CAP_CUDA(cudaSetDevice(ctx->device));
  if (!all_device({Rinv, B, X})) {
    ctx->set_error("cholinv::solve_batched: Rinv, B and X must be device pointers");
    return CAPITAL_ERR_INVALID;
  }
  cudaStream_t st = ctx->stream;
  const int64_t nn = n * n, nbk = n * nrhs, ts = n * SOLVE_W;
  // per matrix: the panel intermediate T and tri_apply's partials (one k chunk per 64-row block: n <= 1024)
  const int64_t per = (ts + round_up(n, 64) * SOLVE_W) * 8;
  const int64_t chunk = std::min<int64_t>({batch, 65535, (int64_t)(BATCHED_WORKSPACE_CAP / per)});
  double* T;
  CAP_TRY(ctx->workspace("batched_T", (size_t)(chunk * ts) * 8, (void**)&T));
  for (int64_t b0 = 0; b0 < batch; b0 += chunk) {
    const int64_t cnt = std::min(chunk, batch - b0);
    const double* U = Rinv + b0 * nn;
    for (int64_t p0 = 0; p0 < nrhs; p0 += SOLVE_W) {
      const int64_t w = std::min<int64_t>(SOLVE_W, nrhs - p0);
      const double* Bp = B + b0 * nbk + p0 * n;
      double* Xp = X + b0 * nbk + p0 * n;
      // X may alias B: every matrix's panel of B is read into T before its panel of X is written
      //                 U  ldu trans r0 r1 c0 c1 nrhs alpha P  pinc ldp beta Cin   ldcin C  cinc ldc full  batch su  sp   scin sc
      CAP_TRY(tri_apply(ctx, st, {U, n, true, 0, n, 0, n, w, 1.0, Bp, 1, n, 0.0, nullptr, 0, T, 1, n, false, cnt, nn, nbk, 0, ts}));  // T = Rinv^T B
      CAP_TRY(tri_apply(ctx, st, {U, n, false, 0, n, 0, n, w, 1.0, T, 1, n, 0.0, nullptr, 0, Xp, 1, n, false, cnt, nn, ts, 0, nbk}));  // X = Rinv T
    }
  }
  return CAPITAL_OK;
}

// Do the byte ranges of a[0, na) and b[0, nb), two arrays of doubles, overlap?
static bool overlaps(const double* a, size_t na, const double* b, size_t nb) {
  if (!a || !b) return false;
  const uintptr_t pa = (uintptr_t)a, pb = (uintptr_t)b;
  return pa < pb + nb * 8 && pb < pa + na * 8;
}

// The top-level Rinv12 block that the factor skipped (complete_inv = 0, top node split at s1), rebuilt in Ri with the two products the
// factor issues for it (cholinv_local.cu), with the same kernel, flags and shapes: T^T = R12^T Rinv11^T into W's lower-left block, then
// Rinv12 = -(T^T)^T Rinv22.  RiT holds Rinv11^T on entry; on return its lower-left block holds Rinv12^T.  R is staged in and unpacked
// into the factor's workspace "Rm".
static capital_status_t rebuild_rinv12(capital_ctx* ctx, cudaStream_t st, int64_t L, int split, bool packed, const double* R_local,
                                       size_t count, double* Ri, double* RiT, double* W, int64_t ld) {
  const int64_t s1 = L >> split, s2 = L - s1;
  const double* dR;
  double* Rm;
  CAP_TRY(ctx->workspace("Rm", (size_t)ld * L * 8, (void**)&Rm));
  CAP_TRY(cap_stage_in(ctx, R_local, count, "R_out", &dR));
  if (packed) CAP_TRY(unpack_upper(ctx, st, L, dR, Rm, ld));
  else CAP_TRY(triu_copy(ctx, st, L, dR, L, Rm, ld, 0));
  CAP_TRY(gemm_tn(ctx, st, s2, s1, s1, 1.0, Rm + s1 * ld, ld, RiT, ld, 0.0, W + s1, ld, CAPITAL_GEMM_B_LOWER));                     // T^T
  CAP_TRY(gemm_tn(ctx, st, s1, s2, s2, -1.0, W + s1, ld, Ri + s1 * ld + s1, ld, 0.0, Ri + s1 * ld, ld, CAPITAL_GEMM_B_UPPER));  // Rinv12
  return transpose_block(ctx, st, s1, s2, Ri + s1 * ld, ld, RiT + s1, ld, 1.0);
}

// A^-1 = Rinv Rinv^T from the factor's outputs: one DMMA product of Rinv^T (lower) with itself, upper tiles only, tile (i, j) running
// k from max(i, j) -- n^3 / 3 flops.  Where the factor skipped the top-level Rinv12 (complete_inv = 0 and the top node splits at s1),
// it is rebuilt first with the two products the factor issues for that block (cholinv_local.cu): T^T = R12^T Rinv11^T, then
// Rinv12 = -(T^T)^T Rinv22, with the same kernel, flags and shapes.  The only buffers are the factor's own workspaces.
capital_status_t capital_cholinv_inverse_f64(capital_ctx* ctx, int64_t n, const capital_cholinv_args_t* args, capital_structure_t structure,
                                             const double* R_local, const double* Rinv_local, double* Ainv_local) {
  if (!ctx) return CAPITAL_ERR_INVALID;
  const bool packed = structure == CAPITAL_UPPERTRI_PACKED;
  const int64_t Lc = n > 0 ? ceil_div(n, std::max(ctx->grid.d, 1)) : 0;
  const size_t count = packed ? (size_t)Lc * (Lc + 1) / 2 : (size_t)Lc * Lc;
  if (!args || !Rinv_local || !Ainv_local || n <= 0 || args->split <= 0 || args->dir != 'U' ||
      (structure != CAPITAL_RECT && structure != CAPITAL_UPPERTRI_PACKED) || overlaps(Ainv_local, count, Rinv_local, count) ||
      overlaps(Ainv_local, count, R_local, count)) {
    ctx->set_error("cholinv::inverse: invalid arguments (Rinv and Ainv non-null, Ainv not overlapping R or Rinv, split > 0 and dir == 'U', "
                   "packed upper or rect)");
    return CAPITAL_ERR_INVALID;
  }
  CAP_CUDA(cudaSetDevice(ctx->device));
  const capital_grid_t& g = ctx->grid;
  if (g.size > 1) return dist_cholinv_inverse(ctx, n, args, structure, R_local, Rinv_local, Ainv_local);
  const int64_t L = n, ld = round_up(L, 16);
  const int64_t bc = capital_cholinv_bc_dimension(L, g.c, g.d, args->bc_mult_dim);
  const bool skipped = args->complete_inv == 0 && cholinv_node_splits(L, bc, (int)args->split);
  if (skipped && !R_local) {
    ctx->set_error("cholinv::inverse: the top-level Rinv12 block was skipped (complete_inv = 0), R is needed");
    return CAPITAL_ERR_INVALID;
  }
  cudaStream_t st = ctx->stream;
  double *W, *Ri, *RiT, *dOut;
  CAP_TRY(ctx->workspace("W", (size_t)ld * L * 8, (void**)&W));
  CAP_TRY(ctx->workspace("Ri", (size_t)ld * L * 8, (void**)&Ri));
  CAP_TRY(ctx->workspace("RiT", (size_t)ld * L * 8, (void**)&RiT));
  // host inputs are staged in the factor's own output buffers; a host output reuses R's once R has been unpacked
  const double* dRi;
  CAP_TRY(cap_stage_in(ctx, Rinv_local, count, "Rinv_out", &dRi));
  if (packed) CAP_TRY(unpack_upper(ctx, st, L, dRi, Ri, ld));
  else CAP_TRY(triu_copy(ctx, st, L, dRi, L, Ri, ld, 0));
  CAP_TRY(transpose_block(ctx, st, L, L, Ri, ld, RiT, ld, 1.0));  // Rinv^T: lower, exact zeros above the diagonal
  if (skipped) CAP_TRY(rebuild_rinv12(ctx, st, L, (int)args->split, packed, R_local, count, Ri, RiT, W, ld));
  // upper tiles of (Rinv^T)^T Rinv^T; the lower-left T^T scratch in W is overwritten or never read
  CAP_TRY(gemm_tn(ctx, st, L, L, L, 1.0, RiT, ld, RiT, ld, 0.0, W, ld,
                  CAPITAL_GEMM_A_LOWER | CAPITAL_GEMM_B_LOWER | CAPITAL_GEMM_C_UPPER));
  CAP_TRY(cap_stage_out_begin(ctx, Ainv_local, count, "R_out", &dOut));
  if (packed) CAP_TRY(pack_upper(ctx, st, L, W, ld, dOut, 0));
  else CAP_TRY(sym_merge(ctx, st, L, W, ld, W, ld, true, dOut, L, 0, 0, 1));  // the lower half is the upper one's mirror, bit for bit
  if (dOut != Ainv_local) {
    CAP_TRY(cap_stage_out_end(ctx, Ainv_local, count, dOut));
    CAP_CUDA(cudaStreamSynchronize(st));
  }
  return CAPITAL_OK;
}

// A x = lambda B x with B = R^T R reduced to C y = lambda y, C = Rinv^T A Rinv (LAPACK dsygst, itype 1), in n^3 DMMA flops by LAPACK's
// split A = U + U^T, U = triu(A) with its diagonal halved, C = M + M^T with M = Rinv^T U Rinv:
//   V = U Rinv = (U^T)^T Rinv                 A_LOWER | B_UPPER | C_UPPER   n^3 / 3   (upper triangular: two upper factors)
//   C_upper = Rinv^T V + V^T Rinv             A_UPPER | B_UPPER | C_UPPER   2 n^3 / 3, one launch with two operand classes
// U^T is A's lower triangle with its diagonal halved (exact), so only that triangle of A is read.  A skipped top-level Rinv12 is rebuilt
// first, as the inverse does.  The only buffers are the factor's four workspaces: Ri = Rinv, RiT = U^T (Rinv11^T for a rebuild first),
// W = V (zeroed: the C_UPPER product leaves the strict lower part of its diagonal tiles unwritten, and the next product reads whole
// diagonal tiles), Rm = C (R for a rebuild first).
capital_status_t capital_cholinv_sygst_f64(capital_ctx* ctx, int64_t n, const capital_cholinv_args_t* args, capital_structure_t structure,
                                           const double* R_local, const double* Rinv_local, const double* A_local, double* C_local) {
  if (!ctx) return CAPITAL_ERR_INVALID;
  const bool packed = structure == CAPITAL_UPPERTRI_PACKED;
  const int64_t Lc = n > 0 ? ceil_div(n, std::max(ctx->grid.d, 1)) : 0;
  const size_t count = packed ? (size_t)Lc * (Lc + 1) / 2 : (size_t)Lc * Lc, a_count = (size_t)Lc * Lc;
  if (!args || !Rinv_local || !A_local || !C_local || n <= 0 || args->split <= 0 || args->dir != 'U' ||
      (structure != CAPITAL_RECT && structure != CAPITAL_UPPERTRI_PACKED) || overlaps(C_local, count, Rinv_local, count) ||
      overlaps(C_local, count, R_local, count) || overlaps(C_local, count, A_local, a_count)) {
    ctx->set_error("cholinv::sygst: invalid arguments (Rinv, A and C non-null, C not overlapping A, R or Rinv, split > 0 and dir == 'U', "
                   "packed upper or rect)");
    return CAPITAL_ERR_INVALID;
  }
  CAP_CUDA(cudaSetDevice(ctx->device));
  const capital_grid_t& g = ctx->grid;
  if (g.size > 1) return dist_cholinv_sygst(ctx, n, args, structure, R_local, Rinv_local, A_local, C_local);
  const int64_t L = n, ld = round_up(L, 16);
  const int64_t bc = capital_cholinv_bc_dimension(L, g.c, g.d, args->bc_mult_dim);
  const bool skipped = args->complete_inv == 0 && cholinv_node_splits(L, bc, (int)args->split);
  if (skipped && !R_local) {
    ctx->set_error("cholinv::sygst: the top-level Rinv12 block was skipped (complete_inv = 0), R is needed");
    return CAPITAL_ERR_INVALID;
  }
  cudaStream_t st = ctx->stream;
  double *W, *Ri, *RiT, *Cm, *dOut;
  CAP_TRY(ctx->workspace("W", (size_t)ld * L * 8, (void**)&W));
  CAP_TRY(ctx->workspace("Ri", (size_t)ld * L * 8, (void**)&Ri));
  CAP_TRY(ctx->workspace("RiT", (size_t)ld * L * 8, (void**)&RiT));
  const double* dRi;
  CAP_TRY(cap_stage_in(ctx, Rinv_local, count, "Rinv_out", &dRi));
  if (packed) CAP_TRY(unpack_upper(ctx, st, L, dRi, Ri, ld));
  else CAP_TRY(triu_copy(ctx, st, L, dRi, L, Ri, ld, 0));
  if (skipped) {
    const int64_t s1 = L >> args->split;
    CAP_TRY(transpose_block(ctx, st, s1, s1, Ri, ld, RiT, ld, 1.0));  // Rinv11^T, the rebuild's only use of RiT's upper-left block
    CAP_TRY(rebuild_rinv12(ctx, st, L, (int)args->split, packed, R_local, count, Ri, RiT, W, ld));
  }
  CAP_TRY(ctx->workspace("Rm", (size_t)ld * L * 8, (void**)&Cm));
  const double* dA;
  CAP_TRY(cap_stage_in(ctx, A_local, a_count, "A_in", &dA));
  CAP_TRY(tril_half_copy(ctx, st, L, dA, L, RiT, ld, 0, 0, 1));  // U^T
  CAP_CUDA(cudaMemsetAsync(W, 0, (size_t)ld * L * 8, st));
  CAP_TRY(gemm_tn(ctx, st, L, L, L, 1.0, RiT, ld, Ri, ld, 0.0, W, ld, CAPITAL_GEMM_A_LOWER | CAPITAL_GEMM_B_UPPER | CAPITAL_GEMM_C_UPPER));
  GemmOperands ops;
  ops.ncls = 2; ops.lda = ops.ldb = ld;
  ops.A[0] = Ri; ops.B[0] = W;  // Rinv^T V
  ops.A[1] = W; ops.B[1] = Ri;  // V^T Rinv
  CAP_TRY(gemm_tn_x(ctx, st, L, L, L, 1.0, ops, 0.0, Cm, ld, CAPITAL_GEMM_A_UPPER | CAPITAL_GEMM_B_UPPER | CAPITAL_GEMM_C_UPPER, 0, nullptr));
  CAP_TRY(cap_stage_out_begin(ctx, C_local, count, "R_out", &dOut));
  if (packed) CAP_TRY(pack_upper(ctx, st, L, Cm, ld, dOut, 0));
  else CAP_TRY(sym_merge(ctx, st, L, Cm, ld, Cm, ld, true, dOut, L, 0, 0, 1));  // the lower half is the upper one's mirror, bit for bit
  if (dOut != C_local) {
    CAP_TRY(cap_stage_out_end(ctx, C_local, count, dOut));
    CAP_CUDA(cudaStreamSynchronize(st));
  }
  return CAPITAL_OK;
}

// A B x = lambda x (itype 2) and B A x = lambda x (itype 3) with B = R^T R, both reduced to C y = lambda y with C = R A R^T (LAPACK
// dsygst, itype 2 / 3, upper), in n^3 DMMA flops by the split of itype 1, A = U + U^T, C = M + M^T with M = R U R^T:
//   W = R U = (R^T)^T U                        A_LOWER | B_UPPER | C_UPPER   n^3 / 3   (upper triangular: two upper factors)
//   C_upper = (W^T)^T R^T + (R^T)^T W^T        A_LOWER | B_LOWER | C_UPPER   2 n^3 / 3, one launch with two operand classes
// Only R is read, never Rinv, so a skipped top-level Rinv12 changes nothing.  U is the transpose of tril_half_copy's U^T, so only A's
// lower triangle is read.  The only buffers are the factor's four workspaces: Ri = R, then U, then W^T; RiT = R^T; W = U^T, then W
// (zeroed: the C_UPPER product leaves the strict lower part of its diagonal tiles unwritten, and W^T's diagonal tiles are read whole);
// Rm = C.
capital_status_t capital_cholinv_sygst_ab_f64(capital_ctx* ctx, int64_t n, const capital_cholinv_args_t* args, capital_structure_t structure,
                                              const double* R_local, const double* A_local, double* C_local) {
  if (!ctx) return CAPITAL_ERR_INVALID;
  const bool packed = structure == CAPITAL_UPPERTRI_PACKED;
  const int64_t Lc = n > 0 ? ceil_div(n, std::max(ctx->grid.d, 1)) : 0;
  const size_t count = packed ? (size_t)Lc * (Lc + 1) / 2 : (size_t)Lc * Lc, a_count = (size_t)Lc * Lc;
  if (!args || !R_local || !A_local || !C_local || n <= 0 || args->split <= 0 || args->dir != 'U' ||
      (structure != CAPITAL_RECT && structure != CAPITAL_UPPERTRI_PACKED) || overlaps(C_local, count, R_local, count) ||
      overlaps(C_local, count, A_local, a_count)) {
    ctx->set_error("cholinv::sygst_ab: invalid arguments (R, A and C non-null, C not overlapping A or R, split > 0 and dir == 'U', "
                   "packed upper or rect)");
    return CAPITAL_ERR_INVALID;
  }
  CAP_CUDA(cudaSetDevice(ctx->device));
  const capital_grid_t& g = ctx->grid;
  if (g.size > 1) return dist_cholinv_sygst_ab(ctx, n, args, structure, R_local, A_local, C_local);
  const int64_t L = n, ld = round_up(L, 16);
  cudaStream_t st = ctx->stream;
  double *W, *Ri, *RiT, *Cm, *dOut;
  CAP_TRY(ctx->workspace("W", (size_t)ld * L * 8, (void**)&W));
  CAP_TRY(ctx->workspace("Ri", (size_t)ld * L * 8, (void**)&Ri));
  CAP_TRY(ctx->workspace("RiT", (size_t)ld * L * 8, (void**)&RiT));
  CAP_TRY(ctx->workspace("Rm", (size_t)ld * L * 8, (void**)&Cm));
  // a host R is staged in the factor's R output buffer, which a host C reuses once R has been unpacked
  const double *dR, *dA;
  CAP_TRY(cap_stage_in(ctx, R_local, count, "R_out", &dR));
  if (packed) CAP_TRY(unpack_upper(ctx, st, L, dR, Ri, ld));
  else CAP_TRY(triu_copy(ctx, st, L, dR, L, Ri, ld, 0));
  CAP_TRY(transpose_block(ctx, st, L, L, Ri, ld, RiT, ld, 1.0));  // R^T: lower, exact zeros above the diagonal
  CAP_TRY(cap_stage_in(ctx, A_local, a_count, "A_in", &dA));
  CAP_TRY(tril_half_copy(ctx, st, L, dA, L, W, ld, 0, 0, 1));      // U^T
  CAP_TRY(transpose_block(ctx, st, L, L, W, ld, Ri, ld, 1.0));     // U
  CAP_CUDA(cudaMemsetAsync(W, 0, (size_t)ld * L * 8, st));
  CAP_TRY(gemm_tn(ctx, st, L, L, L, 1.0, RiT, ld, Ri, ld, 0.0, W, ld, CAPITAL_GEMM_A_LOWER | CAPITAL_GEMM_B_UPPER | CAPITAL_GEMM_C_UPPER));
  CAP_TRY(transpose_block(ctx, st, L, L, W, ld, Ri, ld, 1.0));     // W^T: lower, exact zeros above the diagonal
  GemmOperands ops;
  ops.ncls = 2; ops.lda = ops.ldb = ld;
  ops.A[0] = Ri; ops.B[0] = RiT;  // W R^T
  ops.A[1] = RiT; ops.B[1] = Ri;  // R W^T
  CAP_TRY(gemm_tn_x(ctx, st, L, L, L, 1.0, ops, 0.0, Cm, ld, CAPITAL_GEMM_A_LOWER | CAPITAL_GEMM_B_LOWER | CAPITAL_GEMM_C_UPPER, 0, nullptr));
  CAP_TRY(cap_stage_out_begin(ctx, C_local, count, "R_out", &dOut));
  if (packed) CAP_TRY(pack_upper(ctx, st, L, Cm, ld, dOut, 0));
  else CAP_TRY(sym_merge(ctx, st, L, Cm, ld, Cm, ld, true, dOut, L, 0, 0, 1));  // the lower half is the upper one's mirror, bit for bit
  if (dOut != C_local) {
    CAP_TRY(cap_stage_out_end(ctx, C_local, count, dOut));
    CAP_CUDA(cudaStreamSynchronize(st));
  }
  return CAPITAL_OK;
}

// ---- batched inverse, sygst and products with the factors: the single-GPU sequences above, run over a chunk of matrices ----------------
// Every matrix lives in the workspace as the single call lays it out (ld = round_up(n, 16), n columns) at a stride of ld n, so each pass
// and product of the single call becomes one batched launch with the same flags, k ranges and class order: every matrix gets the
// single call's bits on the same factors.  Chunks of at most 65535 matrices whose intermediates fit BATCHED_WORKSPACE_CAP.

// The arguments every batched entry point shares: non-null, n in [1, 512], batch >= 1, device pointers.
static capital_status_t batched_args(capital_ctx* ctx, const char* what, const char* names, int64_t n, int64_t batch,
                                     std::initializer_list<const void*> ptrs, bool extra_ok = true, const char* extra = "") {
  bool null = false;
  for (const void* p : ptrs) null = null || !p;
  if (null || n < 1 || batch < 1 || !extra_ok) {
    ctx->set_error(std::string("cholinv::") + what + ": invalid arguments (" + names + " non-null, n >= 1, batch >= 1" + extra + ")");
    return CAPITAL_ERR_INVALID;
  }
  if (n > BASECASE_MAX) {
    ctx->set_error(std::string("cholinv::") + what + ": n > 512 is not supported");
    return CAPITAL_ERR_UNSUPPORTED;
  }
  CAP_CUDA(cudaSetDevice(ctx->device));
  if (!all_device(ptrs)) {
    ctx->set_error(std::string("cholinv::") + what + ": " + names + " must be device pointers");
    return CAPITAL_ERR_INVALID;
  }
  return CAPITAL_OK;
}

// matrices per chunk when each holds `per_matrix` bytes of intermediates
static int64_t batched_chunk(int64_t batch, int64_t per_matrix) {
  return std::min<int64_t>({batch, 65535, (int64_t)(BATCHED_WORKSPACE_CAP / per_matrix)});
}

// The workspace of the batched inverse and sygst: `count` buffers of chunk x ld x n doubles, under the batched factor's names (the two
// calls never run at once, so they share the memory).
static capital_status_t batched_buffers(capital_ctx* ctx, int64_t chunk, int64_t s, int count, double** out) {
  static const char* names[4] = {"batched_Ri", "batched_RiT", "batched_W", "batched_R"};
  for (int i = 0; i < count; i++) CAP_TRY(ctx->workspace(names[i], (size_t)(chunk * s) * 8, (void**)&out[i]));
  return CAPITAL_OK;
}

static GemmBatchOps batch_ops(int64_t cnt, const double* A, const double* B, int64_t ld, int64_t s) {
  GemmBatchOps g;
  g.batch = cnt; g.A = A; g.B = B; g.lda = g.ldb = ld; g.sa = g.sb = g.sc = s;
  return g;
}

capital_status_t capital_cholinv_inverse_batched_f64(capital_ctx* ctx, int64_t n, int64_t batch, const double* Rinv, double* Ainv) {
  if (!ctx) return CAPITAL_ERR_INVALID;
  CAP_TRY(batched_args(ctx, "inverse_batched", "Rinv, Ainv", n, batch, {Rinv, Ainv}));
  const int64_t nn = n * n, ld = round_up(n, 16), s = ld * n;
  if (overlaps(Ainv, (size_t)(batch * nn), Rinv, (size_t)(batch * nn))) {
    ctx->set_error("cholinv::inverse_batched: Ainv must not overlap Rinv");
    return CAPITAL_ERR_INVALID;
  }
  cudaStream_t st = ctx->stream;
  const int64_t chunk = batched_chunk(batch, 3 * s * 8);
  double* w[3];
  CAP_TRY(batched_buffers(ctx, chunk, s, 3, w));
  double *Ri = w[0], *RiT = w[1], *W = w[2];
  for (int64_t b0 = 0; b0 < batch; b0 += chunk) {
    const int64_t cnt = std::min(chunk, batch - b0);
    CAP_TRY(triu_out_batched(ctx, st, n, cnt, Rinv + b0 * nn, n, nn, Ri, ld, s));
    CAP_TRY(transpose_batched(ctx, st, n, n, cnt, Ri, ld, s, RiT, ld, s));  // Rinv^T: lower, exact zeros above the diagonal
    CAP_TRY(gemm_tn_batched(ctx, st, n, n, n, 1.0, batch_ops(cnt, RiT, RiT, ld, s), W, ld, nullptr, 0,
                            CAPITAL_GEMM_A_LOWER | CAPITAL_GEMM_B_LOWER | CAPITAL_GEMM_C_UPPER, false));
    CAP_TRY(sym_merge_batched(ctx, st, n, cnt, W, ld, s, Ainv + b0 * nn, n, nn));
  }
  return CAPITAL_OK;
}

capital_status_t capital_cholinv_sygst_batched_f64(capital_ctx* ctx, int64_t n, int64_t batch, const double* Rinv, const double* A,
                                                   double* C) {
  if (!ctx) return CAPITAL_ERR_INVALID;
  CAP_TRY(batched_args(ctx, "sygst_batched", "Rinv, A, C", n, batch, {Rinv, A, C}));
  const int64_t nn = n * n, ld = round_up(n, 16), s = ld * n;
  const size_t all = (size_t)(batch * nn);
  if (overlaps(C, all, Rinv, all) || overlaps(C, all, A, all)) {
    ctx->set_error("cholinv::sygst_batched: C must not overlap Rinv or A");
    return CAPITAL_ERR_INVALID;
  }
  cudaStream_t st = ctx->stream;
  const int64_t chunk = batched_chunk(batch, 4 * s * 8);
  double* w[4];
  CAP_TRY(batched_buffers(ctx, chunk, s, 4, w));
  double *Ri = w[0], *UT = w[1], *V = w[2], *Cm = w[3];
  for (int64_t b0 = 0; b0 < batch; b0 += chunk) {
    const int64_t cnt = std::min(chunk, batch - b0);
    CAP_TRY(triu_out_batched(ctx, st, n, cnt, Rinv + b0 * nn, n, nn, Ri, ld, s));
    CAP_TRY(tril_half_batched(ctx, st, n, cnt, A + b0 * nn, n, nn, UT, ld, s));  // U^T
    CAP_CUDA(cudaMemsetAsync(V, 0, (size_t)(cnt * s) * 8, st));
    CAP_TRY(gemm_tn_batched(ctx, st, n, n, n, 1.0, batch_ops(cnt, UT, Ri, ld, s), V, ld, nullptr, 0,
                            CAPITAL_GEMM_A_LOWER | CAPITAL_GEMM_B_UPPER | CAPITAL_GEMM_C_UPPER, false));  // V = U Rinv
    GemmBatchOps g = batch_ops(cnt, Ri, V, ld, s);  // Rinv^T V
    g.ncls = 2; g.A1 = V; g.B1 = Ri;                // + V^T Rinv
    CAP_TRY(gemm_tn_batched(ctx, st, n, n, n, 1.0, g, Cm, ld, nullptr, 0, CAPITAL_GEMM_A_UPPER | CAPITAL_GEMM_B_UPPER | CAPITAL_GEMM_C_UPPER,
                            false));
    CAP_TRY(sym_merge_batched(ctx, st, n, cnt, Cm, ld, s, C + b0 * nn, n, nn));
  }
  return CAPITAL_OK;
}

capital_status_t capital_cholinv_sygst_ab_batched_f64(capital_ctx* ctx, int64_t n, int64_t batch, const double* R, const double* A,
                                                      double* C) {
  if (!ctx) return CAPITAL_ERR_INVALID;
  CAP_TRY(batched_args(ctx, "sygst_ab_batched", "R, A, C", n, batch, {R, A, C}));
  const int64_t nn = n * n, ld = round_up(n, 16), s = ld * n;
  const size_t all = (size_t)(batch * nn);
  if (overlaps(C, all, R, all) || overlaps(C, all, A, all)) {
    ctx->set_error("cholinv::sygst_ab_batched: C must not overlap R or A");
    return CAPITAL_ERR_INVALID;
  }
  cudaStream_t st = ctx->stream;
  const int64_t chunk = batched_chunk(batch, 4 * s * 8);
  double* w[4];
  CAP_TRY(batched_buffers(ctx, chunk, s, 4, w));
  double *Ri = w[0], *RT = w[1], *W = w[2], *Cm = w[3];  // Ri: R, then U, then W^T (as in the single call)
  for (int64_t b0 = 0; b0 < batch; b0 += chunk) {
    const int64_t cnt = std::min(chunk, batch - b0);
    CAP_TRY(triu_out_batched(ctx, st, n, cnt, R + b0 * nn, n, nn, Ri, ld, s));
    CAP_TRY(transpose_batched(ctx, st, n, n, cnt, Ri, ld, s, RT, ld, s));       // R^T: lower, exact zeros above the diagonal
    CAP_TRY(tril_half_batched(ctx, st, n, cnt, A + b0 * nn, n, nn, W, ld, s));  // U^T
    CAP_TRY(transpose_batched(ctx, st, n, n, cnt, W, ld, s, Ri, ld, s));        // U
    CAP_CUDA(cudaMemsetAsync(W, 0, (size_t)(cnt * s) * 8, st));
    CAP_TRY(gemm_tn_batched(ctx, st, n, n, n, 1.0, batch_ops(cnt, RT, Ri, ld, s), W, ld, nullptr, 0,
                            CAPITAL_GEMM_A_LOWER | CAPITAL_GEMM_B_UPPER | CAPITAL_GEMM_C_UPPER, false));  // W = R U
    CAP_TRY(transpose_batched(ctx, st, n, n, cnt, W, ld, s, Ri, ld, s));        // W^T: lower, exact zeros above the diagonal
    GemmBatchOps g = batch_ops(cnt, Ri, RT, ld, s);  // W R^T
    g.ncls = 2; g.A1 = RT; g.B1 = Ri;                // + R W^T
    CAP_TRY(gemm_tn_batched(ctx, st, n, n, n, 1.0, g, Cm, ld, nullptr, 0, CAPITAL_GEMM_A_LOWER | CAPITAL_GEMM_B_LOWER | CAPITAL_GEMM_C_UPPER,
                            false));
    CAP_TRY(sym_merge_batched(ctx, st, n, cnt, Cm, ld, s, C + b0 * nn, n, nn));
  }
  return CAPITAL_OK;
}

// ---- batched symmetric eigensolver (syevj.cu) ---------------------------------------------------------------------------------------
capital_status_t capital_syevj_batched_f64(capital_ctx* ctx, int64_t n, int64_t batch, const double* A, double* w, double* V, int* info) {
  if (!ctx) return CAPITAL_ERR_INVALID;
  if (!A || !w || !V || !info || n < 1 || batch < 1) {
    ctx->set_error("syevj_batched: invalid arguments (A, w, V, info non-null, n >= 1, batch >= 1)");
    return CAPITAL_ERR_INVALID;
  }
  if (n > BASECASE_MAX) {
    ctx->set_error("syevj_batched: n > 512 is not supported");
    return CAPITAL_ERR_UNSUPPORTED;
  }
  CAP_CUDA(cudaSetDevice(ctx->device));
  if (!all_device({A, w, V, info})) {
    ctx->set_error("syevj_batched: A, w, V and info must be device pointers");
    return CAPITAL_ERR_INVALID;
  }
  const size_t nn = (size_t)(batch * n * n), nw = (size_t)(batch * n);
  if (overlaps(w, nw, A, nn) || overlaps(V, nn, A, nn) || overlaps(w, nw, V, nn) ||
      overlaps((const double*)info, ((size_t)batch + 1) / 2, A, nn) || overlaps((const double*)info, ((size_t)batch + 1) / 2, w, nw) ||
      overlaps((const double*)info, ((size_t)batch + 1) / 2, V, nn)) {
    ctx->set_error("syevj_batched: w, V and info must not overlap each other or A");
    return CAPITAL_ERR_INVALID;
  }
  return syevj_batched(ctx, ctx->stream, n, batch, A, w, V, info);
}

// X_b = op(U_b) B_b with U = R or Rinv: per panel of up to SOLVE_W right-hand sides, the panel of every matrix of the chunk is copied
// into T (so X may alias B), then one batched tri_apply pass over U, as the single call's apply does.
static capital_status_t apply_batched(capital_ctx* ctx, const char* what, const char* names, int64_t n, int64_t batch, const double* U,
                                      int trans, int64_t nrhs, const double* B, double* X) {
  CAP_TRY(batched_args(ctx, what, names, n, batch, {U, B, X}, nrhs >= 1 && (trans == 0 || trans == 1), ", nrhs >= 1, trans 0 or 1"));
  cudaStream_t st = ctx->stream;
  const int64_t nn = n * n, nbk = n * nrhs, ts = n * SOLVE_W;
  // per matrix: the panel T and tri_apply's partials (one k chunk per 64-row block: n <= 1024), as in the batched solve
  const int64_t chunk = batched_chunk(batch, (ts + round_up(n, 64) * SOLVE_W) * 8);
  double* T;
  CAP_TRY(ctx->workspace("batched_T", (size_t)(chunk * ts) * 8, (void**)&T));
  for (int64_t b0 = 0; b0 < batch; b0 += chunk) {
    const int64_t cnt = std::min(chunk, batch - b0);
    const double* Ub = U + b0 * nn;
    for (int64_t p0 = 0; p0 < nrhs; p0 += SOLVE_W) {
      const int64_t w = std::min<int64_t>(SOLVE_W, nrhs - p0);
      CAP_TRY(copy_batched(ctx, st, n, w, cnt, B + b0 * nbk + p0 * n, n, nbk, T, n, ts));
      //                 U   ldu trans  r0 r1 c0 c1 nrhs alpha P  pinc ldp beta Cin   ldcin C                       cinc ldc full  batch su  sp  scin sc
      CAP_TRY(tri_apply(ctx, st, {Ub, n, trans == 1, 0, n, 0, n, w, 1.0, T, 1, n, 0.0, nullptr, 0, X + b0 * nbk + p0 * n, 1, n, false, cnt, nn, ts, 0, nbk}));
    }
  }
  return CAPITAL_OK;
}

capital_status_t capital_cholinv_apply_rinv_batched_f64(capital_ctx* ctx, int64_t n, int64_t batch, const double* Rinv, int trans,
                                                        int64_t nrhs, const double* B, double* X) {
  if (!ctx) return CAPITAL_ERR_INVALID;
  return apply_batched(ctx, "apply_rinv_batched", "Rinv, B, X", n, batch, Rinv, trans, nrhs, B, X);
}

capital_status_t capital_cholinv_apply_r_batched_f64(capital_ctx* ctx, int64_t n, int64_t batch, const double* R, int trans, int64_t nrhs,
                                                     const double* B, double* X) {
  if (!ctx) return CAPITAL_ERR_INVALID;
  return apply_batched(ctx, "apply_r_batched", "R, B, X", n, batch, R, trans, nrhs, B, X);
}

// ||A Ainv - I||_F / ||I||_F (the inverse validator of the reference, test/inverse/validate.hpp:7-34, with the diagonal taken by global
// index).  A: the full symmetric local block; Ainv in `structure` as capital_cholinv_inverse_f64 wrote it.
capital_status_t capital_cholinv_inverse_residual_f64(capital_ctx* ctx, const double* A_local, int64_t n, capital_structure_t structure,
                                                      const double* Ainv_local, double* residual) {
  if (!ctx) return CAPITAL_ERR_INVALID;
  if (!A_local || !Ainv_local || !residual || n <= 0 || (structure != CAPITAL_RECT && structure != CAPITAL_UPPERTRI_PACKED)) {
    ctx->set_error("cholinv::inverse_residual: invalid arguments (A, Ainv, residual non-null, n > 0, packed upper or rect)");
    return CAPITAL_ERR_INVALID;
  }
  CAP_CUDA(cudaSetDevice(ctx->device));
  const capital_grid_t& g = ctx->grid;
  if (g.size > 1) return dist_cholinv_inverse_residual(ctx, A_local, n, structure, Ainv_local, residual);
  const int64_t L = n, ld = round_up(L, 16);
  const bool packed = structure == CAPITAL_UPPERTRI_PACKED;
  cudaStream_t st = ctx->stream;
  const double *dA, *dAi;
  CAP_TRY(cap_stage_in(ctx, A_local, (size_t)L * L, "A_in", &dA));
  CAP_TRY(cap_stage_in(ctx, Ainv_local, packed ? (size_t)L * (L + 1) / 2 : (size_t)L * L, "Ainv_in", &dAi));
  double *E, *Am, *F, *U;
  CAP_TRY(ctx->workspace("W", (size_t)ld * L * 8, (void**)&E));
  CAP_TRY(ctx->workspace("Ri", (size_t)ld * L * 8, (void**)&Am));
  CAP_TRY(ctx->workspace("Rm", (size_t)ld * L * 8, (void**)&F));
  CAP_TRY(copy_block(ctx, st, L, L, dA, L, Am, ld));
  if (packed) {
    CAP_TRY(ctx->workspace("RiT", (size_t)ld * L * 8, (void**)&U));
    CAP_TRY(unpack_upper(ctx, st, L, dAi, U, ld));
    CAP_TRY(sym_merge(ctx, st, L, U, ld, U, ld, true, F, ld, 0, 0, 1));
  } else {
    CAP_TRY(copy_block(ctx, st, L, L, dAi, L, F, ld));
  }
  CAP_TRY(gemm_tn(ctx, st, L, L, L, 1.0, Am, ld, F, ld, 0.0, E, ld, 0));  // A^T Ainv = A Ainv
  CAP_TRY(sub_identity_local(ctx, st, L, E, ld));
  CAP_CUDA(cudaMemsetAsync(ctx->d_scalars, 0, sizeof(double), st));
  CAP_TRY(sumsq_block(ctx, st, L, L, E, ld, 0, 0, 0, 1, ctx->d_scalars));
  double h = 0;
  CAP_CUDA(cudaMemcpyAsync(&h, ctx->d_scalars, sizeof(double), cudaMemcpyDeviceToHost, st));
  CAP_CUDA(cudaStreamSynchronize(st));
  *residual = sqrt(h) / sqrt((double)n);
  return CAPITAL_OK;
}

// ---- CholeskyQR2 ------------------------------------------------------------------------------
capital_status_t capital_cacqr_factor_f64(capital_ctx* ctx, const double* A_local, int64_t m, int64_t n, int num_iter,
                                          const capital_cholinv_args_t* ci_args, capital_structure_t rstruct, double* Q_local,
                                          double* R_local) {
  if (!ctx) return CAPITAL_ERR_INVALID;
  if (!A_local || !Q_local || !R_local || m <= 0 || n <= 0 || num_iter < 1 || num_iter > 3) {
    ctx->set_error("cacqr::factor: invalid arguments (A, Q, R non-null, m, n > 0, num_iter 1, 2 or 3)");
    return CAPITAL_ERR_INVALID;
  }
  CAP_CUDA(cudaSetDevice(ctx->device));
  return dist_cacqr_factor(ctx, A_local, m, n, num_iter, ci_args, rstruct, Q_local, R_local);
}
capital_status_t capital_cacqr_residual_f64(capital_ctx* ctx, const double* A_local, int64_t m, int64_t n, const double* Q_local,
                                            capital_structure_t rstruct, const double* R_local, double* residual,
                                            double* orthogonality) {
  if (!ctx || !A_local || !Q_local || !R_local || !residual || !orthogonality) return CAPITAL_ERR_INVALID;
  CAP_CUDA(cudaSetDevice(ctx->device));
  return dist_cacqr_residual(ctx, A_local, m, n, Q_local, rstruct, R_local, residual, orthogonality);
}

// Q^T B, R^-1 Q^T B and Q Z from the factor's outputs (dist.cu).  B_local / C_local: the rank's lr = ceil(m / d) rows; Y, X, Z: n x nrhs.
capital_status_t capital_cacqr_apply_qt_f64(capital_ctx* ctx, int64_t m, int64_t n, const double* Q_local, int64_t nrhs,
                                            const double* B_local, int64_t ldb, double* Y, int64_t ldy) {
  if (!ctx) return CAPITAL_ERR_INVALID;
  if (!Q_local || !B_local || !Y || n <= 0 || m < n || nrhs < 1 || ldb < ceil_div(m, ctx->grid.d) || ldy < n) {
    ctx->set_error("cacqr::apply_QT: invalid arguments (Q, B, Y non-null, m >= n > 0, nrhs >= 1, ldb >= ceil(m / d), ldy >= n)");
    return CAPITAL_ERR_INVALID;
  }
  CAP_CUDA(cudaSetDevice(ctx->device));
  return dist_cacqr_apply_qt(ctx, m, n, Q_local, CAPITAL_RECT, nullptr, nrhs, B_local, ldb, Y, ldy);
}
capital_status_t capital_cacqr_apply_q_f64(capital_ctx* ctx, int64_t m, int64_t n, const double* Q_local, int64_t nrhs,
                                           const double* Z, int64_t ldz, double* C_local, int64_t ldc) {
  if (!ctx) return CAPITAL_ERR_INVALID;
  if (!Q_local || !Z || !C_local || n <= 0 || m < n || nrhs < 1 || ldz < n || ldc < ceil_div(m, ctx->grid.d)) {
    ctx->set_error("cacqr::apply_Q: invalid arguments (Q, Z, C non-null, m >= n > 0, nrhs >= 1, ldz >= n, ldc >= ceil(m / d))");
    return CAPITAL_ERR_INVALID;
  }
  CAP_CUDA(cudaSetDevice(ctx->device));
  return dist_cacqr_apply_q(ctx, m, n, Q_local, nrhs, Z, ldz, C_local, ldc);
}
capital_status_t capital_cacqr_lstsq_f64(capital_ctx* ctx, int64_t m, int64_t n, const double* Q_local, capital_structure_t rstruct,
                                         const double* R_local, int64_t nrhs, const double* B_local, int64_t ldb, double* X, int64_t ldx) {
  if (!ctx) return CAPITAL_ERR_INVALID;
  if (!Q_local || !R_local || !B_local || !X || n <= 0 || m < n || nrhs < 1 || ldb < ceil_div(m, ctx->grid.d) || ldx < n ||
      (rstruct != CAPITAL_RECT && rstruct != CAPITAL_UPPERTRI_PACKED)) {
    ctx->set_error("cacqr::lstsq: invalid arguments (Q, R, B, X non-null, m >= n > 0, nrhs >= 1, ldb >= ceil(m / d), ldx >= n, "
                   "R packed upper or rect)");
    return CAPITAL_ERR_INVALID;
  }
  CAP_CUDA(cudaSetDevice(ctx->device));
  return dist_cacqr_apply_qt(ctx, m, n, Q_local, rstruct, R_local, nrhs, B_local, ldb, X, ldx);
}

// ---- batched CholeskyQR: many independent m x n matrices, n <= BASECASE_MAX, on this context's GPU (dist.cu) ----------------------
capital_status_t capital_cacqr_factor_batched_f64(capital_ctx* ctx, int64_t m, int64_t n, int64_t batch, int num_iter, const double* A,
                                                  double* Q, double* R, int* info) {
  if (!ctx) return CAPITAL_ERR_INVALID;
  if (!A || !Q || !R || !info || n < 1 || m < n || batch < 1 || num_iter < 1 || num_iter > 3) {
    ctx->set_error("cacqr::factor_batched: invalid arguments (A, Q, R, info non-null, m >= n >= 1, batch >= 1, num_iter 1, 2 or 3)");
    return CAPITAL_ERR_INVALID;
  }
  if (n > BASECASE_MAX) {
    ctx->set_error("cacqr::factor_batched: n > 512 is not supported (factor each matrix with capital_cacqr_factor_f64)");
    return CAPITAL_ERR_UNSUPPORTED;
  }
  CAP_CUDA(cudaSetDevice(ctx->device));
  if (!all_device({A, Q, R, info})) {
    ctx->set_error("cacqr::factor_batched: A, Q, R and info must be device pointers");
    return CAPITAL_ERR_INVALID;
  }
  if (overlaps(A, (size_t)(batch * m * n), Q, (size_t)(batch * m * n))) {
    ctx->set_error("cacqr::factor_batched: Q must not overlap A");
    return CAPITAL_ERR_INVALID;
  }
  return dist_cacqr_factor_batched(ctx, m, n, batch, num_iter, A, Q, R, info);
}

capital_status_t capital_cacqr_lstsq_batched_f64(capital_ctx* ctx, int64_t m, int64_t n, int64_t batch, const double* Q, const double* R,
                                                 int64_t nrhs, const double* B, double* X) {
  if (!ctx) return CAPITAL_ERR_INVALID;
  if (!Q || !R || !B || !X || n < 1 || m < n || batch < 1 || nrhs < 1) {
    ctx->set_error("cacqr::lstsq_batched: invalid arguments (Q, R, B, X non-null, m >= n >= 1, batch >= 1, nrhs >= 1)");
    return CAPITAL_ERR_INVALID;
  }
  if (n > BASECASE_MAX) {
    ctx->set_error("cacqr::lstsq_batched: n > 512 is not supported");
    return CAPITAL_ERR_UNSUPPORTED;
  }
  CAP_CUDA(cudaSetDevice(ctx->device));
  if (!all_device({Q, R, B, X})) {
    ctx->set_error("cacqr::lstsq_batched: Q, R, B and X must be device pointers");
    return CAPITAL_ERR_INVALID;
  }
  if (overlaps(B, (size_t)(batch * m * nrhs), X, (size_t)(batch * n * nrhs))) {
    ctx->set_error("cacqr::lstsq_batched: X must not overlap B");
    return CAPITAL_ERR_INVALID;
  }
  return dist_cacqr_lstsq_batched(ctx, m, n, batch, Q, R, nrhs, B, X);
}

// ---- SUMMA -----------------------------------------------------------------------------------
capital_status_t capital_summa_gemm_tn_f64(capital_ctx* ctx, int64_t m, int64_t n, int64_t k, double alpha, const double* A_local,
                                           const double* B_local, double beta, double* C_local) {
  if (!ctx || !A_local || !B_local || !C_local || m <= 0 || n <= 0 || k <= 0) return CAPITAL_ERR_INVALID;
  CAP_CUDA(cudaSetDevice(ctx->device));
  return dist_summa_gemm_tn(ctx, m, n, k, alpha, A_local, B_local, beta, C_local);
}

// ---- leaf-engine seam -------------------------------------------------------------------------
capital_status_t capital_blas_gemm_tn_f64(capital_ctx* ctx, int64_t m, int64_t n, int64_t k, double alpha, const double* A, int64_t lda,
                                          const double* B, int64_t ldb, double beta, double* C, int64_t ldc, int flags) {
  if (!ctx || !A || !B || !C) return CAPITAL_ERR_INVALID;
  CAP_CUDA(cudaSetDevice(ctx->device));
  if (!cap_is_device_ptr(A) || !cap_is_device_ptr(B) || !cap_is_device_ptr(C)) {
    ctx->set_error("capital_blas_gemm_tn_f64 takes device pointers");
    return CAPITAL_ERR_INVALID;
  }
  return gemm_tn(ctx, ctx->stream, m, n, k, alpha, A, lda, B, ldb, beta, C, ldc, flags);
}
// EXPERIMENTAL (BASELINE config 5): the same product on the TF32 tensor cores (wgmma), FP64 in and out
capital_status_t capital_blas_gemm_tn_tf32(capital_ctx* ctx, int64_t m, int64_t n, int64_t k, double alpha, const double* A, int64_t lda,
                                           const double* B, int64_t ldb, double beta, double* C, int64_t ldc, int flags, int passes) {
  if (!ctx || !A || !B || !C) return CAPITAL_ERR_INVALID;
  CAP_CUDA(cudaSetDevice(ctx->device));
  if (!cap_is_device_ptr(A) || !cap_is_device_ptr(B) || !cap_is_device_ptr(C)) {
    ctx->set_error("capital_blas_gemm_tn_tf32 takes device pointers");
    return CAPITAL_ERR_INVALID;
  }
  CAP_CUDA(cudaMemsetAsync(ctx->d_info, 0, sizeof(int), ctx->stream));
  CAP_TRY(gemm_tn_tf32(ctx, ctx->stream, m, n, k, alpha, A, lda, B, ldb, beta, C, ldc, flags, passes));
  return cap_check_info(ctx);
}
capital_status_t capital_set_trailing_precision(capital_ctx* ctx, int mode) {
  if (!ctx) return CAPITAL_ERR_INVALID;
  if (mode != 0 && mode != 1 && mode != 3) { ctx->set_error("trailing precision: 0 (FP64), 1 (TF32) or 3 (3 x TF32, split operands)"); return CAPITAL_ERR_INVALID; }
  ctx->trailing_mode = mode;
  return CAPITAL_OK;
}
capital_status_t capital_tf32_stats(const capital_ctx* ctx, int64_t* launches, double* flops) {
  if (!ctx || !launches || !flops) return CAPITAL_ERR_INVALID;
  *launches = ctx->tf32_launches; *flops = ctx->tf32_flops;
  return CAPITAL_OK;
}
capital_status_t capital_lapack_potrf_trtri_f64(capital_ctx* ctx, int64_t n, const double* A, int64_t lda, double* R, int64_t ldr,
                                                double* Rinv, int64_t ldri) {
  if (!ctx || !A || !R || !Rinv || n <= 0 || lda < n || ldr < n || ldri < n) return CAPITAL_ERR_INVALID;
  CAP_CUDA(cudaSetDevice(ctx->device));
  if (!cap_is_device_ptr(A) || !cap_is_device_ptr(R) || !cap_is_device_ptr(Rinv)) return CAPITAL_ERR_INVALID;
  if ((ldr & 1) || (ldri & 1)) { ctx->set_error("potrf_trtri: ldr, ldri must be even"); return CAPITAL_ERR_INVALID; }
  cudaStream_t st = ctx->stream;
  const int64_t ld = round_up(n, 16);
  double *W, *RiT;
  CAP_TRY(ctx->workspace("bcW", (size_t)ld * n * 8, (void**)&W));
  CAP_TRY(ctx->workspace("bcRiT", (size_t)ld * n * 8, (void**)&RiT));
  CAP_CUDA(cudaMemsetAsync(ctx->d_info, 0, sizeof(int), st));
  CAP_TRY(copy_block(ctx, st, n, n, A, lda, W, ld));
  CAP_TRY(zero_block(ctx, st, n, n, R, ldr));
  CAP_TRY(zero_block(ctx, st, n, n, Rinv, ldri));
  CAP_CUDA(cudaMemsetAsync(RiT, 0, (size_t)ld * n * 8, st));
  CAP_TRY(cholinv_local(ctx, st, n, W, ld, R, ldr, Rinv, ldri, RiT, ld, true, n, 1));
  return cap_check_info(ctx);
}

}  // extern "C"
