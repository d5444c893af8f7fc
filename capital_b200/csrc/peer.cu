// Peer layer implementation: IPC-mapped control blocks and arenas, flag kernels, device barrier, small all-reduce.
// See peer.cuh for the model.  NCCL is dlopen'ed ("libnccl.so.2": the copy torch already mapped when the caller is a torch
// process, else the system one) and used for ONE thing: the host-visible allgather that exchanges the IPC handles.
#include "peer.cuh"
#include "dist.cuh"
#include <dlfcn.h>
#include <stdlib.h>
#include <string.h>

namespace {

typedef struct ncclComm* ncclComm_t;
typedef struct { char internal[128]; } ncclUniqueId;
enum { ncclSuccess = 0 };
enum { ncclInt8 = 0 };

struct NcclApi {
  void* lib = nullptr;
  int (*GetUniqueId)(ncclUniqueId*) = nullptr;
  int (*CommInitRank)(ncclComm_t*, int, ncclUniqueId, int) = nullptr;
  int (*CommDestroy)(ncclComm_t) = nullptr;
  int (*AllGather)(const void*, void*, size_t, int, ncclComm_t, cudaStream_t) = nullptr;
  const char* (*GetErrorString)(int) = nullptr;
};
NcclApi& nccl() {
  static NcclApi api;
  return api;
}
bool nccl_load(std::string* why) {
  NcclApi& a = nccl();
  if (a.lib) return true;
  const char* names[] = {"libnccl.so.2", "libnccl.so"};
  for (const char* nm : names) {
    a.lib = dlopen(nm, RTLD_NOW | RTLD_GLOBAL);
    if (a.lib) break;
  }
  if (!a.lib) { *why = std::string("dlopen(libnccl.so.2) failed: ") + dlerror(); return false; }
#define LD(field, sym)                                                   \
  *(void**)(&a.field) = dlsym(a.lib, sym);                               \
  if (!a.field) { *why = std::string("missing NCCL symbol ") + sym; a.lib = nullptr; return false; }
  LD(GetUniqueId, "ncclGetUniqueId"); LD(CommInitRank, "ncclCommInitRank"); LD(CommDestroy, "ncclCommDestroy");
  LD(AllGather, "ncclAllGather"); LD(GetErrorString, "ncclGetErrorString");
#undef LD
  return true;
}

// host allgather over the NCCL world communicator (small blobs: staged through a device buffer)
int nccl_allgather(void* user, const void* send, void* recv, int64_t bytes) {
  capital_ctx* ctx = (capital_ctx*)user;
  Peer* P = peer_of(ctx);
  const int size = ctx->grid.size;
  if (bytes > 4096) return 1;
  char* d = (char*)P->d_stage;  // [send 4096][recv size * 4096]
  if (cudaMemcpyAsync(d, send, bytes, cudaMemcpyHostToDevice, ctx->stream) != cudaSuccess) return 2;
  if (nccl().AllGather(d, d + 4096, (size_t)bytes, ncclInt8, (ncclComm_t)ctx->comm_world, ctx->stream) != ncclSuccess) return 3;
  if (cudaMemcpyAsync(recv, d + 4096, (size_t)bytes * size, cudaMemcpyDeviceToHost, ctx->stream) != cudaSuccess) return 4;
  if (cudaStreamSynchronize(ctx->stream) != cudaSuccess) return 5;
  return 0;
}

__global__ void signal_kernel(FlagList fl) {
  const int i = threadIdx.x;
  if (i < fl.n) {
    __threadfence_system();
    asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(fl.p[i]), "l"(fl.v[i]) : "memory");
  }
}
__global__ void wait_kernel(FlagList fl, int* err) {
  const int i = threadIdx.x;
  if (i < fl.n) {
    unsigned long long got, t0, t1;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t0));
    for (;;) {
      asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(got) : "l"(fl.p[i]) : "memory");
      if (got >= fl.v[i]) break;
      __nanosleep(100);
      asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t1));
      // a peer died or the schedules diverged: report, do not hang.  Generous (ranks may legitimately be seconds apart, e.g. while
      // one of them pins host memory); once a wait has given up, the ones queued behind it give up at once.
      if (t1 - t0 > 120000000000ull || *(volatile int*)err == -1) { atomicExch(err, -1); break; }
    }
  }
  __syncthreads();
}
// dst_r[slot(me)][i] = src[i] on every rank r (own copy included): blockIdx.y = destination rank
struct ArDst { double* p[PEER_MAX_RANKS]; };
__global__ void ar_scatter_kernel(const double* src, long long count, ArDst dst) {
  double* d = dst.p[blockIdx.y];
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < count; i += (long long)gridDim.x * blockDim.x) d[i] = src[i];
  __threadfence_system();
}
__global__ void ar_sum_kernel(double* buf, long long count, const double* slots, int size) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < count; i += (long long)gridDim.x * blockDim.x) {
    double s = __ldcg(slots + i);
    for (int r = 1; r < size; r++) s += __ldcg(slots + (long long)r * count + i);  // rank order: the same bits on every rank
    buf[i] = s;
  }
}

// stream memory operations (driver API, resolved at run time: the library does not link libcuda)
typedef CUresult (*fn_batch)(CUstream, unsigned int, CUstreamBatchMemOpParams*, unsigned int);
fn_batch g_batch = nullptr;
bool memops_load() {
  if (g_batch) return true;
  void* p = nullptr;
  cudaDriverEntryPointQueryResult q;
  if (cudaGetDriverEntryPoint("cuStreamBatchMemOp", &p, cudaEnableDefault, &q) != cudaSuccess || !p) return false;
  g_batch = (fn_batch)p;
  return true;
}
capital_status_t memops_issue(capital_ctx* ctx, cudaStream_t st, const FlagList& fl, bool wait, bool flush = false) {
  CUstreamBatchMemOpParams ops[24];
  memset(ops, 0, sizeof(ops));
  for (int i = 0; i < fl.n; i++) {
    if (wait) {
      ops[i].waitValue.operation = CU_STREAM_MEM_OP_WAIT_VALUE_64;
      ops[i].waitValue.address = (CUdeviceptr)fl.p[i];
      ops[i].waitValue.value64 = fl.v[i];
      // FLUSH: "the device is permitted to reorder remote writes internally" (cuda.h, CUstreamWaitValue_flags) -- without it a
      // wait satisfied by a peer's flag does not make that peer's EARLIER stores (partial sums written by its GEMM epilogue over
      // NVLink) visible to the kernels that follow the wait.  Observed as small, run-to-run varying errors of the distributed
      // factorization over real NVLink.
      ops[i].waitValue.flags = CU_STREAM_WAIT_VALUE_GEQ | (flush ? CU_STREAM_WAIT_VALUE_FLUSH : 0);
    } else {
      ops[i].writeValue.operation = CU_STREAM_MEM_OP_WRITE_VALUE_64;
      ops[i].writeValue.address = (CUdeviceptr)fl.p[i];
      ops[i].writeValue.value64 = fl.v[i];
      ops[i].writeValue.flags = CU_STREAM_WRITE_VALUE_DEFAULT;  // ordered after (fenced against) the stream's earlier writes
    }
  }
  const CUresult r = g_batch((CUstream)st, (unsigned)fl.n, ops, 0);
  if (r != CUDA_SUCCESS) {
    ctx->set_error("cuStreamBatchMemOp failed: CUresult " + std::to_string((int)r));
    return CAPITAL_ERR_CUDA;
  }
  return CAPITAL_OK;
}

capital_status_t exchange(capital_ctx* ctx, const void* mine, void* all, int64_t bytes) {
  Peer* P = peer_of(ctx);
  const int rc = P->ag(P->ag_user, mine, all, bytes);
  if (rc != 0) { ctx->set_error("peer bootstrap: host allgather failed (rc " + std::to_string(rc) + ")"); return CAPITAL_ERR_COMM; }
  return CAPITAL_OK;
}
capital_status_t host_barrier(capital_ctx* ctx) {
  Peer* P = peer_of(ctx);
  if (P->size == 1 || !P->ag) return CAPITAL_OK;
  std::vector<char> all((size_t)P->size * 8);
  long long x = 1;
  return exchange(ctx, &x, all.data(), 8);
}

}  // namespace

// all ranks: every stream of this device has drained AND every rank has reached this point
capital_status_t peer_host_barrier(capital_ctx* ctx) {
  CAP_CUDA(cudaDeviceSynchronize());
  return host_barrier(ctx);
}

capital_status_t peer_init(capital_ctx* ctx, peer_allgather_fn ag, void* user) {
  const capital_grid_t& g = ctx->grid;
  if (g.size > PEER_MAX_RANKS) { ctx->set_error("peer layer: at most 16 ranks (one NVSwitch node)"); return CAPITAL_ERR_UNSUPPORTED; }
  Peer* P = peer_of(ctx);
  if (!P) { P = new Peer(); ctx->peer = P; }
  P->size = g.size; P->rank = g.rank; P->ag = ag; P->ag_user = user;
  CAP_CUDA(cudaMalloc(&P->ctrl, CTRL_WORDS * 8));
  CAP_CUDA(cudaMemset(P->ctrl, 0, CTRL_WORDS * 8));
  if (const char* e = getenv("CAPITAL_PEER_MEMOPS")) P->memops = atoi(e) != 0;
  if (P->memops && !memops_load()) P->memops = false;
  // How a stream waits for a flag a peer writes (see memops_issue): a memory-op wait must carry the remote-write flush; where
  // the device cannot flush (or the driver refuses the flag) the wait is a one-warp kernel spinning on ld.acquire.sys instead.
  P->wait_mode = PEER_WAIT_KERNEL;
  if (P->memops) {
    int dev = 0, can = 0;
    CAP_CUDA(cudaGetDevice(&dev));
    if (cudaDeviceGetAttribute(&can, cudaDevAttrCanFlushRemoteWrites, dev) != cudaSuccess) { can = 0; cudaGetLastError(); }
    if (can) {
      // refuse-proof: one already-satisfied flushed wait on this rank's own control block
      FlagList t;
      t.add(P->ctrl + CTRL_WORDS - 1, 0);
      cudaStream_t ts;
      CAP_CUDA(cudaStreamCreateWithFlags(&ts, cudaStreamNonBlocking));
      const bool ok = memops_issue(ctx, ts, t, true, true) == CAPITAL_OK && cudaStreamSynchronize(ts) == cudaSuccess;
      cudaStreamDestroy(ts);
      P->can_flush = ok;
      if (ok) P->wait_mode = PEER_WAIT_MEMOP_FLUSH;
      else { cudaGetLastError(); ctx->set_error(""); }
    }
  }
  if (const char* e = getenv("CAPITAL_PEER_WAIT")) {
    // "memop" = round-2 behaviour up to here (unflushed; kept to reproduce the bug), "flush", "kernel"
    if (!strcmp(e, "kernel")) P->wait_mode = PEER_WAIT_KERNEL;
    else if (P->memops && !strcmp(e, "flush")) P->wait_mode = PEER_WAIT_MEMOP_FLUSH;
    else if (P->memops && !strcmp(e, "memop")) P->wait_mode = PEER_WAIT_MEMOP;
  }
  cudaIpcMemHandle_t mine;
  CAP_CUDA(cudaIpcGetMemHandle(&mine, P->ctrl));
  std::vector<cudaIpcMemHandle_t> all(g.size);
  CAP_TRY(exchange(ctx, &mine, all.data(), sizeof(mine)));
  for (int r = 0; r < g.size; r++) {
    if (r == g.rank) { P->peer_ctrl[r] = P->ctrl; continue; }
    CAP_CUDA(cudaIpcOpenMemHandle((void**)&P->peer_ctrl[r], all[r], cudaIpcMemLazyEnablePeerAccess));
  }
  int lo = 0, hi = 0;
  cudaDeviceGetStreamPriorityRange(&lo, &hi);
  for (int q = 0; q < PEER_Q; q++) CAP_CUDA(cudaStreamCreateWithPriority(&P->push[q], cudaStreamNonBlocking, q == 0 ? hi : lo));
  return host_barrier(ctx);  // nobody proceeds (and possibly tears down) before every rank has mapped every control block
}

void peer_destroy(capital_ctx* ctx) {
  Peer* P = peer_of(ctx);
  if (!P) return;
  cudaDeviceSynchronize();
  for (int r = 0; r < P->size; r++) {
    if (r == P->rank) continue;
    if (P->peer_arena[r]) cudaIpcCloseMemHandle(P->peer_arena[r]);
    if (P->peer_ctrl[r]) cudaIpcCloseMemHandle(P->peer_ctrl[r]);
  }
  if (P->arena) cudaFree(P->arena);
  if (P->ctrl) cudaFree(P->ctrl);
  if (P->d_stage) cudaFree(P->d_stage);
  for (int q = 0; q < PEER_Q; q++) if (P->push[q]) cudaStreamDestroy(P->push[q]);
  if (ctx->comm_world && nccl().lib) nccl().CommDestroy((ncclComm_t)ctx->comm_world);
  ctx->comm_world = nullptr;
  delete P;
  ctx->peer = nullptr;
}

capital_status_t peer_arena_release(capital_ctx* ctx) {
  Peer* P = peer_of(ctx);
  if (!P || !P->arena) return CAPITAL_OK;
  CAP_CUDA(cudaDeviceSynchronize());
  CAP_TRY(host_barrier(ctx));  // every rank has drained its streams: nobody still writes into (or reads from) a peer's arena
  for (int r = 0; r < P->size; r++) {
    if (r == P->rank || !P->peer_arena[r]) continue;
    CAP_CUDA(cudaIpcCloseMemHandle(P->peer_arena[r]));
    P->peer_arena[r] = nullptr;
  }
  CAP_TRY(host_barrier(ctx));  // all mappings are closed before the owner frees
  CAP_CUDA(cudaFree(P->arena));
  P->arena = nullptr; P->arena_bytes = 0;
  return CAPITAL_OK;
}

capital_status_t peer_arena_reserve(capital_ctx* ctx, size_t bytes) {
  Peer* P = peer_of(ctx);
  if (!P) { ctx->set_error("multi-GPU grid but capital_comm_init was not called"); return CAPITAL_ERR_COMM; }
  if (bytes <= P->arena_bytes) return CAPITAL_OK;  // same decision on every rank: sizes are functions of the shape and the grid
  CAP_TRY(peer_arena_release(ctx));
  bytes = (size_t)round_up((int64_t)bytes, (int64_t)2 << 20);
  CAP_CUDA(cudaMalloc(&P->arena, bytes));
  P->arena_bytes = bytes;
  P->peer_arena[P->rank] = P->arena;
  cudaIpcMemHandle_t mine;
  CAP_CUDA(cudaIpcGetMemHandle(&mine, P->arena));
  std::vector<cudaIpcMemHandle_t> all(P->size);
  CAP_TRY(exchange(ctx, &mine, all.data(), sizeof(mine)));
  for (int r = 0; r < P->size; r++) {
    if (r == P->rank) continue;
    CAP_CUDA(cudaIpcOpenMemHandle((void**)&P->peer_arena[r], all[r], cudaIpcMemLazyEnablePeerAccess));
  }
  return host_barrier(ctx);
}

capital_status_t peer_signal(capital_ctx* ctx, cudaStream_t st, const FlagList& fl) {
  if (fl.n == 0) return CAPITAL_OK;
  const int tli = ctx->tl_begin(st, 6, fl.n);
  if (peer_of(ctx)->memops) {
    const capital_status_t rs = memops_issue(ctx, st, fl, false);
    ctx->tl_end(st, tli);
    return rs;
  }
  signal_kernel<<<1, 32, 0, st>>>(fl);
  ctx->tl_end(st, tli);
  ctx->counters.kernel_launches++;
  CAP_CUDA(cudaGetLastError());
  return CAPITAL_OK;
}
capital_status_t peer_wait(capital_ctx* ctx, cudaStream_t st, const FlagList& fl) {
  if (fl.n == 0) return CAPITAL_OK;
  const int tli = ctx->tl_begin(st, 5, fl.n);
  const int wm = peer_of(ctx)->wait_mode;
  if (wm != PEER_WAIT_KERNEL) {
    const capital_status_t rs = memops_issue(ctx, st, fl, true, wm == PEER_WAIT_MEMOP_FLUSH);
    ctx->tl_end(st, tli);
    return rs;
  }
  wait_kernel<<<1, 32, 0, st>>>(fl, ctx->d_info);
  ctx->tl_end(st, tli);
  ctx->counters.kernel_launches++;
  CAP_CUDA(cudaGetLastError());
  return CAPITAL_OK;
}

capital_status_t peer_barrier(capital_ctx* ctx, cudaStream_t st) {
  Peer* P = peer_of(ctx);
  const unsigned long long e = ++P->bar_epoch;
  FlagList s, w;
  for (int r = 0; r < P->size; r++) {
    if (r == P->rank) continue;
    if (s.n == 24) { CAP_TRY(peer_signal(ctx, st, s)); s.n = 0; }
    s.add(ctrl_ptr(P, r, CTRL_BAR + P->rank), e);
    w.add(P->ctrl + CTRL_BAR + r, e);
  }
  CAP_TRY(peer_signal(ctx, st, s));
  return peer_wait(ctx, st, w);
}

capital_status_t peer_allreduce_sum(capital_ctx* ctx, cudaStream_t st, double* buf, int64_t count, const ArSlots& slots) {
  Peer* P = peer_of(ctx);
  if (!P || P->size == 1) return CAPITAL_OK;
  if (count > slots.cap) {
    ctx->set_error("peer_allreduce_sum: " + std::to_string(count) + " doubles exceed the slot capacity " + std::to_string(slots.cap));
    return CAPITAL_ERR_INVALID;
  }
  const unsigned long long e = ++P->ar_epoch;
  double* half = slots.base + (e & 1) * (size_t)P->size * slots.cap;
  ArDst dst;
  for (int r = 0; r < P->size; r++) dst.p[r] = peer_ptr(P, r, half) + (size_t)P->rank * count;
  const int gx = (int)(count >= 1 << 16 ? 32 : ceil_div(count, 2048) > 0 ? ceil_div(count, 2048) : 1);
  ar_scatter_kernel<<<dim3(gx, P->size), 256, 0, st>>>(buf, count, dst);
  FlagList s, w;
  for (int r = 0; r < P->size; r++) {
    if (r == P->rank) continue;
    s.add(ctrl_ptr(P, r, CTRL_AR + P->rank), e);
    w.add(P->ctrl + CTRL_AR + r, e);
  }
  CAP_TRY(peer_signal(ctx, st, s));
  CAP_TRY(peer_wait(ctx, st, w));
  ar_sum_kernel<<<gx, 256, 0, st>>>(buf, count, half, P->size);
  ctx->counters.kernel_launches += 2;
  CAP_CUDA(cudaGetLastError());
  return CAPITAL_OK;
}

// ---- C ABI: bootstrap ---------------------------------------------------------------------------------------------
extern "C" capital_status_t capital_comm_unique_id(void* out128) {
  std::string why;
  if (!out128 || !nccl_load(&why)) return CAPITAL_ERR_COMM;
  ncclUniqueId id;
  if (nccl().GetUniqueId(&id) != ncclSuccess) return CAPITAL_ERR_COMM;
  memcpy(out128, &id, 128);
  return CAPITAL_OK;
}

extern "C" capital_status_t capital_comm_init(capital_ctx* ctx, const void* uid) {
  if (!ctx || !uid) return CAPITAL_ERR_INVALID;
  if (ctx->peer) { ctx->set_error("capital_comm_init: the context already joined a clique"); return CAPITAL_ERR_INVALID; }
  CAP_CUDA(cudaSetDevice(ctx->device));
  std::string why;
  if (!nccl_load(&why)) { ctx->set_error(why); return CAPITAL_ERR_COMM; }
  const capital_grid_t& g = ctx->grid;
  ncclUniqueId id;
  memcpy(&id, uid, 128);
  ncclComm_t world = nullptr;
  const int r = nccl().CommInitRank(&world, g.size, id, g.rank);
  if (r != ncclSuccess) { ctx->set_error(std::string("ncclCommInitRank: ") + nccl().GetErrorString(r)); return CAPITAL_ERR_COMM; }
  ctx->comm_world = world;
  Peer* P = new Peer();
  ctx->peer = P;
  CAP_CUDA(cudaMalloc(&P->d_stage, 4096 * (size_t)(g.size + 1)));
  const capital_status_t st = peer_init(ctx, nccl_allgather, ctx);
  if (st != CAPITAL_OK) peer_destroy(ctx);  // never leave a half-built clique behind
  return st;
}

extern "C" int capital_peer_wait_mode(const capital_ctx* ctx) {
  if (!ctx || !ctx->peer) return -1;
  return ((const Peer*)ctx->peer)->wait_mode;
}

// between calls only (every stream of the context idle): waits enqueued afterwards use the new flavour
extern "C" capital_status_t capital_set_peer_wait_mode(capital_ctx* ctx, int mode) {
  if (!ctx || !ctx->peer) return CAPITAL_ERR_INVALID;
  Peer* P = (Peer*)ctx->peer;
  if (mode == PEER_WAIT_KERNEL) { P->wait_mode = mode; return CAPITAL_OK; }
  if (mode == PEER_WAIT_MEMOP && P->memops) { P->wait_mode = mode; return CAPITAL_OK; }
  if (mode == PEER_WAIT_MEMOP_FLUSH && P->memops && P->can_flush) { P->wait_mode = mode; return CAPITAL_OK; }
  ctx->set_error("peer wait mode: 0 (memory op), 1 (flushed memory op; needs device support) or 2 (acquire-spin kernel)");
  return CAPITAL_ERR_UNSUPPORTED;
}

extern "C" capital_status_t capital_comm_init_host(capital_ctx* ctx, capital_allgather_fn allgather, void* user) {
  if (!ctx || !allgather) return CAPITAL_ERR_INVALID;
  if (ctx->peer) { ctx->set_error("capital_comm_init_host: the context already joined a clique"); return CAPITAL_ERR_INVALID; }
  CAP_CUDA(cudaSetDevice(ctx->device));
  const capital_status_t st = peer_init(ctx, (peer_allgather_fn)allgather, user);
  if (st != CAPITAL_OK) peer_destroy(ctx);
  return st;
}
