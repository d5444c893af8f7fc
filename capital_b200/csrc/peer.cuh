// Peer layer: what replaces the reference's MPI calls on one NVSwitch node.
//
// One process per GPU.  Every rank owns (a) a small CONTROL block of 64-bit flags and (b) one big data ARENA; both are
// cudaMalloc'ed, exported with cudaIpcGetMemHandle and mapped by every other rank, so that any rank can
//   * DMA a finished block into a consumer's mirror buffer (copy engines, cudaMemcpy2DAsync on a push stream),
//   * store GEMM partials / final tiles straight from the epilogue into a depth partner's memory (gemm_tn.cu, GemmXDev),
//   * raise a flag in another rank's control block -- a stream memory operation (cuStreamWriteValue64: no SM is needed, so a flag
//     is never stuck behind the CTAs of a running GEMM) -- and wait on its own flags: a flushed memory-operation wait where the device
//     can flush remote writes, else a one-warp kernel spinning on ld.acquire.sys (peer_init; an unflushed memory-op wait does not
//     make the peer's earlier stores visible to the kernels behind it).
// The arena layout is a pure function of the problem shape and of the grid, identical on every rank, so an offset computed
// locally addresses the same object in every peer's arena ("symmetric heap").  Flags carry monotonically increasing sequence
// numbers (never reset), which makes "wait until flag >= v" race-free across repeated factorizations.
//
// Bootstrap (exchange of the IPC handles) goes through a host allgather: NCCL's (capital_comm_init: the ncclUniqueId comes from
// torch.distributed / MPI) or a caller-supplied one (capital_comm_init_host: MPI_Allgather in a C caller; also what lets several
// ranks share one GPU in tests, which NCCL refuses).  NCCL moves no matrix data.
#pragma once
#include "common.cuh"

constexpr int PEER_MAX_RANKS = 16;
constexpr int PEER_NFAR = 3;                 // deferred classes: one per recursion depth 0 .. 2 (a deeper node's deferred work is needed sooner
                                             // than its ancestors' and must not queue behind it on one FIFO stream)
constexpr int PEER_QC = 1 + PEER_NFAR;       // classes that run products (own compute stream, exchange buffers): 0 = critical chain, 1 .. = deferred
constexpr int PEER_Q = PEER_QC + 1;          // flag / push-stream classes: the product classes + bulk pushes (node-entry operands)
// control block layout (units of 8 bytes)
constexpr size_t CTRL_PUSH = 0;                                   // [src][q]   "all I pushed to you on class q up to id v has landed"
constexpr size_t CTRL_DONE = CTRL_PUSH + PEER_MAX_RANKS * PEER_Q; // [src][q]   "my fused product v on class q has retired"
constexpr size_t CTRL_BAR = CTRL_DONE + PEER_MAX_RANKS * PEER_Q;  // [src]      world barrier epochs
constexpr size_t CTRL_AR = CTRL_BAR + PEER_MAX_RANKS;             // [src]      small all-reduce epochs
constexpr size_t CTRL_RED = CTRL_AR + PEER_MAX_RANKS;             // [src][q]   "I have added up the partials of product v of class q"
constexpr size_t CTRL_GAR = CTRL_RED + PEER_MAX_RANKS * PEER_Q;   // [src]      "my Gram partial of cross-cube all-reduce v has landed"
constexpr size_t CTRL_SAR = CTRL_GAR + PEER_MAX_RANKS;             // [src]      "my trace partial of Gram shift v has landed" (sCQR3)
constexpr size_t CTRL_WORDS = 512;
enum { PEER_WAIT_MEMOP = 0, PEER_WAIT_MEMOP_FLUSH = 1, PEER_WAIT_KERNEL = 2 };
static_assert(CTRL_SAR + PEER_MAX_RANKS <= CTRL_WORDS, "control block too small");

typedef int (*peer_allgather_fn)(void* user, const void* send, void* recv, int64_t bytes_per_rank);

struct FlagList {
  int n = 0;
  unsigned long long* p[24];
  unsigned long long v[24];
  void add(unsigned long long* ptr, unsigned long long val) { p[n] = ptr; v[n] = val; n++; }
};

struct Peer {
  int size = 0, rank = 0;
  peer_allgather_fn ag = nullptr;
  void* ag_user = nullptr;
  unsigned long long* ctrl = nullptr;
  unsigned long long* peer_ctrl[PEER_MAX_RANKS] = {};
  char* arena = nullptr;
  size_t arena_bytes = 0;
  char* peer_arena[PEER_MAX_RANKS] = {};
  cudaStream_t push[PEER_Q] = {};
  unsigned long long push_id[PEER_Q] = {};          // logical push events issued so far (same on every rank)
  unsigned long long prod_seq[PEER_QC] = {};        // products with a depth exchange issued so far
  unsigned long long bar_epoch = 0, ar_epoch = 0;
  unsigned long long gar_epoch = 0;                 // cross-cube all-reduces of the tunable grid issued so far (dist.cu)
  unsigned long long sar_epoch = 0;                 // Gram shifts of shifted CholeskyQR3 on the 3D / tunable grids issued so far
  bool can_flush = false;  // the device accepts CU_STREAM_WAIT_VALUE_FLUSH (attribute + self test at init)
  int wait_mode = 2;    // PEER_WAIT_*: how a stream waits for a peer-written flag [env CAPITAL_PEER_WAIT]
  bool memops = true;   // flags through stream memory operations (no SM needed) instead of one-warp kernels [env CAPITAL_PEER_MEMOPS]
  // NCCL bootstrap (only when capital_comm_init was used)
  void* d_stage = nullptr;
};

inline Peer* peer_of(capital_ctx* ctx) { return (Peer*)ctx->peer; }

capital_status_t peer_init(capital_ctx* ctx, peer_allgather_fn ag, void* user);
void peer_destroy(capital_ctx* ctx);
// collective: make the arena at least `bytes` big (re-allocates and re-exchanges the handle when it has to grow)
capital_status_t peer_arena_reserve(capital_ctx* ctx, size_t bytes);
// collective: unmap the peers' arenas, free the own one (capital_release_workspace)
capital_status_t peer_arena_release(capital_ctx* ctx);
capital_status_t peer_host_barrier(capital_ctx* ctx);  // device drained on every rank, and every rank is here
// address of my arena object `p` inside rank r's arena
template <typename T>
inline T* peer_ptr(const Peer* P, int r, T* p) { return r == P->rank ? p : (T*)(P->peer_arena[r] + ((char*)p - P->arena)); }
inline unsigned long long* ctrl_ptr(const Peer* P, int r, size_t word) { return (r == P->rank ? P->ctrl : P->peer_ctrl[r]) + word; }

capital_status_t peer_signal(capital_ctx* ctx, cudaStream_t st, const FlagList& fl);  // remote (or local) flag stores, ordered after the stream's earlier work
capital_status_t peer_wait(capital_ctx* ctx, cudaStream_t st, const FlagList& fl);    // the stream stalls until every LOCAL flag has reached its value
capital_status_t peer_barrier(capital_ctx* ctx, cudaStream_t st);                     // all ranks: everything enqueued on `st` before has completed everywhere
// Slot set of the small all-reduce: an arena region of two halves of size * cap doubles (room for `cap` doubles per rank).  All-reduce e
// scatters into half e & 1, whose place does not depend on the count.  Two halves suffice when a rank's consecutive all-reduces are
// ordered on its stream or separated by a call's opening barrier: a rank raises flag e only after its sum e - 1, so no rank can scatter
// e + 1 into a half that someone is still summing e - 1 from.
struct ArSlots {
  double* base = nullptr;
  int64_t cap = 0;
};
// sum of `count` <= slots.cap doubles over all ranks, in rank order on every rank (bit-identical results)
capital_status_t peer_allreduce_sum(capital_ctx* ctx, cudaStream_t st, double* buf, int64_t count, const ArSlots& slots);
