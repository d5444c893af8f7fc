// Probe: cross-process peer memory on one node (what the multi-GPU schedule of dist.cu is built on).
//   probe_p2p NP [same_device]
// NP processes (fork before CUDA init), rank r on GPU r % ndev (or all on GPU 0 with same_device=1).
// Measures: IPC mapping, DMA push bandwidth (contiguous / strided 2D), SM remote-store and remote-load bandwidth,
// flag ping-pong latency with signal/wait kernels and with stream memory ops (cuStreamWriteValue64 / WaitValue64).
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o probe_p2p probe_p2p.cu -lcuda
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <sys/mman.h>
#include <sys/wait.h>
#include <unistd.h>

#define CK(x) do { cudaError_t e = (x); if (e != cudaSuccess) { printf("[r%d] CUDA error %s at line %d\n", g_rank, cudaGetErrorString(e), __LINE__); fflush(stdout); _exit(2); } } while (0)
#define CKD(x) do { CUresult e = (x); if (e != CUDA_SUCCESS) { const char* s; cuGetErrorString(e, &s); printf("[r%d] driver error %s at line %d\n", g_rank, s, __LINE__); fflush(stdout); g_drv_fail = 1; } } while (0)
static int g_rank = 0, g_drv_fail = 0;

struct Shared {
  volatile int barrier[64];
  cudaIpcMemHandle_t data[16], flags[16];
};

static void host_barrier(Shared* sh, int np, int idx) {
  __sync_fetch_and_add(&sh->barrier[idx], 1);
  while (sh->barrier[idx] < np) usleep(50);
}

__global__ void signal_kernel(unsigned long long* peer_flag, unsigned long long v) {
  __threadfence_system();
  asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(peer_flag), "l"(v) : "memory");
}
__global__ void wait_kernel(const unsigned long long* my_flag, unsigned long long v, int* timeout) {
  unsigned long long got;
  long long t0 = clock64();
  do {
    asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(got) : "l"(my_flag) : "memory");
    if (clock64() - t0 > 20000000000LL) { *timeout = 1; break; }
  } while (got < v);
}
__global__ void store16_kernel(double2* dst, size_t n2, double v) {
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n2; i += (size_t)gridDim.x * blockDim.x) dst[i] = make_double2(v, v + 1);
}
// the GEMM epilogue's pattern: a warp instruction covers 8 consecutive doubles in each of 4 columns
__global__ void store_epi_kernel(double* dst, long long ld, int rows, int cols, double v) {
  const int lane = threadIdx.x & 31, g = lane >> 2, q = lane & 3;
  const int warps = (gridDim.x * blockDim.x) >> 5, w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const long long nblk = (long long)(rows / 8) * (cols / 8);
  for (long long b = w; b < nblk; b += warps) {
    const int r0 = (int)(b % (rows / 8)) * 8, c0 = (int)(b / (rows / 8)) * 8;
    dst[(long long)(c0 + 2 * q) * ld + r0 + g] = v;
    dst[(long long)(c0 + 2 * q + 1) * ld + r0 + g] = v;
  }
}
__global__ void load16_kernel(const double2* src, size_t n2, double* out) {
  double s = 0;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n2; i += (size_t)gridDim.x * blockDim.x) { double2 v = src[i]; s += v.x + v.y; }
  if (s == 1.2345) out[0] = s;
}

int main(int argc, char** argv) {
  const int np = argc > 1 ? atoi(argv[1]) : 2;
  const int same = argc > 2 ? atoi(argv[2]) : 0;
  Shared* sh = (Shared*)mmap(nullptr, sizeof(Shared), PROT_READ | PROT_WRITE, MAP_SHARED | MAP_ANONYMOUS, -1, 0);
  memset((void*)sh, 0, sizeof(Shared));
  for (int r = 1; r < np; r++) { pid_t p = fork(); if (p == 0) { g_rank = r; break; } }
  const int rank = g_rank;
  int ndev = 0;
  CK(cudaGetDeviceCount(&ndev));
  const int dev = same ? 0 : rank % ndev;
  CK(cudaSetDevice(dev));
  const size_t BYTES = 256u << 20;
  double* data; unsigned long long* flags; int* d_to; double* d_out;
  CK(cudaMalloc(&data, BYTES)); CK(cudaMalloc(&flags, 4096)); CK(cudaMalloc(&d_to, 4)); CK(cudaMalloc(&d_out, 8));
  CK(cudaMemset(flags, 0, 4096)); CK(cudaMemset(d_to, 0, 4)); CK(cudaMemset(data, 0, BYTES));
  CK(cudaIpcGetMemHandle(&sh->data[rank], data)); CK(cudaIpcGetMemHandle(&sh->flags[rank], flags));
  CK(cudaDeviceSynchronize());
  host_barrier(sh, np, 0);
  double* pdata[16]; unsigned long long* pflags[16];
  for (int r = 0; r < np; r++) {
    if (r == rank) { pdata[r] = data; pflags[r] = flags; continue; }
    CK(cudaIpcOpenMemHandle((void**)&pdata[r], sh->data[r], cudaIpcMemLazyEnablePeerAccess));
    CK(cudaIpcOpenMemHandle((void**)&pflags[r], sh->flags[r], cudaIpcMemLazyEnablePeerAccess));
  }
  if (rank == 0) printf("np=%d ndev=%d same_device=%d: IPC handles opened on all ranks\n", np, ndev, same);
  host_barrier(sh, np, 1);
  cudaStream_t st; CK(cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking));
  cudaEvent_t e0, e1; CK(cudaEventCreate(&e0)); CK(cudaEventCreate(&e1));
  float ms;
  const int peer = (rank + 1) % np;
  // ---- A: DMA push (rank 0 -> 1), then all ranks at once ----
  for (int pass = 0; pass < 2; pass++) {
    host_barrier(sh, np, 2 + pass);
    if (pass == 1 || rank == 0) {
      CK(cudaMemcpyAsync(pdata[peer], data, BYTES, cudaMemcpyDefault, st));
      CK(cudaEventRecord(e0, st));
      for (int i = 0; i < 5; i++) CK(cudaMemcpyAsync(pdata[peer], data, BYTES, cudaMemcpyDefault, st));
      CK(cudaEventRecord(e1, st)); CK(cudaEventSynchronize(e1)); CK(cudaEventElapsedTime(&ms, e0, e1));
      if (rank == 0) printf("A%d DMA push contiguous 256 MB (%s): %.1f GB/s\n", pass, pass ? "all ranks concurrently" : "rank 0 only", 5 * BYTES / ms / 1e6);
      // strided: 4096 rows of 8192 columns window out of ld = 4112 ... (rows*8 bytes per column)
      const size_t rows = 4096, cols = 4096, ld = 8192;
      CK(cudaEventRecord(e0, st));
      for (int i = 0; i < 5; i++) CK(cudaMemcpy2DAsync(pdata[peer], ld * 8, data, ld * 8, rows * 8, cols, cudaMemcpyDefault, st));
      CK(cudaEventRecord(e1, st)); CK(cudaEventSynchronize(e1)); CK(cudaEventElapsedTime(&ms, e0, e1));
      if (rank == 0) printf("A%d DMA push 2D window 4096x4096 of ld 8192 (134 MB): %.1f GB/s\n", pass, 5 * rows * cols * 8 / ms / 1e6);
      const size_t r2 = 512, c2 = 512;
      CK(cudaEventRecord(e0, st));
      for (int i = 0; i < 20; i++) CK(cudaMemcpy2DAsync(pdata[peer], ld * 8, data, ld * 8, r2 * 8, c2, cudaMemcpyDefault, st));
      CK(cudaEventRecord(e1, st)); CK(cudaEventSynchronize(e1)); CK(cudaEventElapsedTime(&ms, e0, e1));
      if (rank == 0) printf("A%d DMA push 2D window 512x512 (2 MB): %.1f us each\n", pass, ms * 1e3 / 20);
    }
  }
  // ---- D: SM remote stores / loads (rank 0 -> 1) ----
  host_barrier(sh, np, 4);
  if (rank == 0) {
    for (int blocks : {16, 132, 528}) {
      store16_kernel<<<blocks, 256, 0, st>>>((double2*)pdata[peer], BYTES / 16, 1.0);
      CK(cudaEventRecord(e0, st));
      for (int i = 0; i < 3; i++) store16_kernel<<<blocks, 256, 0, st>>>((double2*)pdata[peer], BYTES / 16, 1.0);
      CK(cudaEventRecord(e1, st)); CK(cudaEventSynchronize(e1)); CK(cudaEventElapsedTime(&ms, e0, e1));
      printf("D SM remote store 16B, %d CTAs: %.1f GB/s\n", blocks, 3 * BYTES / ms / 1e6);
    }
    {
      CK(cudaEventRecord(e0, st));
      for (int i = 0; i < 3; i++) store_epi_kernel<<<132, 256, 0, st>>>(pdata[peer], 4096, 4096, 4096, 2.0);
      CK(cudaEventRecord(e1, st)); CK(cudaEventSynchronize(e1)); CK(cudaEventElapsedTime(&ms, e0, e1));
      printf("D SM remote store, epilogue pattern (8B, 64B runs) 4096x4096: %.1f GB/s\n", 3 * 4096.0 * 4096 * 8 / ms / 1e6);
      CK(cudaEventRecord(e0, st));
      for (int i = 0; i < 3; i++) store_epi_kernel<<<132, 256, 0, st>>>(data, 4096, 4096, 4096, 2.0);
      CK(cudaEventRecord(e1, st)); CK(cudaEventSynchronize(e1)); CK(cudaEventElapsedTime(&ms, e0, e1));
      printf("D SM LOCAL store, epilogue pattern 4096x4096: %.1f GB/s\n", 3 * 4096.0 * 4096 * 8 / ms / 1e6);
    }
    for (int blocks : {132, 528}) {
      CK(cudaEventRecord(e0, st));
      for (int i = 0; i < 3; i++) load16_kernel<<<blocks, 256, 0, st>>>((const double2*)pdata[peer], BYTES / 16, d_out);
      CK(cudaEventRecord(e1, st)); CK(cudaEventSynchronize(e1)); CK(cudaEventElapsedTime(&ms, e0, e1));
      printf("D SM remote load 16B, %d CTAs: %.1f GB/s\n", blocks, 3 * BYTES / ms / 1e6);
    }
  }
  // ---- B: flag ping-pong with kernels between rank 0 and 1 ----
  host_barrier(sh, np, 5);
  const int N = same ? 50 : 2000;
  if (rank < 2 && np >= 2) {
    const int other = 1 - rank;
    CK(cudaEventRecord(e0, st));
    for (int i = 1; i <= N; i++) {
      if (rank == 0) { signal_kernel<<<1, 1, 0, st>>>(pflags[other], i); wait_kernel<<<1, 1, 0, st>>>(flags, i, d_to); }
      else { wait_kernel<<<1, 1, 0, st>>>(flags, i, d_to); signal_kernel<<<1, 1, 0, st>>>(pflags[other], i); }
    }
    CK(cudaEventRecord(e1, st)); CK(cudaEventSynchronize(e1)); CK(cudaEventElapsedTime(&ms, e0, e1));
    int to = 0; CK(cudaMemcpy(&to, d_to, 4, cudaMemcpyDeviceToHost));
    if (rank == 0) printf("B kernel flag ping-pong: %.2f us per round trip (%d trips, timeout=%d)\n", ms * 1e3 / N, N, to);
  }
  // ---- C: stream memory operations on peer memory ----
  host_barrier(sh, np, 6);
  if (rank < 2 && np >= 2) {
    const int other = 1 - rank;
    CUstream cs = (CUstream)st;
    CK(cudaMemsetAsync(flags + 8, 0, 8, st)); CK(cudaStreamSynchronize(st));
    host_barrier(sh, 2, 7);
    CK(cudaEventRecord(e0, st));
    for (int i = 1; i <= N && !g_drv_fail; i++) {
      if (rank == 0) { CKD(cuStreamWriteValue64(cs, (CUdeviceptr)(pflags[other] + 8), i, 0)); CKD(cuStreamWaitValue64(cs, (CUdeviceptr)(flags + 8), i, CU_STREAM_WAIT_VALUE_GEQ)); }
      else { CKD(cuStreamWaitValue64(cs, (CUdeviceptr)(flags + 8), i, CU_STREAM_WAIT_VALUE_GEQ)); CKD(cuStreamWriteValue64(cs, (CUdeviceptr)(pflags[other] + 8), i, 0)); }
    }
    if (g_drv_fail) {  // unblock the partner
      CK(cudaMemset(pflags[other] + 8, 0x7f, 8));
      printf("[r%d] C stream memory ops on peer memory: NOT usable\n", rank);
    } else {
      CK(cudaEventRecord(e1, st)); CK(cudaEventSynchronize(e1)); CK(cudaEventElapsedTime(&ms, e0, e1));
      if (rank == 0) printf("C stream-memop flag ping-pong: %.2f us per round trip\n", ms * 1e3 / N);
    }
  } else if (np >= 2) { /* ranks >= 2 skip barrier 7 (it counts 2) */ }
  CK(cudaDeviceSynchronize());
  host_barrier(sh, np, 8);
  if (rank == 0) { printf("probe_p2p done\n"); for (int r = 1; r < np; r++) wait(nullptr); }
  fflush(stdout);
  return 0;
}
