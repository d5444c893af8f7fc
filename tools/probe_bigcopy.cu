// Probe: does a flag written after a LARGE peer copy ever overtake the tail of the data?  (2 processes, 2 GPUs)
// rank 0: [memcpy N bytes to rank 1's buffer] [cuStreamWriteValue64 flag on rank 1]   rank 1: [cuStreamWaitValue64] [kernel counts wrong words, tail first]
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o probe_bigcopy probe_bigcopy.cu -lcuda
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <sys/mman.h>
#include <sys/wait.h>
#include <unistd.h>
static int g_rank = 0;
#define CK(x) do { cudaError_t e = (x); if (e != cudaSuccess) { printf("[r%d] CUDA error %s at line %d\n", g_rank, cudaGetErrorString(e), __LINE__); fflush(stdout); _exit(2); } } while (0)
#define CKD(x) do { CUresult e = (x); if (e != CUDA_SUCCESS) { printf("[r%d] driver error %d at line %d\n", g_rank, (int)e, __LINE__); fflush(stdout); _exit(2); } } while (0)
struct Shared { volatile int barrier[256]; cudaIpcMemHandle_t data[2], flags[2]; };
static void hb(Shared* sh, int idx) { __sync_fetch_and_add(&sh->barrier[idx], 1); while (sh->barrier[idx] < 2) usleep(50); }
__global__ void fill_kernel(unsigned long long* p, size_t n, unsigned long long v) {
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) p[i] = v + i;
}
// walk the buffer from the END (the tail of the copy is what a racing reader would miss)
__global__ void check_kernel(const unsigned long long* p, size_t n, unsigned long long v, unsigned long long* bad) {
  unsigned long long cnt = 0;
  for (size_t k = blockIdx.x * (size_t)blockDim.x + threadIdx.x; k < n; k += (size_t)gridDim.x * blockDim.x) {
    const size_t i = n - 1 - k;
    unsigned long long got;
    asm volatile("ld.global.cg.u64 %0, [%1];" : "=l"(got) : "l"(p + i));
    if (got != v + i) cnt++;
  }
  if (cnt) atomicAdd(bad, cnt);
}
int main() {
  Shared* sh = (Shared*)mmap(nullptr, sizeof(Shared), PROT_READ | PROT_WRITE, MAP_SHARED | MAP_ANONYMOUS, -1, 0);
  memset((void*)sh, 0, sizeof(Shared));
  if (fork() == 0) g_rank = 1;
  const int rank = g_rank;
  CK(cudaSetDevice(rank));
  const size_t CAP = (size_t)9 << 30;
  unsigned long long *data, *flags, *bad;
  CK(cudaMalloc(&data, CAP)); CK(cudaMalloc(&flags, 4096)); CK(cudaMalloc(&bad, 8));
  CK(cudaMemset(flags, 0, 4096));
  CK(cudaIpcGetMemHandle(&sh->data[rank], data)); CK(cudaIpcGetMemHandle(&sh->flags[rank], flags));
  hb(sh, 0);
  unsigned long long *pdata, *pflags;
  CK(cudaIpcOpenMemHandle((void**)&pdata, sh->data[1 - rank], cudaIpcMemLazyEnablePeerAccess));
  CK(cudaIpcOpenMemHandle((void**)&pflags, sh->flags[1 - rank], cudaIpcMemLazyEnablePeerAccess));
  cudaStream_t st; CK(cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking));
  const size_t sizes[] = {(size_t)1 << 30, ((size_t)1 << 31) - 65536, (size_t)1 << 31, ((size_t)1 << 31) + 65536, (size_t)1 << 32, (size_t)1 << 33};
  int bi = 1;
  unsigned long long seq = 0;
  for (int mode = 0; mode < 2; mode++)  // 0: one copy; 1: 512 MiB pieces
    for (size_t bytes : sizes)
      for (int rep = 0; rep < 4; rep++) {
        seq++;
        const size_t n = bytes / 8;
        if (rank == 0) fill_kernel<<<592, 256, 0, st>>>(data, n, seq << 40);
        else CK(cudaMemsetAsync(data, 0, bytes, st));
        CK(cudaStreamSynchronize(st));
        hb(sh, bi++);
        if (rank == 0) {
          if (mode == 0) CK(cudaMemcpyAsync(pdata, data, bytes, cudaMemcpyDefault, st));
          else for (size_t off = 0; off < bytes; off += (size_t)512 << 20) CK(cudaMemcpyAsync((char*)pdata + off, (char*)data + off, bytes - off < ((size_t)512 << 20) ? bytes - off : (size_t)512 << 20, cudaMemcpyDefault, st));
          CKD(cuStreamWriteValue64((CUstream)st, (CUdeviceptr)pflags, seq, 0));
          CK(cudaStreamSynchronize(st));
        } else {
          CK(cudaMemsetAsync(bad, 0, 8, st));
          CKD(cuStreamWaitValue64((CUstream)st, (CUdeviceptr)flags, seq, CU_STREAM_WAIT_VALUE_GEQ));
          check_kernel<<<592, 256, 0, st>>>(data, n, seq << 40, bad);
          unsigned long long h = 0;
          CK(cudaMemcpyAsync(&h, bad, 8, cudaMemcpyDeviceToHost, st));
          CK(cudaStreamSynchronize(st));
          printf("mode %d bytes %zu (2^31%+lld) rep %d: %llu wrong words\n", mode, bytes, (long long)bytes - (1ll << 31), rep, h);
        }
        hb(sh, bi++);
      }
  if (rank == 0) wait(nullptr);
  fflush(stdout);
  return 0;
}
