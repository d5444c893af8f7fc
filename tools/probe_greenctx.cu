// Probe: green contexts (SM partitions) driven through runtime-API launches.
// Question: can the deferred ("far") GEMMs be confined to N-8k SMs so that the latency-critical chain kernels (8-CTA cluster,
// 146 KB smem per CTA) always find free SMs instead of waiting ~1 ms for a 128x128 tile to retire?
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o probe_greenctx probe_greenctx.cu -lcuda
#include <cuda.h>
#include <cuda_runtime.h>
#include <cooperative_groups.h>
#include <stdio.h>
#include <stdlib.h>
#include <vector>
#include <set>
namespace cg = cooperative_groups;
#define CK(x) do { cudaError_t e = (x); if (e != cudaSuccess) { printf("CUDA error %s at line %d\n", cudaGetErrorString(e), __LINE__); return 1; } } while (0)
#define CKD(x) do { CUresult e = (x); if (e != CUDA_SUCCESS) { const char* s; cuGetErrorString(e, &s); printf("driver error %s at line %d\n", s, __LINE__); return 1; } } while (0)

__global__ void smid_kernel(int* out) {
  extern __shared__ double sm[];
  unsigned id;
  asm volatile("mov.u32 %0, %%smid;" : "=r"(id));
  if (threadIdx.x == 0) out[blockIdx.x] = (int)id;
  sm[threadIdx.x] = id;
}
__global__ void spin_kernel(long long cycles, int* out) {
  extern __shared__ double sm[];
  unsigned id;
  asm volatile("mov.u32 %0, %%smid;" : "=r"(id));
  if (threadIdx.x == 0 && out) out[blockIdx.x] = (int)id;
  sm[threadIdx.x] = 1.0;
  const long long t0 = clock64();
  while (clock64() - t0 < cycles) { }
}
__global__ void __cluster_dims__(8, 1, 1) cluster_kernel(long long cycles, int* out) {
  extern __shared__ double sm[];
  cg::cluster_group cl = cg::this_cluster();
  unsigned id;
  asm volatile("mov.u32 %0, %%smid;" : "=r"(id));
  if (threadIdx.x == 0 && out) out[blockIdx.x] = (int)id;
  sm[threadIdx.x] = 1.0;
  cl.sync();
  const long long t0 = clock64();
  while (clock64() - t0 < cycles) { }
  cl.sync();
}

int main() {
  CK(cudaSetDevice(0));
  CK(cudaFree(0));
  CUdevice dev;
  CKD(cuDeviceGet(&dev, 0));
  CUdevResource all;
  CKD(cuDeviceGetDevResource(dev, &all, CU_DEV_RESOURCE_TYPE_SM));
  printf("device SMs: %u\n", all.sm.smCount);
  unsigned nb = 0;
  CKD(cuDevSmResourceSplitByCount(nullptr, &nb, &all, nullptr, 0, 8));
  printf("groups of >=8: %u\n", nb);
  std::vector<CUdevResource> groups(nb);
  CUdevResource rem;
  CKD(cuDevSmResourceSplitByCount(groups.data(), &nb, &all, &rem, 0, 8));
  printf("split: %u groups, sizes:", nb);
  for (unsigned i = 0; i < nb; i++) printf(" %u", groups[i].sm.smCount);
  printf(" remaining %u\n", rem.sm.smCount);
  for (int reserve_groups = 1; reserve_groups <= 2; reserve_groups++) {
    // far partition = all groups but the first `reserve_groups` (+ the remainder)
    std::vector<CUdevResource> farres(groups.begin() + reserve_groups, groups.end());
    if (rem.sm.smCount) farres.push_back(rem);
    CUdevResourceDesc desc;
    CUresult r = cuDevResourceGenerateDesc(&desc, farres.data(), (unsigned)farres.size());
    if (r != CUDA_SUCCESS) {
      const char* s; cuGetErrorString(r, &s);
      printf("GenerateDesc over %zu resources failed: %s -- trying without the remainder\n", farres.size(), s);
      farres.pop_back();
      CKD(cuDevResourceGenerateDesc(&desc, farres.data(), (unsigned)farres.size()));
    }
    CUgreenCtx g;
    CKD(cuGreenCtxCreate(&g, desc, dev, CU_GREEN_CTX_DEFAULT_STREAM));
    CUstream gs;
    CKD(cuGreenCtxStreamCreate(&gs, g, CU_STREAM_NON_BLOCKING, 0));
    cudaStream_t far = (cudaStream_t)gs;
    int lo, hi;
    CK(cudaDeviceGetStreamPriorityRange(&lo, &hi));
    cudaStream_t chain;
    CK(cudaStreamCreateWithPriority(&chain, cudaStreamNonBlocking, hi));
    int* d_ids; CK(cudaMalloc(&d_ids, 4096 * 4));
    const int smem = 160 * 1024;
    CK(cudaFuncSetAttribute(smid_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    CK(cudaFuncSetAttribute(spin_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    CK(cudaFuncSetAttribute(cluster_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    // 1. which SMs does a runtime launch on the green stream use?
    CK(cudaMemset(d_ids, 0xff, 4096 * 4));
    smid_kernel<<<1024, 128, smem, far>>>(d_ids);
    CK(cudaStreamSynchronize(far));
    std::vector<int> ids(1024);
    CK(cudaMemcpy(ids.data(), d_ids, 1024 * 4, cudaMemcpyDeviceToHost));
    std::set<int> farset(ids.begin(), ids.end());
    printf("[reserve %d groups] green stream launch ran on %zu distinct SMs\n", reserve_groups, farset.size());
    // 2. chain latency: cluster kernel (8 CTAs x 146 KB) on the primary-context stream while the far partition is saturated
    cudaEvent_t e0, e1; CK(cudaEventCreate(&e0)); CK(cudaEventCreate(&e1));
    float ms;
    for (int mode = 0; mode < 3; mode++) {
      // mode 0: idle GPU; mode 1: far work on the green stream; mode 2: far work on an ordinary low-priority stream (today's schedule)
      cudaStream_t lowp;
      CK(cudaStreamCreateWithPriority(&lowp, cudaStreamNonBlocking, lo));
      cudaStream_t fs = mode == 1 ? far : lowp;
      const long long far_cycles = 4000000;  // ~2 ms per CTA
      if (mode) spin_kernel<<<132 * 4, 128, smem, fs>>>(far_cycles, nullptr);
      // give the far kernel time to occupy the machine
      spin_kernel<<<1, 32, 1024, chain>>>(400000, nullptr);
      CK(cudaEventRecord(e0, chain));
      for (int i = 0; i < 10; i++) cluster_kernel<<<8, 256, 146 * 1024, chain>>>(20000, d_ids);
      CK(cudaEventRecord(e1, chain));
      CK(cudaEventSynchronize(e1));
      CK(cudaEventElapsedTime(&ms, e0, e1));
      CK(cudaDeviceSynchronize());
      CK(cudaMemcpy(ids.data(), d_ids, 8 * 4, cudaMemcpyDeviceToHost));
      int inside = 0;
      for (int i = 0; i < 8; i++) inside += farset.count(ids[i]) ? 1 : 0;
      printf("  mode %d (%s): 10 chain cluster kernels (10 us each) took %.1f us; last cluster on SMs", mode,
             mode == 0 ? "idle" : mode == 1 ? "far work in green partition" : "far work on low-priority stream", ms * 1e3);
      for (int i = 0; i < 8; i++) printf(" %d", ids[i]);
      printf("  (%d of 8 inside the far partition)\n", inside);
      CK(cudaStreamDestroy(lowp));
    }
    // 3. does a full-machine kernel on the primary context still get all SMs while the green context exists?
    CK(cudaMemset(d_ids, 0xff, 4096 * 4));
    smid_kernel<<<1024, 128, smem, chain>>>(d_ids);
    CK(cudaStreamSynchronize(chain));
    ids.resize(1024);
    CK(cudaMemcpy(ids.data(), d_ids, 1024 * 4, cudaMemcpyDeviceToHost));
    std::set<int> allset(ids.begin(), ids.end());
    printf("  primary-context launch ran on %zu distinct SMs\n", allset.size());
    CK(cudaStreamDestroy(chain));
    CKD(cuStreamDestroy(gs));
    CKD(cuGreenCtxDestroy(g));
    CK(cudaFree(d_ids));
  }
  printf("probe_greenctx done\n");
  return 0;
}
