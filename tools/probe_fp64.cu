// Microbenchmark: FP64 pipe ceilings on sm_90a (DFMA vs DMMA.8x8x4). Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o probe_fp64 probe_fp64.cu
#include <cstdio>
#include <cuda_runtime.h>
#define CK(x) do{cudaError_t e=(x); if(e!=cudaSuccess){printf("CUDA error %s at %d\n",cudaGetErrorString(e),__LINE__); return 1;}}while(0)

template<int ILP>
__global__ void dfma_kernel(double* out, int iters, double s){
  double acc[ILP];
  #pragma unroll
  for(int i=0;i<ILP;i++) acc[i]=threadIdx.x*1e-9+i;
  double a=s, b=1.0-s*1e-3;
  for(int it=0;it<iters;it++){
    #pragma unroll
    for(int i=0;i<ILP;i++) acc[i]=fma(acc[i],b,a);
  }
  double r=0;
  #pragma unroll
  for(int i=0;i<ILP;i++) r+=acc[i];
  if(r==123.456) out[0]=r;
}

template<int NACC>
__global__ void dmma_kernel(double* out, int iters, double s){
  double c[NACC][2];
  #pragma unroll
  for(int i=0;i<NACC;i++){c[i][0]=0;c[i][1]=0;}
  double a=s+threadIdx.x*1e-6, b=1.0-s;
  for(int it=0;it<iters;it++){
    #pragma unroll
    for(int i=0;i<NACC;i++)
      asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1},{%2},{%3},{%0,%1};"
                   :"+d"(c[i][0]),"+d"(c[i][1]):"d"(a),"d"(b));
  }
  double r=0;
  #pragma unroll
  for(int i=0;i<NACC;i++) r+=c[i][0]+c[i][1];
  if(r==123.456) out[0]=r;
}

template<typename F>
float time_it(F f){
  cudaEvent_t e0,e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
  f(); cudaDeviceSynchronize();
  cudaEventRecord(e0); f(); cudaEventRecord(e1); cudaEventSynchronize(e1);
  float ms; cudaEventElapsedTime(&ms,e0,e1); return ms;
}

int main(){
  cudaDeviceProp p; CK(cudaGetDeviceProperties(&p,0));
  printf("device %s SMs=%d clock=%d kHz\n",p.name,p.multiProcessorCount,p.clockRate);
  double* out; CK(cudaMalloc(&out,8));
  int sms=p.multiProcessorCount;
  int iters=20000;
  for(int tpb: {128,256,512,1024}){
    for(int bps: {1,2}){
      int blocks=sms*bps;
      float ms=time_it([&]{dfma_kernel<8><<<blocks,tpb>>>(out,iters,0.5);});
      double fl=2.0*8*iters*(double)tpb*blocks;
      printf("DFMA ilp8 tpb=%d bps=%d: %.3f ms  %.2f TFLOP/s\n",tpb,bps,ms,fl/ms/1e9);
    }
  }
  for(int tpb: {32,64,128,256,512,1024}){
    int blocks=sms;
    float ms=time_it([&]{dmma_kernel<8><<<blocks,tpb>>>(out,iters,0.5);});
    double fl=2.0*256*8*iters*(double)(tpb/32)*blocks;
    printf("DMMA884 acc8 tpb=%d: %.3f ms  %.2f TFLOP/s\n",tpb,ms,fl/ms/1e9);
    ms=time_it([&]{dmma_kernel<2><<<blocks,tpb>>>(out,iters,0.5);});
    fl=2.0*256*2*iters*(double)(tpb/32)*blocks;
    printf("DMMA884 acc2 tpb=%d: %.3f ms  %.2f TFLOP/s\n",tpb,ms,fl/ms/1e9);
    ms=time_it([&]{dmma_kernel<1><<<blocks,tpb>>>(out,iters,0.5);});
    fl=2.0*256*1*iters*(double)(tpb/32)*blocks;
    printf("DMMA884 acc1 tpb=%d: %.3f ms  %.2f TFLOP/s (latency-bound: %.1f cyc/mma @1.9GHz)\n",tpb,ms,fl/ms/1e9, ms*1e-3*1.9e9/iters);
  }
  // sustained run ~2 s to see power-capped rate
  {
    int blocks=sms, tpb=256; int it2=iters*50;
    float ms=time_it([&]{dmma_kernel<8><<<blocks,tpb>>>(out,it2,0.5);});
    double fl=2.0*256*8*it2*(double)(tpb/32)*blocks;
    printf("DMMA884 sustained tpb=256: %.3f ms  %.2f TFLOP/s\n",ms,fl/ms/1e9);
    ms=time_it([&]{dfma_kernel<8><<<blocks*2,512>>>(out,it2,0.5);});
    fl=2.0*8*it2*512.0*blocks*2;
    printf("DFMA sustained: %.3f ms  %.2f TFLOP/s\n",ms,fl/ms/1e9);
  }
  return 0;
}
