// 64x64x64 DMMA tile products out of shared memory (256 threads), shared by the cluster base case (leaf.cu) and the block Jacobi
// eigensolver (syevj.cu).  Internal linkage, as before the move: every kernel that uses them inlines its own copy.
#pragma once
#include "common.cuh"

namespace {
constexpr int TLD = 68;            // DMMA tiles: rows of 64 k-contiguous doubles, padded so that fragment loads
                                   // (row g, k q) of a half-warp touch 16 distinct bank pairs
constexpr int TILE_DOUBLES = 64 * TLD;

__device__ __forceinline__ void dmma884(double& c0, double& c1, double a, double b) {
  asm("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};" : "+d"(c0), "+d"(c1) : "d"(a), "d"(b));
}
// copy a 64 (k) x 64 (cols) global block (k contiguous, 16-byte aligned, even ld) into a padded tile: dst[col * TLD + k]
__device__ __forceinline__ void tile_load(double* __restrict__ dst, const double* src, long long ld) {
  const int k2 = (threadIdx.x & 31) * 2, c0 = threadIdx.x >> 5;
  double2 v[8];
#pragma unroll
  for (int r = 0; r < 8; r++) v[r] = __ldcg(reinterpret_cast<const double2*>(src + k2 + (long long)(c0 + 8 * r) * ld));
#pragma unroll
  for (int r = 0; r < 8; r++) *reinterpret_cast<double2*>(dst + (c0 + 8 * r) * TLD + k2) = v[r];
}
// acc += As^T Bs for the 64x64 tile; warp w owns rows (w&1)*32.., cols (w>>1)*16..; As/Bs: [row][k] padded tiles.
__device__ __forceinline__ void tile_mma(double (&acc)[4][2][2], const double* As, const double* Bs) {
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, g = lane >> 2, q = lane & 3;
  const double* ap = As + ((w & 1) * 32 + g) * TLD + q;
  const double* bp = Bs + ((w >> 1) * 16 + g) * TLD + q;
#pragma unroll 4
  for (int k0 = 0; k0 < 64; k0 += 4) {
    double af[4], bf[2];
#pragma unroll
    for (int i = 0; i < 4; i++) af[i] = ap[i * 8 * TLD + k0];
#pragma unroll
    for (int j = 0; j < 2; j++) bf[j] = bp[j * 8 * TLD + k0];
#pragma unroll
    for (int i = 0; i < 4; i++)
#pragma unroll
      for (int j = 0; j < 2; j++) dmma884(acc[i][j][0], acc[i][j][1], af[i], bf[j]);
  }
}
__device__ __forceinline__ void acc_zero(double (&acc)[4][2][2]) {
#pragma unroll
  for (int i = 0; i < 4; i++)
#pragma unroll
    for (int j = 0; j < 2; j++) acc[i][j][0] = acc[i][j][1] = 0.0;
}
#define TILE_ROW(i) ((w & 1) * 32 + (i) * 8 + g)
#define TILE_COL(j, e) ((w >> 1) * 16 + (j) * 8 + 2 * q + (e))
// accumulators -> shared tile in [col][row] order (row contiguous), scaled
__device__ __forceinline__ void acc_to_smem_colmajor(const double (&acc)[4][2][2], double* __restrict__ sC, double scale) {
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, g = lane >> 2, q = lane & 3;
#pragma unroll
  for (int i = 0; i < 4; i++)
#pragma unroll
    for (int j = 0; j < 2; j++)
#pragma unroll
      for (int e = 0; e < 2; e++) sC[TILE_COL(j, e) * TLD + TILE_ROW(i)] = scale * acc[i][j][e];
}
// accumulators -> shared tile in [row][col] order (used as the next A operand: rows = output rows, k = columns)
__device__ __forceinline__ void acc_to_smem_rowmajor(const double (&acc)[4][2][2], double* __restrict__ sC, double scale) {
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, g = lane >> 2, q = lane & 3;
#pragma unroll
  for (int i = 0; i < 4; i++)
#pragma unroll
    for (int j = 0; j < 2; j++)
#pragma unroll
      for (int e = 0; e < 2; e++) sC[TILE_ROW(i) * TLD + TILE_COL(j, e)] = scale * acc[i][j][e];
}
}  // namespace
