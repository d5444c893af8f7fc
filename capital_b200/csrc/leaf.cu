// Bottom of the CholInv recursion: potrf('U') + trtri('U','N') of one diagonal block.  Replaces the LAPACKE_dpotrf /
// LAPACKE_dtrtri pair the reference calls on its gathered base-case block (cholinv/policy.h:199-201,
// lapack/interface.hpp:30-58); unlike the reference the pivot sign is checked and reported (CAPITAL_ERR_NOT_SPD).
//
// Two kernels share one device routine:
//   leaf_kernel      one CTA, nb <= 64, everything in shared memory.
//   basecase_kernel  one thread-block cluster (CW = 2, 4 or 8 CTAs) for nb = 64 t (t <= 8): blocked right-looking Cholesky
//                    with 64-wide panels -- diagonal block by the leaf routine, row panel and trailing update as 64x64x64
//                    DMMA tile products spread over the cluster, hardware cluster barriers between phases -- followed
//                    by the blocked triangular inverse.  One launch replaces ~60 latency-bound launches of the
//                    recursion below 512, where leaves and small GEMMs are latency-bound.
// Both take a batch of independent matrices (cholinv_factor_batched, api.cu): matrix b is blockIdx.x of the leaf kernel and
// blockIdx.y of the cluster kernel (clusters stay along x), at per-matrix strides, with its own info[b].  The width CW only
// decides which CTA computes which tile; every tile keeps its k range and k order, so a matrix gets the same bits at every width.
// The critical path of a leaf is the pivot chain (64 dependent rsqrt + rank-1 updates), so the leaf keeps all
// 256 threads on a fixed 16x16 grid (no index division), scales the pivot row with two warps, and uses one
// rsqrt per pivot instead of a sqrt and a divide.
#include "common.cuh"
#include "tile64.cuh"
#include <cooperative_groups.h>
#include <cfloat>
#include <stdlib.h>
#include <type_traits>
namespace cg = cooperative_groups;

namespace {
constexpr int LD = LEAF_MAX + 1;   // leaf arrays: conflict-free row and column walks

// 1/sqrt(d) off the critical path's slow library routine: FP32 seed + two FP64 Newton steps (relative error ~1e-16 for
// d inside the FP32 range; outside it the library routine is used)
__device__ __forceinline__ double fast_rsqrt(double d) {
  if (!(d > 1e-30 && d < 1e30)) return rsqrt(d);
  double y = (double)rsqrtf((float)d);
  const double h = 0.5 * d;
  y = y * fma(-h, y * y, 1.5);  // three dependent FP64 ops per Newton step
  y = y * fma(-h, y * y, 1.5);
  return y;
}

// ---- leaf: factor + invert an nb x nb block held in shared memory ---------------------------------------------
// a : in  upper triangle of the SPD block (destroyed), out R^{-1} (upper, zeros below)
// r : out R (upper, zeros below)
// t : scratch
__device__ void leaf_factor_invert(int nb, double* __restrict__ a, double* __restrict__ r, double* __restrict__ t, int* info,
                                   int pivot_base) {
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  for (int k = 0; k < nb; k++) {
    if (tid < 64 && tid >= k && tid < nb) {
      double d = a[k + k * LD];
      if (!(d > 0.0)) {
        if (tid == k) atomicCAS(info, 0, pivot_base + k + 1);
        d = 1.0;
      }
      const double rs = rsqrt(d);
      r[k + tid * LD] = (tid == k) ? d * rs : a[k + tid * LD] * rs;
    }
    __syncthreads();
#pragma unroll
    for (int ia = 0; ia < 4; ia++) {
      const int i = ty + 16 * ia;
      if (i > k && i < nb) {
        const double ri = r[k + i * LD];
#pragma unroll
        for (int jb = 0; jb < 4; jb++) {
          const int j = tx + 16 * jb;
          if (j >= i && j < nb) a[i + j * LD] -= ri * r[k + j * LD];
        }
      }
    }
    __syncthreads();
  }
  // zero the strictly lower part of r, start the inverse with the reciprocal diagonal
#pragma unroll
  for (int ia = 0; ia < 4; ia++) {
    const int i = ty + 16 * ia;
#pragma unroll
    for (int jb = 0; jb < 4; jb++) {
      const int j = tx + 16 * jb;
      if (i < nb && j < nb) {
        if (i > j) r[i + j * LD] = 0.0;
        a[i + j * LD] = (i == j) ? 1.0 / r[i + i * LD] : 0.0;
      }
    }
  }
  __syncthreads();
  // recursive doubling: X12 = -X11 R12 X22 for block sizes 1, 2, 4, ...
  int lg = 0;
  for (int bs = 1; bs < nb; bs <<= 1, lg++) {
    const int span = 2 * bs;
    const int npairs = (nb + span - 1) / span;
    const int per = bs * bs, total = npairs * per;
    for (int idx = tid; idx < total; idx += 256) {  // T = X11 R12
      const int p = idx >> (2 * lg), e = idx & (per - 1);
      const int li = e & (bs - 1), lj = e >> lg;
      const int o = p * span, i = o + li, j = o + bs + lj;
      if (j < nb) {
        double s = 0.0;
        const int kend = o + bs;
        for (int k = i; k < kend; k++) s += a[i + k * LD] * r[k + j * LD];
        t[i + j * LD] = s;
      }
    }
    __syncthreads();
    for (int idx = tid; idx < total; idx += 256) {  // X12 = -T X22
      const int p = idx >> (2 * lg), e = idx & (per - 1);
      const int li = e & (bs - 1), lj = e >> lg;
      const int o = p * span, i = o + li, j = o + bs + lj;
      if (j < nb) {
        double s = 0.0;
        for (int k = o + bs; k <= j; k++) s += t[i + k * LD] * a[k + j * LD];
        a[i + j * LD] = -s;
      }
    }
    __syncthreads();
  }
}

__device__ __forceinline__ void leaf_load(int nb, const double* W, long long ldw, double* __restrict__ a) {
  for (int idx = threadIdx.x; idx < nb * nb; idx += 256) {
    const int i = idx % nb, j = idx / nb;
    a[i + j * LD] = (i <= j) ? __ldcg(W + i + (long long)j * ldw) : 0.0;
  }
}
__device__ __forceinline__ void leaf_store(int nb, const double* a, const double* r, double* __restrict__ R,
                                           long long ldr, double* __restrict__ Ri, long long ldri, double* __restrict__ RiT,
                                           long long ldrit) {
  for (int idx = threadIdx.x; idx < nb * nb; idx += 256) {
    const int i = idx % nb, j = idx / nb;
    R[i + (long long)j * ldr] = r[i + j * LD];
    Ri[i + (long long)j * ldri] = a[i + j * LD];
  }
  if (RiT != nullptr) {
    for (int idx = threadIdx.x; idx < nb * nb; idx += 256) {
      const int j = idx % nb, i = idx / nb;  // RiT(j, i) = Ri(i, j)
      RiT[j + (long long)i * ldrit] = a[i + j * LD];
    }
  }
}

__global__ void __launch_bounds__(256, 1)
    leaf_kernel(int nb, const double* W, long long ldw, double* __restrict__ R, long long ldr, double* __restrict__ Ri,
                long long ldri, double* __restrict__ RiT, long long ldrit, int* __restrict__ info, BatchStrides bs,
                int pivot_base) {
  extern __shared__ double sm[];
  double* a = sm;
  double* r = sm + LEAF_MAX * LD;
  double* t = sm + 2 * LEAF_MAX * LD;
  const long long b = blockIdx.x;
  W += b * bs.w; R += b * bs.r; Ri += b * bs.ri; info += b;
  if (RiT != nullptr) RiT += b * bs.rit;
  leaf_load(nb, W, ldw, a);
  __syncthreads();
  leaf_factor_invert(nb, a, r, t, info, pivot_base);
  leaf_store(nb, a, r, R, ldr, Ri, ldri, RiT, ldrit);
}

// ---- 64x64 tile stores (the products themselves: tile64.cuh) ------------------------------------------------
// global(64 x 64 block, column-major) = [beta * global +] sC ([col][row]) with 16-byte coalesced accesses
template <bool ACCUM>
__device__ __forceinline__ void tile_store(double* __restrict__ dst, long long ld, const double* sC) {
  const int r2 = (threadIdx.x & 31) * 2, c0 = threadIdx.x >> 5;
#pragma unroll
  for (int r = 0; r < 8; r++) {
    const int c = c0 + 8 * r;
    double2 v = *reinterpret_cast<const double2*>(sC + c * TLD + r2);
    double2* p = reinterpret_cast<double2*>(dst + r2 + (long long)c * ld);
    if (ACCUM) { const double2 o = __ldcg(p); v.x += o.x; v.y += o.y; }
    *p = v;
  }
}
// transposed store: global(col-block rows, row-block cols) = sC^T, reading sC ([row][col] order) so that accesses stay coalesced
__device__ __forceinline__ void tile_store_from_rowmajor(double* __restrict__ dst, long long ld, const double* sCr) {
  // sCr[row * TLD + col] holds value(row, col); we write dst(col, row) = value(row, col): dst column index = row
  const int c2 = (threadIdx.x & 31) * 2, r0 = threadIdx.x >> 5;
#pragma unroll
  for (int r = 0; r < 8; r++) {
    const int row = r0 + 8 * r;
    const double2 v = *reinterpret_cast<const double2*>(sCr + row * TLD + c2);
    *reinterpret_cast<double2*>(dst + c2 + (long long)row * ld) = v;
  }
}

// ---- fast 64 x 64 leaf: two warp-resident 32 x 32 factor+invert steps glued by DMMA products ------------------
// The pivot chain is the critical path of the whole factorization (16384 dependent pivots at n = 16384).  A block-wide
// formulation pays two __syncthreads and several shared-memory round trips per pivot; here
// a single warp holds a 32 x 32 block in registers (lane j = column j), pivots are broadcast by shuffles, and the
// reciprocal square root is an FP32 seed + two FP64 Newton steps: no barrier in the chain.
__device__ __forceinline__ double shfl_d(double v, int src) { return __shfl_sync(0xffffffffu, v, src); }

// compile-time loop: register arrays must only ever be indexed by constants (a loop the unroller leaves rolled would push
// them to local memory)
template <int I, int END, int STEP = 1, typename F>
__device__ __forceinline__ void static_for(F&& f) {
  if constexpr (I < END) {
    f(std::integral_constant<int, I>{});
    static_for<I + STEP, END, STEP>(f);
  }
}

// c[i] = A(i, lane) (upper part meaningful) -> R written to sRb (element (i, j) at sRb[j * TLD + i]), x[i] = Rinv(i, lane).
// ub: 896 doubles of shared scratch (the scaled pivot row is broadcast through it: one conflict-free store and
// pipelined broadcast loads per pivot instead of 2 x 31 dependent shuffles).  The next pivot's rsqrt is started as
// soon as its diagonal entry is final, so it overlaps with the rest of the rank-1 update.
__device__ __forceinline__ void warp_potrf_trtri_32(double (&c)[32], double* __restrict__ sRb, double* __restrict__ sXb, double* __restrict__ sXTb,
                                                    double* __restrict__ ub, int lane, int* info, int pivot_base, long long* dbg2) {
  double myrs = 0.0;
  if (dbg2 && lane == 0) dbg2[0] = clock64();
  // Two pivots per step.  With a = A(k,k), l = A(k,k+1), b = A(k+1,k+1) the second pivot is det / a, det = a b - l^2, so
  // rsqrt(a) and rsqrt(det) are independent and overlap: one rsqrt latency per TWO pivots on the chain.
  //   R(k,k) = a ra          R(k,j)   = A(k,j) ra                       (ra = 1/sqrt(a))
  //   R(k+1,k+1) = det rdet ra         R(k+1,j) = (A(k+1,j) - l ra R(k,j)) sqrt(a) rdet   (rdet = 1/sqrt(det))
  // a b and l^2 leave the double range long before the matrix does (diagonal entries below ~1e-154 or above ~1e154, or a graded
  // block whose neighbouring diagonal entries multiply past 2^+-1024).  Pivots never exceed their diagonal entries and fall 2^111
  // below them only in a matrix that is singular to working precision, so a block whose diagonal lies in [2^-400, 2^400] -- every
  // block of ordinary scale -- keeps all pairs in range.  Any other block is equilibrated first: S = D^-1 A D^-1 with
  // D = diag(2^e), diag(S) in [1, 4), exact in powers of two; then R = R(S) D and 1/R(k,k) = 2^-e_k / R_S(k,k).  The vote makes
  // the branch warp-uniform, and the pivot loop itself is the same for both.
  double dl = 0.0;  // A(lane, lane)
  static_for<0, 32>([&](auto ic) { constexpr int i = decltype(ic)::value; if (lane == i) dl = c[i]; });
  const bool equil = !__all_sync(0xffffffffu, dl >= 0x1p-400 && dl <= 0x1p400);
  double fl = 1.0;  // 2^-e of this lane's row and column (1 for a non-positive diagonal entry, which is then reported as before)
  if (equil) {
    if (dl > 0.0 && dl <= DBL_MAX) fl = ldexp(1.0, -(ilogb(dl) >> 1));
    static_for<0, 32>([&](auto ic) { constexpr int i = decltype(ic)::value; c[i] = c[i] * shfl_d(fl, i) * fl; });
  }
  double a = shfl_d(c[0], 0), l = shfl_d(c[0], 1), b = shfl_d(c[1], 1);
  static_for<0, 32, 2>([&](auto kc) {
    constexpr int k = decltype(kc)::value;
    if (!(a > 0.0)) { if (lane == k) atomicCAS(info, 0, pivot_base + k + 1); a = 1.0; }
    double det = fma(b, a, -(l * l));
    if (!(det > 0.0)) { if (lane == k + 1) atomicCAS(info, 0, pivot_base + k + 2); det = 1.0; }
    const double ra = fast_rsqrt(a), rdet = fast_rsqrt(det);
    const double sa = a * ra, lk = l * ra, rs2 = sa * rdet;
    const double u0 = (lane > k) ? c[k] * ra : (lane == k ? sa : 0.0);                                  // R(k, lane)
    const double t1 = fma(-lk, u0, c[k + 1]);
    const double u1 = (lane > k + 1) ? t1 * rs2 : (lane == k + 1 ? det * rdet * ra : 0.0);            // R(k+1, lane)
    c[k] = u0;
    c[k + 1] = u1;
    if (lane == k) myrs = ra;
    if (lane == k + 1) myrs = rs2;
    double* row0 = ub + (k & 2) * 32;
    double* row1 = row0 + 32;
    row0[lane] = u0;
    row1[lane] = u1;
    __syncwarp();
    if constexpr (k + 2 < 32) {
      c[k + 2] = fma(-row1[k + 2], u1, fma(-row0[k + 2], u0, c[k + 2]));
      c[k + 3] = fma(-row1[k + 3], u1, fma(-row0[k + 3], u0, c[k + 3]));
      a = shfl_d(c[k + 2], k + 2);  // next pair: final already
      l = shfl_d(c[k + 2], k + 3);
      b = shfl_d(c[k + 3], k + 3);
      static_for<k + 4, 32>([&](auto ic) {  // rank-2 update of column `lane`
        constexpr int i = decltype(ic)::value;
        c[i] = fma(-row1[i], u1, fma(-row0[i], u0, c[i]));
      });
    }
  });
  if (equil) {
    const double gl = 1.0 / fl;  // 2^e_lane, exact
    static_for<0, 32>([&](auto ic) { constexpr int i = decltype(ic)::value; c[i] *= gl; });
    myrs *= fl;
  }
  if (dbg2 && lane == 0) dbg2[1] = clock64();
#pragma unroll
  for (int i = 0; i < 32; i++) sRb[lane * TLD + i] = c[i];  // c[i] == 0 below the diagonal by construction (u = 0 for lane < k)
  __syncwarp();
  // ---- inverse.  Phase A: the two 16 x 16 diagonal blocks at once (half-warp g owns block g; lane = column), so the
  // back-substitution chain is 15 steps instead of 31.  xl[r] = X(16 g + r, lane).
  const int g16 = lane >> 4, jl = lane & 15, base = 16 * g16;
  double xl[16];
  static_for<0, 16>([&](auto rc_) { constexpr int r = decltype(rc_)::value; xl[r] = (r == jl) ? myrs : 0.0; });
  static_for<0, 15>([&](auto sc) {
    constexpr int il = 14 - decltype(sc)::value;
    const double rsi = shfl_d(myrs, base + il);
    double s0 = 0.0, s1 = 0.0, s2 = 0.0, s3 = 0.0;
    static_for<il + 1, 16>([&](auto tc) {  // xl[t] == 0 for t > jl
      constexpr int t = decltype(tc)::value;
      const double rit = sRb[(base + t) * TLD + base + il];
      if constexpr ((t & 3) == 0) s0 = fma(rit, xl[t], s0);
      else if constexpr ((t & 3) == 1) s1 = fma(rit, xl[t], s1);
      else if constexpr ((t & 3) == 2) s2 = fma(rit, xl[t], s2);
      else s3 = fma(rit, xl[t], s3);
    });
    if (jl > il) xl[il] = -rsi * ((s0 + s1) + (s2 + s3));
  });
  // publish the diagonal blocks: xs[lane * 16 + r] (scratch, for phase B) and the output tiles
  double* xs = ub + 128;        // 32 x 16
  double* ts = ub + 128 + 512;  // 16 x 16
  static_for<0, 16>([&](auto rc_) {
    constexpr int r = decltype(rc_)::value;
    xs[lane * 16 + r] = xl[r];
    sXb[lane * TLD + base + r] = xl[r];
    sXTb[(base + r) * TLD + lane] = xl[r];
  });
  __syncwarp();
  // Phase B: X12 = -X11 R12 X22 (16 x 16 blocks).  Lane (g, jl) owns column jl of the block and rows 8 g .. 8 g + 7.
  {
    double rc[16], tr[8];
    static_for<0, 16>([&](auto tc) { constexpr int t = decltype(tc)::value; rc[t] = sRb[(16 + jl) * TLD + t]; });  // R(t, 16 + jl)
    static_for<0, 8>([&](auto rr) {
      constexpr int r = decltype(rr)::value;
      const int i = 8 * g16 + r;
      double s = 0.0;
      static_for<0, 16>([&](auto tc) {  // X11(i, t) = xs[t * 16 + i], zero for t < i
        constexpr int t = decltype(tc)::value;
        s = fma(xs[t * 16 + i], rc[t], s);
      });
      tr[r] = s;
      ts[jl * 16 + i] = s;  // T(i, jl)
    });
    __syncwarp();
    double xc[16];
    static_for<0, 16>([&](auto tc) { constexpr int t = decltype(tc)::value; xc[t] = xs[(16 + jl) * 16 + t]; });  // X22(t, jl), zero for t > jl
    static_for<0, 8>([&](auto rr) {
      constexpr int r = decltype(rr)::value;
      const int i = 8 * g16 + r;
      double s = 0.0;
      static_for<0, 16>([&](auto tc) {
        constexpr int t = decltype(tc)::value;
        s = fma(ts[t * 16 + i], xc[t], s);
      });
      sXb[(16 + jl) * TLD + i] = -s;
      sXTb[i * TLD + 16 + jl] = -s;
    });
    (void)tr;
  }
  __syncwarp();
  if (dbg2 && lane == 0) dbg2[2] = clock64();
}

// acc(8 x 16 per warp) += A^T B over k in [k0, k0 + 32) for the 32 x 32 output block at (rows ar.., cols bc..) of the tiles
// As ([row][k]) and Bs ([col][k]); warp w owns fragment row (w & 3) and fragment columns 2 (w >> 2) + {0, 1}.
__device__ __forceinline__ void mma32(double (&acc)[2][2], const double* As, int ar, const double* Bs, int bc, int k0) {
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, g = lane >> 2, q = lane & 3;
  const double* ap = As + (ar + (w & 3) * 8 + g) * TLD + k0 + q;
  const double* bp = Bs + (bc + (w >> 2) * 16 + g) * TLD + k0 + q;
#pragma unroll
  for (int k = 0; k < 32; k += 4) {
    const double a = ap[k], b0 = bp[k], b1 = bp[8 * TLD + k];
    dmma884(acc[0][0], acc[0][1], a, b0);
    dmma884(acc[1][0], acc[1][1], a, b1);
  }
}
#define M32_ROW ((w & 3) * 8 + g)
#define M32_COL(j, e) ((w >> 2) * 16 + (j) * 8 + 2 * q + (e))

// sA: the block, element (row, col) at sA[col * TLD + row] (upper part read).  Outputs as full 64 x 64 tiles:
//   sR [col][row] = R,   sX [col][row] = Rinv,   sXT [col][row] = Rinv^T   (zeros in the other triangle)
// sA is destroyed.  All 256 threads must call.
__device__ void leaf64_fast(double* __restrict__ sA, double* __restrict__ sR, double* __restrict__ sX, double* __restrict__ sXT,
                            double* __restrict__ ub, int* info, int pivot_base, long long* dbg2 = nullptr) {
  const int tid = threadIdx.x, lane = tid & 31, w = tid >> 5, g = lane >> 2, q = lane & 3;
  for (int idx = tid; idx < 64 * 64; idx += 256) {
    const int r = idx & 63, cidx = idx >> 6;
    sR[cidx * TLD + r] = 0.0; sX[cidx * TLD + r] = 0.0; sXT[cidx * TLD + r] = 0.0;
  }
  __syncthreads();
  double c[32];
#pragma unroll 1
  for (int half = 0; half < 2; half++) {
    const int o = half * 32;
    if (half == 1) {
      // R12 = X11^T A12  (A operand X11: [row i][k] = X11(k, i) = sX[i * TLD + k];  B operand A12: [col][k] = sA[(32 + col) * TLD + k])
      double acc[2][2] = {{0.0, 0.0}, {0.0, 0.0}};
      mma32(acc, sX, 0, sA, 32, 0);
#pragma unroll
      for (int j = 0; j < 2; j++)
#pragma unroll
        for (int e = 0; e < 2; e++) sR[(32 + M32_COL(j, e)) * TLD + M32_ROW] = acc[j][e];
      __syncthreads();
      // A22 -= R12^T R12
      double acc2[2][2] = {{0.0, 0.0}, {0.0, 0.0}};
      mma32(acc2, sR + 32 * TLD, 0, sR + 32 * TLD, 0, 0);  // both operands: rows = columns 32.. of sR, k = rows 0..31
#pragma unroll
      for (int j = 0; j < 2; j++)
#pragma unroll
        for (int e = 0; e < 2; e++) sA[(32 + M32_COL(j, e)) * TLD + 32 + M32_ROW] -= acc2[j][e];
      __syncthreads();
    }
    if (w == 0) {
#pragma unroll
      for (int i = 0; i < 32; i++) c[i] = sA[(o + lane) * TLD + o + i];
      warp_potrf_trtri_32(c, sR + o * TLD + o, sX + o * TLD + o, sXT + o * TLD + o, ub, lane, info, pivot_base + o,
                          (dbg2 && half == 0) ? dbg2 : nullptr);
      if (dbg2 && half == 0 && lane == 0) dbg2[3] = clock64();
    }
    __syncthreads();
  }
  // X12 = -X11 R12 X22:  T = X11 R12  (A operand [row i][k] = X11(i, k) = sXT[i * TLD + k]; B operand R12: sR[(32 + col) * TLD + k])
  {
    double acc[2][2] = {{0.0, 0.0}, {0.0, 0.0}};
    mma32(acc, sXT, 0, sR, 32, 0);
    __syncthreads();  // everyone is done reading sA's leftovers; reuse sA rows 0..31 as T in [row][32 + k] order
#pragma unroll
    for (int j = 0; j < 2; j++)
#pragma unroll
      for (int e = 0; e < 2; e++) sA[M32_ROW * TLD + 32 + M32_COL(j, e)] = acc[j][e];  // k offset 32 to line up with X22's rows
    __syncthreads();
    double acc2[2][2] = {{0.0, 0.0}, {0.0, 0.0}};
    mma32(acc2, sA, 0, sX, 32, 32);  // A operand T: [row i][k = t]; B operand X22: sX[(32 + col) * TLD + 32 + t]
#pragma unroll
    for (int j = 0; j < 2; j++)
#pragma unroll
      for (int e = 0; e < 2; e++) {
        const double v = -acc2[j][e];
        sX[(32 + M32_COL(j, e)) * TLD + M32_ROW] = v;
        sXT[M32_ROW * TLD + 32 + M32_COL(j, e)] = v;
      }
  }
  __syncthreads();
}

// ---- cluster base case ----------------------------------------------------------------------------------------
// W (nb x nb, upper read, destroyed) -> R, Ri, RiT blocks (full nb x nb blocks written: zeros in the other triangle).
// Per block column jb:   [row panel over the cluster]  barrier  [trailing update over 7 CTAs  ||  the 8th: diagonal tile of
// the next column first, then its leaf (lookahead)]  barrier.
template <int CW>
__global__ void __cluster_dims__(CW, 1, 1) __launch_bounds__(256, 1)
    basecase_kernel(int nb, double* __restrict__ W, long long ldw, double* __restrict__ R, long long ldr, double* __restrict__ Ri,
                    long long ldri, double* __restrict__ RiT, long long ldrit, int* __restrict__ info, long long* __restrict__ dbg,
                    BatchStrides bstr, int pivot_base) {
  {
    const long long b = blockIdx.y;
    W += b * bstr.w; R += b * bstr.r; Ri += b * bstr.ri; RiT += b * bstr.rit; info += b;
  }
  extern __shared__ __align__(16) double sm[];
  double* sA = sm;                     // tile / leaf array a
  double* sB = sm + TILE_DOUBLES;      // tile / leaf array r
  double* sT = sm + 2 * TILE_DOUBLES;  // tile / leaf scratch
  cg::cluster_group cluster = cg::this_cluster();
  const int rank = (int)cluster.block_rank();
  const int T = nb >> 6;
  double acc[4][2][2];
  int dbgi = 0;
#define DBG_STAMP() do { if (dbg && rank == 0 && threadIdx.x == 0) dbg[dbgi++] = clock64(); } while (0)
  DBG_STAMP();

  double* sU = sm + 3 * TILE_DOUBLES;  // fourth tile (fast leaf only)
  auto do_leaf = [&](int jb) {
    const long long o = (long long)jb * 64;
    __syncthreads();  // the caller's global writes (trailing update of this very tile) are complete block-wide
    tile_load(sA, W + o + o * ldw, ldw);
    __syncthreads();
    if (dbg && jb == 0 && threadIdx.x == 0) dbg[20] = clock64();
    leaf64_fast(sA, sB, sT, sU, sm + 4 * TILE_DOUBLES, info, pivot_base + jb * 64, (dbg && jb == 0) ? dbg + 24 : nullptr);
    if (dbg && jb == 0 && threadIdx.x == 0) dbg[21] = clock64();
    tile_store<false>(R + o + o * ldr, ldr, sB);
    tile_store<false>(Ri + o + o * ldri, ldri, sT);
    tile_store<false>(RiT + o + o * ldrit, ldrit, sU);
    __syncthreads();
  };
  // trailing tile (i, j) of step jb: W(i, j) -= R(jb, i)^T R(jb, j)
  auto do_trailing = [&](int jb, int i, int j) {
    const long long o = (long long)jb * 64;
    __syncthreads();
    tile_load(sA, R + o + (long long)i * 64 * ldr, ldr);
    tile_load(sB, R + o + (long long)j * 64 * ldr, ldr);
    __syncthreads();
    acc_zero(acc);
    tile_mma(acc, sA, sB);
    acc_to_smem_colmajor(acc, sT, -1.0);
    __syncthreads();
    tile_store<true>(W + (long long)i * 64 + (long long)j * 64 * ldw, ldw, sT);
  };

  if (rank == 0) do_leaf(0);
  DBG_STAMP();
  __threadfence();
  cluster.sync();
  DBG_STAMP();
  // ---------------- Cholesky: right-looking over 64-wide block columns ----------------
  for (int jb = 0; jb < T; jb++) {
    const long long o = (long long)jb * 64;
    // row panel: R(jb, j) = Rinv_jj^T W(jb, j), j > jb
    int work = 0;
    for (int j = jb + 1; j < T; j++, work++) {
      if (work % CW != rank) continue;
      __syncthreads();
      tile_load(sA, Ri + o + o * ldri, ldri);                         // A[k][i] = Rinv_jj(k, i)
      tile_load(sB, W + o + (long long)j * 64 * ldw, ldw);            // B[k][c] = W(jb rows, j cols)
      __syncthreads();
      acc_zero(acc);
      tile_mma(acc, sA, sB);
      acc_to_smem_colmajor(acc, sT, 1.0);
      __syncthreads();
      tile_store<false>(R + o + (long long)j * 64 * ldr, ldr, sT);
    }
    if (jb == 0) DBG_STAMP();
    __threadfence();
    cluster.sync();
    if (jb == 0) DBG_STAMP();
    if (jb + 1 < T) {
      const int leaf_rank = (jb + 1) % CW;
      if (rank == leaf_rank) {
        do_trailing(jb, jb + 1, jb + 1);   // lookahead: finish the next diagonal block first ...
        __threadfence_block();
        do_leaf(jb + 1);                   // ... and factor it while the other CTAs update the rest
      } else {
        const int slot = rank > leaf_rank ? rank - 1 : rank;
        work = 0;
        for (int j = jb + 1; j < T; j++)
          for (int i = jb + 1; i <= j; i++) {
            if (i == jb + 1 && j == jb + 1) continue;
            if (work++ % (CW - 1) != slot) continue;
            do_trailing(jb, i, j);
          }
      }
    }
    if (jb == 0) DBG_STAMP();
    __threadfence();
    cluster.sync();
    if (jb == 0) DBG_STAMP();
  }
  DBG_STAMP();
  // zero the strictly-lower blocks of R (the leaf wrote the diagonal blocks completely)
  {
    int work = 0;
    for (int j = 0; j < T; j++)
      for (int i = j + 1; i < T; i++, work++) {
        if (work % CW != rank) continue;
        for (int idx = threadIdx.x; idx < 4096; idx += 256)
          R[(long long)i * 64 + (idx & 63) + ((long long)j * 64 + (idx >> 6)) * ldr] = 0.0;
      }
  }
  // ---------------- inverse by recursive doubling over 64-wide blocks ----------------
  //   level bs (1, 2, 4 tiles): for every pair of neighbouring diagonal blocks [o, o+bs) / [o+bs, o+2bs):
  //     phase 1   T(i, j)    =  sum_{k = i}^{o+bs-1} Rinv(i, k) R(k, j)          (stored transposed in the dead W block)
  //     phase 2   Rinv(i, j) = -sum_{k = o+bs}^{j}   T(i, k)    Rinv(k, j)
  //   Depth 18 tile products for T = 8 instead of 35 for the column-by-column order; W is dead after the Cholesky phase.
  for (int bs = 1; bs < T; bs <<= 1) {
    const int span = 2 * bs;
    // phase 1
    int work = 0;
    for (int o = 0; o + bs < T; o += span) {
      const int jend = min(o + span, T);
      for (int j = o + bs; j < jend; j++)
        for (int i = o; i < o + bs; i++, work++) {
          if (work % CW != rank) continue;
          acc_zero(acc);
          for (int k = i; k < o + bs; k++) {
            __syncthreads();
            tile_load(sA, RiT + (long long)k * 64 + (long long)i * 64 * ldrit, ldrit);  // A[row i_][k_] = Rinv(i, k)
            tile_load(sB, R + (long long)k * 64 + (long long)j * 64 * ldr, ldr);
            __syncthreads();
            tile_mma(acc, sA, sB);
          }
          __syncthreads();
          acc_to_smem_rowmajor(acc, sT, 1.0);  // value(i_, t_) at sT[i_ * TLD + t_]
          __syncthreads();
          // T(i, j)^T into the W tile (j, i): W[(j*64 + t_) + (i*64 + i_) * ldw] = T(i, j)(i_, t_)
          tile_store_from_rowmajor(W + (long long)j * 64 + (long long)i * 64 * ldw, ldw, sT);
        }
    }
    __threadfence();
    cluster.sync();
    // phase 2
    work = 0;
    for (int o = 0; o + bs < T; o += span) {
      const int jend = min(o + span, T);
      for (int j = o + bs; j < jend; j++)
        for (int i = o; i < o + bs; i++, work++) {
          if (work % CW != rank) continue;
          acc_zero(acc);
          for (int k = o + bs; k <= j; k++) {
            __syncthreads();
            tile_load(sA, W + (long long)k * 64 + (long long)i * 64 * ldw, ldw);        // A[row i_][t_] = T(i, k)(i_, t_)
            tile_load(sB, Ri + (long long)k * 64 + (long long)j * 64 * ldri, ldri);     // B[t_][c] = Rinv(k, j)
            __syncthreads();
            tile_mma(acc, sA, sB);
          }
          __syncthreads();
          acc_to_smem_colmajor(acc, sA, -1.0);  // value(row, col) at sA[col][row]
          acc_to_smem_rowmajor(acc, sB, -1.0);  // value(row, col) at sB[row][col]
          __syncthreads();
          tile_store<false>(Ri + (long long)i * 64 + (long long)j * 64 * ldri, ldri, sA);
          tile_store_from_rowmajor(RiT + (long long)j * 64 + (long long)i * 64 * ldrit, ldrit, sB);
        }
    }
    __threadfence();
    cluster.sync();
  }
  DBG_STAMP();
}
}  // namespace

namespace {
constexpr int LEAF_SMEM = 3 * LEAF_MAX * LD * (int)sizeof(double);
constexpr int BASECASE_SMEM = (4 * TILE_DOUBLES + 128 + 512 + 256) * (int)sizeof(double);
}  // namespace
// per-device shared-memory opt-in of the kernels (called from capital_create after cudaSetDevice)
capital_status_t leaf_init(capital_ctx* ctx) {
  CAP_CUDA(cudaFuncSetAttribute(leaf_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, LEAF_SMEM));
  CAP_CUDA(cudaFuncSetAttribute(basecase_kernel<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, BASECASE_SMEM));
  CAP_CUDA(cudaFuncSetAttribute(basecase_kernel<4>, cudaFuncAttributeMaxDynamicSharedMemorySize, BASECASE_SMEM));
  CAP_CUDA(cudaFuncSetAttribute(basecase_kernel<8>, cudaFuncAttributeMaxDynamicSharedMemorySize, BASECASE_SMEM));
  return CAPITAL_OK;
}

capital_status_t leaf_cholinv(capital_ctx* ctx, cudaStream_t st, int nb, const double* W, int64_t ldw, double* R, int64_t ldr, double* Ri,
                              int64_t ldri, double* RiT, int64_t ldrit, const LeafBatch* bt, int pivot_base) {
  if (nb <= 0) return CAPITAL_OK;
  if (nb > LEAF_MAX || (bt && (bt->batch < 1 || bt->batch > INT32_MAX))) return CAPITAL_ERR_INVALID;
  constexpr int smem = LEAF_SMEM;
  const int tli = ctx->tl_begin(st, 4, nb);
  leaf_kernel<<<bt ? (unsigned)bt->batch : 1u, 256, smem, st>>>(nb, W, ldw, R, ldr, Ri, ldri, RiT, ldrit, bt ? bt->info : ctx->d_info,
                                                                bt ? bt->s : BatchStrides{}, pivot_base);
  ctx->tl_end(st, tli);
  ctx->counters.kernel_launches++;
  ctx->counters.leaf_launches++;
  CAP_CUDA(cudaGetLastError());
  return CAPITAL_OK;
}

// nb must be a multiple of 64, 128 <= nb <= BASECASE_MAX, and RiT non-null.
capital_status_t basecase_cholinv(capital_ctx* ctx, cudaStream_t st, int nb, double* W, int64_t ldw, double* R, int64_t ldr, double* Ri,
                                  int64_t ldri, double* RiT, int64_t ldrit, const LeafBatch* bt, int pivot_base) {
  if (nb % 64 != 0 || nb < 64 || nb > BASECASE_MAX || RiT == nullptr) return CAPITAL_ERR_INVALID;
  const int cw = bt ? bt->cw : 8;
  if (bt && (bt->batch < 1 || bt->batch > 65535)) return CAPITAL_ERR_INVALID;  // grid y
  auto kernel = cw == 2 ? basecase_kernel<2> : cw == 4 ? basecase_kernel<4> : cw == 8 ? basecase_kernel<8> : nullptr;
  if (!kernel) return CAPITAL_ERR_INVALID;
  constexpr int smem = BASECASE_SMEM;
  long long* dbg = nullptr;
  if (getenv("CAPITAL_BC_DEBUG") && !bt) {
    CAP_TRY(ctx->workspace("bc_dbg", 64 * sizeof(long long), (void**)&dbg));
    CAP_CUDA(cudaMemsetAsync(dbg, 0, 64 * sizeof(long long), st));
  }
  const int tli = ctx->tl_begin(st, 3, nb);
  kernel<<<dim3(cw, bt ? (unsigned)bt->batch : 1u), 256, smem, st>>>(nb, W, ldw, R, ldr, Ri, ldri, RiT, ldrit, bt ? bt->info : ctx->d_info,
                                                                      dbg, bt ? bt->s : BatchStrides{}, pivot_base);
  ctx->tl_end(st, tli);
  if (dbg) {
    long long h[32];
    CAP_CUDA(cudaMemcpyAsync(h, dbg, sizeof(h), cudaMemcpyDeviceToHost, st));
    CAP_CUDA(cudaStreamSynchronize(st));
    fprintf(stderr, "[bc nb=%d] leaf0=%lld bar=%lld panel0=%lld bar=%lld trail0+leaf1=%lld bar=%lld | chol_total=%lld inverse=%lld total=%lld cycles\n", nb,
            h[1] - h[0], h[2] - h[1], h[3] - h[2], h[4] - h[3], h[5] - h[4], h[6] - h[5], h[7] - h[0], h[8] - h[7], h[8] - h[0]);
    fprintf(stderr, "   leaf64: load=%lld total=%lld | warp32: pre=%lld potrf=%lld trtri=%lld store=%lld\n", h[20] - h[0], h[21] - h[20], h[24] - h[20],
            h[25] - h[24], h[26] - h[25], h[27] - h[26]);
  }
  ctx->counters.kernel_launches++;
  ctx->counters.leaf_launches++;
  CAP_CUDA(cudaGetLastError());
  return CAPITAL_OK;
}
