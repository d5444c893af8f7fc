// Triangular apply for cholinv::solve:  C = beta Cin + alpha op(U[r0:r1, c0:c1]) P,  op = N or T, for a panel of at most SOLVE_W
// right-hand sides.  U is an upper-triangular local factor read in place -- packed (column i at i(i+1)/2) or rect (ld) -- and
// entries below its diagonal are never read.  The factor is never unpacked: one pass over the window is the whole HBM traffic.
//
// Shape.  The window is walked in 64 x 64 tiles.  Every tile is 64 column segments of at most 512 contiguous bytes (8-byte loads:
// packed columns start on any 8-byte boundary), staged in shared memory next to the 64-row slice of the panel, so the panel is
// read once per tile and not once per column.  One index of the tile is OWNED by the CTA (op T: a block of 64 columns, whose dot
// products with the panel it computes; op N: a block of 64 rows), the other is the contraction index k, walked tile by tile.
// A triangle makes the owned blocks' k extents very uneven, so the k range of every block is cut into chunks of TA_KC tiles, one
// CTA each, longest blocks first; stage 1 writes one partial per chunk, stage 2 adds the chunks of a block in chunk order and
// applies alpha, beta.  No atomics anywhere: the same inputs give the same bits (the grid solve relies on it).
#include "common.cuh"
#include <algorithm>

namespace {

constexpr int TT = 64;          // tile edge
constexpr int TA_THREADS = 256;
constexpr int TA_KC = 16;       // k tiles (1024 values of k) per chunk
constexpr int TA_PER = TT * TT / TA_THREADS;  // factor elements each thread moves per tile

struct TriDev {
  const double* U;
  int64_t ldu;  // 0: packed
  int64_t r0, r1, c0, c1;
  int nrhs;
  const double* P;
  int64_t pinc, ldp;
  double* part;
  int64_t nob, cmax;
};

// k range of owned block [olo, ohi): op T owns columns, k runs over the rows j <= i of the window; op N owns rows, k over the
// columns i >= j
__host__ __device__ inline void k_range(bool trans, int64_t r0, int64_t r1, int64_t c0, int64_t c1, int64_t olo, int64_t ohi,
                                        int64_t* klo, int64_t* khi) {
  if (trans) { *klo = r0; *khi = r1 < ohi ? r1 : ohi; }
  else { *klo = c0 > olo ? c0 : olo; *khi = c1; }
}
__host__ __device__ inline int64_t n_chunks(int64_t klo, int64_t khi) {
  const int64_t tiles = khi > klo ? (khi - klo + TT - 1) / TT : 0;
  return (tiles + TA_KC - 1) / TA_KC;
}

template <int W, bool TRANS>
__global__ void __launch_bounds__(TA_THREADS, 2) tri_apply_kernel(TriDev a) {
  constexpr int WG = W >= 4 ? 4 : 1;  // w groups (each owns WPT right-hand sides)
  constexpr int KG = 4 / WG;           // k groups (narrow panels split k instead, summed in group order at the end)
  constexpr int WPT = W / WG;
  constexpr int KS = TT / KG;
  constexpr int PP = W == 1 ? 1 : W + 2;  // panel pitch in shared memory (even: 16-byte reads of pairs)
  constexpr int PE = (TT * W + TA_THREADS - 1) / TA_THREADS;
  extern __shared__ double sm[];
  double* Us = sm;                  // [o][k], pitch TT + 1
  double* Ps = sm + TT * (TT + 1);  // [k][w], pitch PP
  const int t = threadIdx.x;
  const int64_t b = TRANS ? a.nob - 1 - (int64_t)blockIdx.y : (int64_t)blockIdx.y;  // longest blocks first
  const int64_t o0 = TRANS ? a.c0 : a.r0, o1 = TRANS ? a.c1 : a.r1;
  const int64_t olo = o0 + b * TT, ohi = o1 < olo + TT ? o1 : olo + TT;
  int64_t klo, khi;
  k_range(TRANS, a.r0, a.r1, a.c0, a.c1, olo, ohi, &klo, &khi);
  const int64_t ktiles = khi > klo ? (khi - klo + TT - 1) / TT : 0;
  const int64_t t0 = (int64_t)blockIdx.x * TA_KC, t1 = ktiles < t0 + TA_KC ? ktiles : t0 + TA_KC;
  if (t0 >= t1) return;
  const bool packed = a.ldu == 0;
  const int oo = t & (TT - 1), g = t >> 6, wg = g % WG, kg = g / WG;

  double ur[TA_PER], pr[PE];
  auto load = [&](int64_t tt) {
    const int64_t kb = klo + tt * TT;
    // element it of this thread: column i = ib + 4 it, row j (the contiguous index of a column segment runs over the lanes: the
    // row, which is k for op T and o for op N)
    const int64_t j = (TRANS ? kb : olo) + oo;
    const int64_t iend = TRANS ? ohi : khi;
    const bool row_ok = j < (TRANS ? khi : ohi);
    int64_t i = (TRANS ? olo : kb) + g;
    const double* col = a.U + (packed ? i * (i + 1) / 2 : i * a.ldu);
#pragma unroll
    for (int it = 0; it < TA_PER; it++) {
      double v = 0.0;
      if (row_ok && i < iend && j <= i) v = col[j];
      ur[it] = v;
      col += packed ? 4 * i + 10 : 4 * a.ldu;  // start of column i + 4
      i += 4;
    }
#pragma unroll
    for (int p = 0; p < PE; p++) {
      const int e = p * TA_THREADS + t;
      const int kk = e & (TT - 1), w = e >> 6;
      const int64_t k = kb + kk;
      double v = 0.0;
      if (e < TT * W && k < khi && w < a.nrhs) v = a.P[k * a.pinc + w * a.ldp];
      pr[p] = v;
    }
  };

  double acc[WPT];
#pragma unroll
  for (int q = 0; q < WPT; q++) acc[q] = 0.0;
  load(t0);
  for (int64_t tt = t0; tt < t1; tt++) {
    __syncthreads();  // the previous tile has been consumed
#pragma unroll
    for (int it = 0; it < TA_PER; it++) {
      const int ci = 4 * it + g;  // column of the element inside the tile; its row is oo
      Us[TRANS ? ci * (TT + 1) + oo : oo * (TT + 1) + ci] = ur[it];
    }
#pragma unroll
    for (int p = 0; p < PE; p++) {
      const int e = p * TA_THREADS + t;
      if (e < TT * W) Ps[(e & (TT - 1)) * PP + (e >> 6)] = pr[p];
    }
    __syncthreads();
    if (tt + 1 < t1) load(tt + 1);  // the next tile is in flight while this one is multiplied
    const double* u = Us + oo * (TT + 1) + kg * KS;
    const double* pp = Ps + kg * KS * PP + wg * WPT;
#pragma unroll 8
    for (int kk = 0; kk < KS; kk++) {
      const double uv = u[kk];
      if constexpr (WPT % 2 == 0) {
#pragma unroll
        for (int q = 0; q < WPT; q += 2) {
          const double2 pv = *reinterpret_cast<const double2*>(pp + kk * PP + q);
          acc[q] = fma(uv, pv.x, acc[q]);
          acc[q + 1] = fma(uv, pv.y, acc[q + 1]);
        }
      } else {
#pragma unroll
        for (int q = 0; q < WPT; q++) acc[q] = fma(uv, pp[kk * PP + q], acc[q]);
      }
    }
  }
  if constexpr (KG > 1) {  // k groups: summed in group order
    __syncthreads();
    double* red = sm;
#pragma unroll
    for (int q = 0; q < WPT; q++) red[(kg * TT + oo) * W + q] = acc[q];
    __syncthreads();
    if (kg == 0) {
#pragma unroll
      for (int q = 0; q < WPT; q++) {
        double s = red[oo * W + q];
        for (int g2 = 1; g2 < KG; g2++) s += red[(g2 * TT + oo) * W + q];
        acc[q] = s;
      }
    }
  }
  if (kg == 0 && olo + oo < ohi) {
    double* dst = a.part + ((b * a.cmax + blockIdx.x) * TT + oo) * W + wg * WPT;
#pragma unroll
    for (int q = 0; q < WPT; q++) dst[q] = acc[q];
  }
}

struct TriFin {
  bool trans;
  int64_t r0, r1, c0, c1, o0, olen;
  int nrhs, w;
  const double* part;
  int64_t cmax;
  double alpha, beta;
  const double* Cin;
  int64_t ldcin;
  double* C;
  int64_t cinc, ldc;
};

// C(o, w) = alpha * (sum of the block's chunk partials, in chunk order) + beta * Cin(o, w)
__global__ void tri_finish_kernel(TriFin f) {
  const int64_t total = f.olen * f.nrhs;
  for (int64_t idx = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
    const int64_t orel = idx % f.olen, w = idx / f.olen;
    const int64_t b = orel / TT, oo = orel % TT;
    const int64_t olo = f.o0 + b * TT, ohi = (f.o0 + f.olen) < olo + TT ? f.o0 + f.olen : olo + TT;
    int64_t klo, khi;
    k_range(f.trans, f.r0, f.r1, f.c0, f.c1, olo, ohi, &klo, &khi);
    const int64_t nch = n_chunks(klo, khi);
    double s = 0.0;
    for (int64_t c = 0; c < nch; c++) s += f.part[((b * f.cmax + c) * TT + oo) * f.w + w];
    const int64_t o = f.o0 + orel;
    double v = f.alpha * s;
    if (f.Cin) v += f.beta * f.Cin[o * f.cinc + w * f.ldcin];
    f.C[o * f.cinc + w * f.ldc] = v;
  }
}

template <int W, bool TRANS>
capital_status_t launch_w(capital_ctx* ctx, cudaStream_t st, const TriDev& a, dim3 grid) {
  constexpr int PP = W == 1 ? 1 : W + 2;
  const size_t smem = (size_t)(TT * (TT + 1) + TT * PP) * 8;
  CAP_CUDA(cudaFuncSetAttribute(tri_apply_kernel<W, TRANS>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  tri_apply_kernel<W, TRANS><<<grid, TA_THREADS, smem, st>>>(a);
  CAP_CUDA(cudaGetLastError());
  return CAPITAL_OK;
}

template <bool TRANS>
capital_status_t launch_op(capital_ctx* ctx, cudaStream_t st, int w, const TriDev& a, dim3 grid) {
  switch (w) {
    case 1: return launch_w<1, TRANS>(ctx, st, a, grid);
    case 2: return launch_w<2, TRANS>(ctx, st, a, grid);
    case 4: return launch_w<4, TRANS>(ctx, st, a, grid);
    case 8: return launch_w<8, TRANS>(ctx, st, a, grid);
    case 16: return launch_w<16, TRANS>(ctx, st, a, grid);
    default: return launch_w<32, TRANS>(ctx, st, a, grid);
  }
}

}  // namespace

capital_status_t tri_apply(capital_ctx* ctx, cudaStream_t st, const TriApply& x) {
  if (x.nrhs < 1 || x.nrhs > SOLVE_W) { ctx->set_error("tri_apply: 1 <= nrhs <= SOLVE_W"); return CAPITAL_ERR_INVALID; }
  const int64_t o0 = x.trans ? x.c0 : x.r0, o1 = x.trans ? x.c1 : x.r1;
  if (o1 <= o0) return CAPITAL_OK;
  int w = 1;
  while (w < x.nrhs) w *= 2;  // smallest instantiated panel width that holds the panel
  const int64_t nob = ceil_div(o1 - o0, TT);
  // the k extent grows (op T) or shrinks (op N) monotonically with the block: the longest is at one end
  int64_t cmax = 0;
  for (int64_t b : {(int64_t)0, nob - 1}) {
    const int64_t olo = o0 + b * TT, ohi = std::min(o1, olo + TT);
    int64_t klo, khi;
    k_range(x.trans, x.r0, x.r1, x.c0, x.c1, olo, ohi, &klo, &khi);
    cmax = std::max(cmax, n_chunks(klo, khi));
  }
  double* part = nullptr;
  if (cmax > 0) {
    CAP_TRY(ctx->workspace("solve_part", (size_t)nob * cmax * TT * w * 8, (void**)&part));
    TriDev a{x.U, x.ldu, x.r0, x.r1, x.c0, x.c1, (int)x.nrhs, x.P, x.pinc, x.ldp, part, nob, cmax};
    const dim3 grid((unsigned)cmax, (unsigned)nob);
    if (x.trans) CAP_TRY(launch_op<true>(ctx, st, w, a, grid));
    else CAP_TRY(launch_op<false>(ctx, st, w, a, grid));
    ctx->counters.kernel_launches++;
  }
  TriFin f{x.trans, x.r0, x.r1, x.c0, x.c1, o0, o1 - o0, (int)x.nrhs, w, part, cmax, x.alpha, x.beta, x.Cin, x.ldcin, x.C, x.cinc, x.ldc};
  const int64_t total = (o1 - o0) * x.nrhs;
  const int blocks = (int)std::min<int64_t>(ceil_div(total, 256), 4 * (int64_t)ctx->num_sms);
  tri_finish_kernel<<<blocks, 256, 0, st>>>(f);
  CAP_CUDA(cudaGetLastError());
  ctx->counters.kernel_launches++;
  return CAPITAL_OK;
}

namespace {
__global__ void panel_add_kernel(int64_t rows, int64_t w, const double* S, int64_t lds, const double* Cin, int64_t ldcin, double* Out,
                                 int64_t ldo) {
  const int64_t total = rows * w;
  for (int64_t idx = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = idx % rows, c = idx / rows;
    double v = S[r + c * lds];
    if (Cin) v += Cin[r + c * ldcin];
    Out[r + c * ldo] = v;
  }
}
}  // namespace

capital_status_t panel_add(capital_ctx* ctx, cudaStream_t st, int64_t rows, int64_t w, const double* S, int64_t lds, const double* Cin,
                           int64_t ldcin, double* Out, int64_t ldo) {
  if (rows <= 0 || w <= 0) return CAPITAL_OK;
  const int blocks = (int)std::min<int64_t>(ceil_div(rows * w, 256), 4 * (int64_t)ctx->num_sms);
  panel_add_kernel<<<blocks, 256, 0, st>>>(rows, w, S, lds, Cin, ldcin, Out, ldo);
  CAP_CUDA(cudaGetLastError());
  ctx->counters.kernel_launches++;
  return CAPITAL_OK;
}
