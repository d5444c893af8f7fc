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
//
// Batches (cholinv::solve_batched, and with FULL windows cacqr::lstsq_batched): blockIdx.z of stage 1 and the flat output index of
// stage 2 pick the matrix; U, P, the partials, Cin and C advance by per-matrix strides.  Batch 1 is the single-matrix call, with the
// same arithmetic.
//
// FULL windows (cacqr::apply_QT / apply_Q / lstsq): the same kernel without the j <= i mask and with k over the whole other extent, so
// a tall rect Q is read once for Q^T P (op T) or Q P (op N).  The substitution Y <- R^-1 Y of lstsq is tri_solve, at the end.
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
  int64_t su, sp, spart;  // per-matrix strides (blockIdx.z)
};

// k range of owned block [olo, ohi): op T owns columns, k runs over the rows j <= i of the window; op N owns rows, k over the
// columns i >= j.  FULL (a rect, non-triangular window): k runs over the whole other extent
template <bool FULL = false>
__host__ __device__ inline void k_range(bool trans, int64_t r0, int64_t r1, int64_t c0, int64_t c1, int64_t olo, int64_t ohi,
                                        int64_t* klo, int64_t* khi) {
  if (FULL) { *klo = trans ? r0 : c0; *khi = trans ? r1 : c1; }
  else if (trans) { *klo = r0; *khi = r1 < ohi ? r1 : ohi; }
  else { *klo = c0 > olo ? c0 : olo; *khi = c1; }
}
__host__ __device__ inline int64_t n_chunks(int64_t klo, int64_t khi) {
  const int64_t tiles = khi > klo ? (khi - klo + TT - 1) / TT : 0;
  return (tiles + TA_KC - 1) / TA_KC;
}

// BATCH: blockIdx.z is the matrix (a separate instantiation, so that the single-matrix kernels keep their code and registers)
template <int W, bool TRANS, bool FULL = false, bool BATCH = false>
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
  k_range<FULL>(TRANS, a.r0, a.r1, a.c0, a.c1, olo, ohi, &klo, &khi);
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
    const double* col = a.U + (BATCH ? blockIdx.z * a.su : 0) + (packed ? i * (i + 1) / 2 : i * a.ldu);
#pragma unroll
    for (int it = 0; it < TA_PER; it++) {
      double v = 0.0;
      if (row_ok && i < iend && (FULL || j <= i)) v = col[j];
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
      if (e < TT * W && k < khi && w < a.nrhs) v = a.P[(BATCH ? blockIdx.z * a.sp : 0) + k * a.pinc + w * a.ldp];
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
    double* dst = a.part + (BATCH ? blockIdx.z * a.spart : 0) + ((b * a.cmax + blockIdx.x) * TT + oo) * W + wg * WPT;
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
  int64_t batch, spart, scin, sc;  // matrices, per-matrix strides of part, Cin, C
};

// C(o, w) = alpha * (sum of the block's chunk partials, in chunk order) + beta * Cin(o, w)
template <bool FULL = false>
__global__ void tri_finish_kernel(TriFin f) {
  const int64_t per = f.olen * f.nrhs, total = per * f.batch;
  for (int64_t gidx = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; gidx < total; gidx += (int64_t)gridDim.x * blockDim.x) {
    const int64_t mb = gidx / per, idx = gidx - mb * per;
    const double* part = f.part + mb * f.spart;
    const double* Cin = f.Cin ? f.Cin + mb * f.scin : nullptr;
    double* C = f.C + mb * f.sc;
    const int64_t orel = idx % f.olen, w = idx / f.olen;
    const int64_t b = orel / TT, oo = orel % TT;
    const int64_t olo = f.o0 + b * TT, ohi = (f.o0 + f.olen) < olo + TT ? f.o0 + f.olen : olo + TT;
    int64_t klo, khi;
    k_range<FULL>(f.trans, f.r0, f.r1, f.c0, f.c1, olo, ohi, &klo, &khi);
    const int64_t nch = n_chunks(klo, khi);
    double s = 0.0;
    for (int64_t c = 0; c < nch; c++) s += part[((b * f.cmax + c) * TT + oo) * f.w + w];
    const int64_t o = f.o0 + orel;
    double v = f.alpha * s;
    if (Cin) v += f.beta * Cin[o * f.cinc + w * f.ldcin];
    C[o * f.cinc + w * f.ldc] = v;
  }
}

// Stage 2 for a full window whose k range is long (Q^T B: the k index runs over the rows of a tall Q, about a thousand chunks at
// 2^20 rows): one warp per output, lane l adds chunks l, l + 32, ... in order, then a fixed butterfly adds the lanes -- still the
// same bits for the same inputs
__global__ void full_finish_kernel(TriFin f) {
  const int lane = threadIdx.x & 31;
  const int64_t per = f.olen * f.nrhs, total = per * f.batch;
  int64_t klo, khi;
  k_range<true>(f.trans, f.r0, f.r1, f.c0, f.c1, 0, 0, &klo, &khi);
  const int64_t nch = n_chunks(klo, khi);
  const int64_t warps = (int64_t)gridDim.x * blockDim.x / 32;
  for (int64_t gidx = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) / 32; gidx < total; gidx += warps) {
    const int64_t mb = gidx / per, idx = gidx - mb * per;
    const double* part = f.part + mb * f.spart;
    const int64_t orel = idx % f.olen, w = idx / f.olen;
    const int64_t b = orel / TT, oo = orel % TT;
    double s = 0.0;
    for (int64_t c = lane; c < nch; c += 32) s += part[((b * f.cmax + c) * TT + oo) * f.w + w];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (lane == 0) {
      const int64_t o = f.o0 + orel;
      double v = f.alpha * s;
      if (f.Cin) v += f.beta * f.Cin[mb * f.scin + o * f.cinc + w * f.ldcin];
      f.C[mb * f.sc + o * f.cinc + w * f.ldc] = v;
    }
  }
}

template <int W, bool TRANS, bool FULL, bool BATCH>
capital_status_t launch_w(capital_ctx* ctx, cudaStream_t st, const TriDev& a, dim3 grid) {
  constexpr int PP = W == 1 ? 1 : W + 2;
  const size_t smem = (size_t)(TT * (TT + 1) + TT * PP) * 8;
  CAP_CUDA(cudaFuncSetAttribute(tri_apply_kernel<W, TRANS, FULL, BATCH>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  tri_apply_kernel<W, TRANS, FULL, BATCH><<<grid, TA_THREADS, smem, st>>>(a);
  CAP_CUDA(cudaGetLastError());
  return CAPITAL_OK;
}

template <bool TRANS, bool FULL, bool BATCH = false>
capital_status_t launch_op(capital_ctx* ctx, cudaStream_t st, int w, const TriDev& a, dim3 grid) {
  switch (w) {
    case 1: return launch_w<1, TRANS, FULL, BATCH>(ctx, st, a, grid);
    case 2: return launch_w<2, TRANS, FULL, BATCH>(ctx, st, a, grid);
    case 4: return launch_w<4, TRANS, FULL, BATCH>(ctx, st, a, grid);
    case 8: return launch_w<8, TRANS, FULL, BATCH>(ctx, st, a, grid);
    case 16: return launch_w<16, TRANS, FULL, BATCH>(ctx, st, a, grid);
    default: return launch_w<32, TRANS, FULL, BATCH>(ctx, st, a, grid);
  }
}

constexpr int64_t TA_MAX_BLOCKS = 65535;  // owned blocks per launch (grid.y)

}  // namespace

capital_status_t tri_apply(capital_ctx* ctx, cudaStream_t st, const TriApply& x) {
  if (x.nrhs < 1 || x.nrhs > SOLVE_W) { ctx->set_error("tri_apply: 1 <= nrhs <= SOLVE_W"); return CAPITAL_ERR_INVALID; }
  if (x.full && x.ldu == 0) { ctx->set_error("tri_apply: a full window needs rect storage"); return CAPITAL_ERR_INVALID; }
  if (x.batch < 1 || x.batch > TA_MAX_BLOCKS) {
    ctx->set_error("tri_apply: 1 <= batch <= 65535");
    return CAPITAL_ERR_INVALID;
  }
  const int64_t o0 = x.trans ? x.c0 : x.r0, o1 = x.trans ? x.c1 : x.r1;
  if (o1 <= o0) return CAPITAL_OK;
  if (ceil_div(o1 - o0, TT) > TA_MAX_BLOCKS) {  // owned rows (columns) are independent: one launch per slab of them
    for (int64_t s0 = o0; s0 < o1; s0 += TA_MAX_BLOCKS * TT) {
      TriApply y = x;
      (x.trans ? y.c0 : y.r0) = s0;
      (x.trans ? y.c1 : y.r1) = std::min(o1, s0 + TA_MAX_BLOCKS * TT);
      CAP_TRY(tri_apply(ctx, st, y));
    }
    return CAPITAL_OK;
  }
  int w = 1;
  while (w < x.nrhs) w *= 2;  // smallest instantiated panel width that holds the panel
  const int64_t nob = ceil_div(o1 - o0, TT);
  // the k extent grows (op T) or shrinks (op N) monotonically with the block: the longest is at one end
  int64_t cmax = 0;
  for (int64_t b : {(int64_t)0, nob - 1}) {
    const int64_t olo = o0 + b * TT, ohi = std::min(o1, olo + TT);
    int64_t klo, khi;
    if (x.full) k_range<true>(x.trans, x.r0, x.r1, x.c0, x.c1, olo, ohi, &klo, &khi);
    else k_range(x.trans, x.r0, x.r1, x.c0, x.c1, olo, ohi, &klo, &khi);
    cmax = std::max(cmax, n_chunks(klo, khi));
  }
  double* part = nullptr;
  if (cmax > 0) {
    CAP_TRY(ctx->workspace("solve_part", (size_t)(nob * cmax * TT * w * x.batch) * 8, (void**)&part));
    TriDev a{x.U, x.ldu, x.r0, x.r1, x.c0, x.c1, (int)x.nrhs, x.P, x.pinc, x.ldp, part, nob, cmax, x.su, x.sp, nob * cmax * TT * w};
    const dim3 grid((unsigned)cmax, (unsigned)nob, (unsigned)x.batch);
    auto launch = x.batch > 1 ? (x.full ? (x.trans ? launch_op<true, true, true> : launch_op<false, true, true>)
                                        : (x.trans ? launch_op<true, false, true> : launch_op<false, false, true>))
                  : x.full    ? (x.trans ? launch_op<true, true> : launch_op<false, true>)
                              : (x.trans ? launch_op<true, false> : launch_op<false, false>);
    CAP_TRY(launch(ctx, st, w, a, grid));
    ctx->counters.kernel_launches++;
  }
  TriFin f{x.trans, x.r0, x.r1, x.c0, x.c1, o0, o1 - o0, (int)x.nrhs, w, part, cmax, x.alpha, x.beta, x.Cin, x.ldcin, x.C, x.cinc, x.ldc,
           x.batch, nob * cmax * TT * w, x.scin, x.sc};
  const int64_t total = (o1 - o0) * x.nrhs * x.batch;
  if (x.full && cmax > 32) {
    const int blocks = (int)std::min<int64_t>(ceil_div(total * 32, 256), 16 * (int64_t)ctx->num_sms);
    full_finish_kernel<<<blocks, 256, 0, st>>>(f);
  } else {
    const int blocks = (int)std::min<int64_t>(ceil_div(total, 256), 4 * (int64_t)ctx->num_sms);
    if (x.full) tri_finish_kernel<true><<<blocks, 256, 0, st>>>(f);
    else tri_finish_kernel<<<blocks, 256, 0, st>>>(f);
  }
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

// ---- triangular substitution: Y <- U^-1 Y ------------------------------------------------------------------------------------
// Blocked from the bottom right in diagonal blocks of TS columns.  Each diagonal block is solved by one CTA: the block's triangle is
// staged in shared memory (packed, column c at c(c+1)/2, with the reciprocals of its diagonal), one warp per right-hand side holds
// the block's rows of its column in registers (row 32 s + lane in slot s), and back substitution runs warp-synchronously -- the
// solved value is broadcast by shuffle, and no block barrier sits in the chain.  The rows above the block are then updated by tri_apply (op N, alpha = -1): that window
// lies wholly above the diagonal, and the panel rows it reads are not the rows it writes.
namespace {
constexpr int TS = 128;
constexpr int TS_SLOTS = TS / 32;
constexpr int TS_THREADS = 1024;  // 32 warps: up to SOLVE_W right-hand sides, and all of them stage the triangle

struct SolveDev {
  const double* U;
  int64_t ldu;  // 0: packed
  int64_t b0, b1;
  int nrhs;
  double* Y;
  int64_t ldy;
  int64_t su, sy;  // per-problem strides (batched kernel)
};

// BATCH: blockIdx.x is the problem, at strides su (U) and sy (Y) -- a separate instantiation, so the single solve keeps its code
template <bool BATCH = false>
__global__ void __launch_bounds__(TS_THREADS) tri_block_solve_kernel(SolveDev a) {
  extern __shared__ double Ts[];       // the triangle, packed
  __shared__ double dinv[TS];          // reciprocals of its diagonal: the chain multiplies
  if constexpr (BATCH) {
    a.U += (int64_t)blockIdx.x * a.su;
    a.Y += (int64_t)blockIdx.x * a.sy;
  }
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int nb = (int)(a.b1 - a.b0);
  const bool packed = a.ldu == 0;
  // staging: every thread walks the nb x nb square with many independent loads in flight, rows of a column on consecutive threads
#pragma unroll 8
  for (int e = threadIdx.x; e < nb * nb; e += TS_THREADS) {
    const int c = e / nb, r = e - c * nb;
    if (r <= c) {
      const int64_t i = a.b0 + c;
      const double v = a.U[(packed ? i * (i + 1) / 2 : i * a.ldu) + a.b0 + r];
      Ts[c * (c + 1) / 2 + r] = v;
      if (r == c) dinv[c] = 1.0 / v;
    }
  }
  const bool active = warp < a.nrhs;
  double* yc = a.Y + (int64_t)warp * a.ldy + a.b0;
  double y[TS_SLOTS];
#pragma unroll
  for (int s = 0; s < TS_SLOTS; s++) {
    const int r = 32 * s + lane;
    y[s] = active && r < nb ? yc[r] : 0.0;
  }
  __syncthreads();
  if (!active) return;
#pragma unroll
  for (int s = TS_SLOTS - 1; s >= 0; s--) {
    if (32 * s >= nb) continue;
    for (int q = 31; q >= 0; q--) {
      const int i = 32 * s + q;
      if (i >= nb) continue;
      const double* ci = Ts + i * (i + 1) / 2;
      const double x = __shfl_sync(0xffffffffu, y[s], q) * dinv[i];
      if (lane == q) y[s] = x;
#pragma unroll
      for (int s2 = 0; s2 <= s; s2++)
        if (s2 < s || lane < q) y[s2] = fma(-ci[32 * s2 + lane], x, y[s2]);
    }
  }
#pragma unroll
  for (int s = 0; s < TS_SLOTS; s++) {
    const int r = 32 * s + lane;
    if (r < nb) yc[r] = y[s];
  }
}
}  // namespace

capital_status_t tri_solve(capital_ctx* ctx, cudaStream_t st, const double* U, int64_t ldu, int64_t n, int64_t nrhs, double* Y,
                           int64_t ldy) {
  if (nrhs < 1 || nrhs > SOLVE_W) { ctx->set_error("tri_solve: 1 <= nrhs <= SOLVE_W"); return CAPITAL_ERR_INVALID; }
  if (n <= 0) return CAPITAL_OK;
  CAP_CUDA(cudaFuncSetAttribute(tri_block_solve_kernel<>, cudaFuncAttributeMaxDynamicSharedMemorySize, TS * (TS + 1) / 2 * 8));
  for (int64_t b0 = (n - 1) / TS * TS; b0 >= 0; b0 -= TS) {
    const int64_t b1 = std::min(n, b0 + TS), nb = b1 - b0;
    tri_block_solve_kernel<<<1, TS_THREADS, (size_t)nb * (nb + 1) / 2 * 8, st>>>(SolveDev{U, ldu, b0, b1, (int)nrhs, Y, ldy, 0, 0});
    CAP_CUDA(cudaGetLastError());
    ctx->counters.kernel_launches++;
    //                           U  ldu  trans r0  r1  c0  c1  nrhs  alpha P  pinc ldp  beta Cin ldcin C  cinc ldc
    if (b0 > 0) CAP_TRY(tri_apply(ctx, st, {U, ldu, false, 0, b0, b0, b1, nrhs, -1.0, Y, 1, ldy, 1.0, Y, ldy, Y, 1, ldy}));
  }
  return CAPITAL_OK;
}

// The same blocks and updates as tri_solve, one problem per CTA of the block solve and per grid z of the (batched) update
capital_status_t tri_solve_batched(capital_ctx* ctx, cudaStream_t st, const double* U, int64_t ldu, int64_t su, int64_t n, int64_t nrhs,
                                   double* Y, int64_t ldy, int64_t sy, int64_t batch) {
  if (nrhs < 1 || nrhs > SOLVE_W || ldu < n || batch > 65535) {
    ctx->set_error("tri_solve_batched: 1 <= nrhs <= SOLVE_W, rect U, batch <= 65535");
    return CAPITAL_ERR_INVALID;
  }
  if (n <= 0 || batch <= 0) return CAPITAL_OK;
  CAP_CUDA(cudaFuncSetAttribute(tri_block_solve_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, TS * (TS + 1) / 2 * 8));
  for (int64_t b0 = (n - 1) / TS * TS; b0 >= 0; b0 -= TS) {
    const int64_t b1 = std::min(n, b0 + TS), nb = b1 - b0;
    tri_block_solve_kernel<true><<<(unsigned)batch, TS_THREADS, (size_t)nb * (nb + 1) / 2 * 8, st>>>(
        SolveDev{U, ldu, b0, b1, (int)nrhs, Y, ldy, su, sy});
    CAP_CUDA(cudaGetLastError());
    ctx->counters.kernel_launches++;
    //                           U  ldu  trans r0  r1  c0  c1  nrhs  alpha P  pinc ldp  beta Cin ldcin C  cinc ldc  full   batch  su  sp  scin sc
    if (b0 > 0) CAP_TRY(tri_apply(ctx, st, {U, ldu, false, 0, b0, b0, b1, nrhs, -1.0, Y, 1, ldy, 1.0, Y, ldy, Y, 1, ldy, false, batch, su, sy, sy, sy}));
  }
  return CAPITAL_OK;
}
