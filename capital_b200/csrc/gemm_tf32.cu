// TF32 tensor-core (wgmma) product for the MIXED-PRECISION trailing update of BASELINE config 5:
//     C[m x n] (FP64) = beta * C + alpha * sum_p A_p^T B_p        A_p: k x m, B_p: k x n  (FP32 copies of FP64 operands, col-major)
//
// EXPERIMENTAL -- OFF BY DEFAULT (capital_set_trailing_precision).  The default FP64 path never touches this file's kernels.
//
// Why it exists: the reference has no float BLAS path (src/blas/interface.hpp:43-97 is double only); the FP64 trailing update
// (summa::syrk, summa.hpp:143-145) is the one place of the hot path whose arithmetic a user may trade for speed: Hopper's FP64
// tensor rate is a fraction of its TF32 rate.  The panel / base case, R12 and the inverse stay FP64.
//
// H100 design.  Both operands are K-contiguous ("K-major" for wgmma, the only major-ness wgmma accepts for TF32), so a
// (128 rows x 32 k) FP32 tile is 128 rows of 128 bytes: one TMA box per operand per stage (SWIZZLE_128B), consumed in place by
// wgmma.mma_async.m64n128k8.f32.tf32.tf32 through shared-memory matrix descriptors (four per stage, K = 8 each).  Two consumer
// warpgroups each own 64 rows of the 128 x 128 tile; a third warpgroup, of which one lane drives TMA, hands its registers to them
// (setmaxnreg).  A consumer warpgroup releases a stage once its wgmma group has retired (wgmma.wait_group 0).
// The tensor cores' FP32 accumulation truncates, so its error grows with the length of the contraction (measured on H100: a 3-pass
// product at k = 8192 was off by 7e-6 of max |A|^T |B|, no better than the operand rounding it is meant to remove).  Each stage
// therefore starts a fresh FP32 partial (scale-d = 0) that is added into FP64 register accumulators once the stage has retired:
// only 32 products are ever summed in FP32.  The epilogue stores the FP64 accumulators (beta * C added) straight from registers.
// passes = 3: every operand is split as x = hi + lo (both TF32-representable) and the product accumulates hi*hi + hi*lo + lo*hi in
// the same accumulators: FP32-class accuracy at three times the tensor work.
// Every mbarrier wait is bounded (2 s of %globaltimer): a protocol error ends the kernel with info = -3 instead of hanging the GPU.
#include "common.cuh"
#include <algorithm>

namespace {

constexpr int TBM = 128, TBN = 128, TBK = 32;  // tile; TBK floats = one 128-byte swizzle row
constexpr int TSTAGES = 6;
constexpr int T_CWG = TBM / 64;                  // consumer warpgroups, 64 rows each
constexpr int T_THREADS = (T_CWG + 1) * 128;     // + one producer warpgroup
constexpr int T_REG_CONSUMER = 232, T_REG_PRODUCER = 40;  // 2 x 128 x 232 + 128 x 40 <= 64 K registers
constexpr int T_A_BYTES = TBM * 128, T_B_BYTES = TBN * 128, T_STAGE_BYTES = T_A_BYTES + T_B_BYTES;
constexpr int T_SMEM = TSTAGES * T_STAGE_BYTES + 2 * TSTAGES * 8 + 1024;
static_assert(T_SMEM <= 227 * 1024, "shared memory of one H100 block");
constexpr int T_PAIRS_MAX = 6;  // operand classes (<= 2) x passes (<= 3)

struct Tf32Maps {
  CUtensorMap a[T_PAIRS_MAX];
  CUtensorMap b[T_PAIRS_MAX];
};
struct Tf32Params {
  int M, N, K;
  int npair;
  int flags, noff;
  int gm, gn;
  double alpha, beta;
  double* C;
  long long ldc;
  int* err;
};

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
// false = gave up (2 s): the caller leaves its loop, the kernel ends, the host sees info = -3
__device__ __forceinline__ bool mbar_wait_bounded(uint32_t bar, uint32_t parity, int* err) {
  unsigned long long t0 = 0;
  for (unsigned spin = 0;; spin++) {
    uint32_t ok;
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(ok)
        : "r"(bar), "r"(parity)
        : "memory");
    if (ok) return true;
    if ((spin & 1023u) == 1023u) {
      unsigned long long t;
      asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
      if (t0 == 0) t0 = t;
      else if (t - t0 > 2000000000ull || *(volatile int*)err == -3) { atomicExch(err, -3); return false; }
    }
  }
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void tma_load_2d(uint32_t dst, const CUtensorMap* map, uint32_t bar, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];" ::"r"(dst),
      "l"(map), "r"(bar), "r"(c0), "r"(c1)
      : "memory");
}
// AND of `ok` over the 128 threads of a warpgroup (named barrier 1 + wg): every lane takes the same branch around the
// .sync.aligned wgmma instructions even when the watchdog fires in some threads only
__device__ __forceinline__ bool wg_all(bool ok, int wg) {
  uint32_t r;
  asm volatile(
      "{\n\t.reg .pred p, q;\n\t"
      "setp.ne.u32 p, %1, 0;\n\t"
      "barrier.red.and.pred q, %2, 128, p;\n\t"
      "selp.u32 %0, 1, 0, q;\n\t}"
      : "=r"(r)
      : "r"((uint32_t)ok), "r"(1 + wg)
      : "memory");
  return r != 0;
}
// wgmma shared-memory matrix descriptor, K-major operand, 128-byte swizzle: start address >> 4 @ [0,14), leading byte offset @
// [16,30) (unused for a swizzled K-major operand with one atom along K; 1 by convention), stride byte offset = 8 rows x 128 B =
// 1024 (>> 4) @ [32,46), base offset 0 @ [49,52) (tiles are 1024-byte aligned), layout SWIZZLE_128B = 1 @ [62,64).
__device__ __forceinline__ uint64_t wgmma_desc_k_sw128(uint32_t smem_addr) {
  return (uint64_t)((smem_addr >> 4) & 0x3FFFu) | (1ull << 16) | ((uint64_t)(1024u >> 4) << 32) | (1ull << 62);
}
// d[64] = A (64 x 8, K-major in shared memory) * B (8 x 128, K-major in shared memory) [+ d when ACC], warpgroup-wide, asynchronous
template <int ACC>
__device__ __forceinline__ void wgmma_m64n128k8_tf32(float (&d)[64], uint64_t desc_a, uint64_t desc_b) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
      "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
      "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
      "%64, %65, p, 1, 1;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
        "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
        "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
        "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
        "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(desc_a), "l"(desc_b), "n"(ACC)
      : "memory");
}

__global__ void __launch_bounds__(T_THREADS, 1) gemm_tn_tf32_kernel(const __grid_constant__ Tf32Maps maps, const Tf32Params p) {
  extern __shared__ uint8_t smem_raw[];
  const int tm = blockIdx.x, tn = blockIdx.y;
  const int m0 = tm * TBM, n0 = tn * TBN;
  if ((p.flags & CAPITAL_GEMM_C_UPPER) && m0 > n0 + p.noff + TBN - 1) return;  // tile strictly below the diagonal (whole CTA)
  // an earlier CTA's watchdog fired: the launch is lost, do not spend 2 s per remaining tile (block-uniform decision)
  if (__syncthreads_or(*(volatile int*)p.err == -3)) return;
  const int nk = (p.K + TBK - 1) / TBK;
  const int niter = nk * p.npair;

  const uint32_t raw_u32 = smem_u32(smem_raw);
  const uint32_t smem_base = (raw_u32 + 1023u) & ~1023u;
  const uint32_t full0 = smem_base + TSTAGES * T_STAGE_BYTES;
  const uint32_t empty0 = full0 + TSTAGES * 8;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (threadIdx.x == 0) {
    for (int s = 0; s < TSTAGES; s++) {
      mbar_init(full0 + s * 8, 1);
      mbar_init(empty0 + s * 8, T_CWG);
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  }
  __syncthreads();

  if (warp >= T_CWG * 4) {
    // ---------------- TMA producer warpgroup: one lane issues, the group gives its registers to the consumers ----------------
    asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(T_REG_PRODUCER));
    if (warp != T_CWG * 4 || lane != 0) return;
    int it = 0;
    for (int pr = 0; pr < p.npair; pr++) {
      const CUtensorMap* ma = &maps.a[pr];
      const CUtensorMap* mb = &maps.b[pr];
      for (int j = 0; j < nk; j++, it++) {
        const int s = it % TSTAGES;
        const uint32_t ph = (it / TSTAGES) & 1;
        if (!mbar_wait_bounded(empty0 + s * 8, ph ^ 1, p.err)) return;
        mbar_expect_tx(full0 + s * 8, T_STAGE_BYTES);
        tma_load_2d(smem_base + s * T_STAGE_BYTES, ma, full0 + s * 8, j * TBK, m0);
        tma_load_2d(smem_base + s * T_STAGE_BYTES + T_A_BYTES, mb, full0 + s * 8, j * TBK, n0);
      }
    }
    return;
  }

  // ---------------- wgmma consumers: warpgroup wg owns rows [64 wg, 64 wg + 64) of the tile ----------------
  asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(T_REG_CONSUMER));
  const int wg = warp >> 2;
  float part[64];  // FP32 partial of one stage
  double acc[64];  // FP64 sum of the partials
#pragma unroll
  for (int i = 0; i < 64; i++) acc[i] = 0.0;
  bool have = true;
  for (int it = 0; it < niter; it++) {
    const int s = it % TSTAGES;
    const uint32_t ph = (it / TSTAGES) & 1;
    if (!wg_all(mbar_wait_bounded(full0 + s * 8, ph, p.err), wg)) { have = false; break; }
    const uint64_t da = wgmma_desc_k_sw128(smem_base + s * T_STAGE_BYTES + wg * 64 * 128);
    const uint64_t db = wgmma_desc_k_sw128(smem_base + s * T_STAGE_BYTES + T_A_BYTES);
    asm volatile("wgmma.fence.sync.aligned;" ::: "memory");
    // 8 floats = 32 bytes further along K inside the swizzle row: start address + 2 (>> 4)
    wgmma_m64n128k8_tf32<0>(part, da, db);
#pragma unroll
    for (int k8 = 1; k8 < TBK / 8; k8++) wgmma_m64n128k8_tf32<1>(part, da + (uint64_t)(2 * k8), db + (uint64_t)(2 * k8));
    asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory");
    asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory");
    if ((threadIdx.x & 127) == 0) mbar_arrive(empty0 + s * 8);  // this warpgroup has finished reading the stage
#pragma unroll
    for (int i = 0; i < 64; i++) acc[i] += (double)part[i];
  }
  if (!have) return;

  // ---------------- epilogue: fragment (j, i, e) of thread (warp w, lane l) is row 16 w + l / 4 + 8 i, column 8 j + 2 (l % 4) + e ----------------
  const double alpha = p.alpha, beta = p.beta;
  const bool upper_only = p.flags & CAPITAL_GEMM_C_UPPER;
  const int rbase = m0 + wg * 64 + (warp & 3) * 16 + (lane >> 2);
#pragma unroll
  for (int j = 0; j < TBN / 8; j++) {
#pragma unroll
    for (int e = 0; e < 2; e++) {
      const int col = n0 + j * 8 + 2 * (lane & 3) + e;
      if (col >= p.N) continue;
#pragma unroll
      for (int i = 0; i < 2; i++) {
        const int row = rbase + 8 * i;
        if (row >= p.M || (upper_only && row > col + p.noff)) continue;
        double* cc = p.C + (long long)col * p.ldc + row;
        double r = alpha * acc[4 * j + 2 * i + e];
        if (beta != 0.0) r += beta * *cc;
        *cc = r;
      }
    }
  }
}

// FP64 window (k x cols, ld) -> FP32 copies rounded to TF32 (cvt.rna): hi, and optionally lo = tf32(x - hi)
__global__ void to_tf32_kernel(long long k, long long cols, const double* src, long long ld, float* hi, float* lo, long long ldf) {
  const long long total = k * cols;
  for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < total; idx += (long long)gridDim.x * blockDim.x) {
    const long long c = idx / k, r = idx - c * k;
    const double x = src[c * ld + r];
    uint32_t h;
    asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(h) : "f"((float)x));
    const float hf = __uint_as_float(h);
    hi[c * ldf + r] = hf;
    if (lo) {
      uint32_t l;
      asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(l) : "f"((float)(x - (double)hf)));
      lo[c * ldf + r] = __uint_as_float(l);
    }
  }
}

capital_status_t make_map_f32(capital_ctx* ctx, CUtensorMap* map, const float* base, int64_t k, int64_t cols, int64_t ldf, int box_cols) {
  cuuint64_t dims[2] = {(cuuint64_t)k, (cuuint64_t)cols};
  cuuint64_t strides[1] = {(cuuint64_t)ldf * 4};
  cuuint32_t box[2] = {(cuuint32_t)TBK, (cuuint32_t)box_cols};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = ctx->encode(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, (void*)base, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                           CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    ctx->set_error("cuTensorMapEncodeTiled (f32) failed: CUresult " + std::to_string((int)r));
    return CAPITAL_ERR_CUDA;
  }
  return CAPITAL_OK;
}

const char* stream_tag(const capital_ctx* ctx, cudaStream_t st) {
  if (st == ctx->side) return "_s0";
  if (st == ctx->side_deep[0]) return "_s1";
  if (st == ctx->side_deep[1]) return "_s2";
  if (st == ctx->hi) return "_hi";
  return "";
}

}  // namespace

capital_status_t gemm_tf32_init(capital_ctx* ctx) {
  CAP_CUDA(cudaFuncSetAttribute(gemm_tn_tf32_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, T_SMEM));
  return CAPITAL_OK;
}

// C = beta C + alpha sum over classes A_c^T B_c, operands given in FP64 and converted here (workspaces are per stream: a product on the
// deferred stream must not reuse the buffers of one in flight on the chain).  passes = 1 (TF32) or 3 (split operands).
capital_status_t gemm_tn_tf32_x(capital_ctx* ctx, cudaStream_t st, int64_t m, int64_t n, int64_t k, double alpha, const GemmOperands& ops,
                                double beta, double* C, int64_t ldc, int flags, int noff, int passes) {
  if (m <= 0 || n <= 0 || k <= 0) return CAPITAL_OK;
  if ((passes != 1 && passes != 3) || ops.ncls < 1 || ops.ncls > GEMM_NCLS_MAX || ops.lda < k || ops.ldb < k || ldc < m ||
      (flags & ~CAPITAL_GEMM_C_UPPER) || m >= (1LL << 31) - 256 || n >= (1LL << 31) - 256 || k >= (1LL << 31) - 256) {
    ctx->set_error("gemm_tn_tf32: unsupported arguments (passes 1 or 3, only the C_UPPER structure flag)");
    return CAPITAL_ERR_INVALID;
  }
  if (!ctx->tf32_ready) {
    CAP_TRY(gemm_tf32_init(ctx));
    ctx->tf32_ready = true;
  }
  const std::string tag = stream_tag(ctx, st);
  const int64_t ldf = round_up(k, 4);  // 16-byte rows for TMA
  Tf32Maps maps;
  memset(&maps, 0, sizeof(maps));
  Tf32Params p{};
  int np = 0;
  for (int c = 0; c < ops.ncls; c++) {
    const bool same = ops.A[c] == ops.B[c] && ops.lda == ops.ldb && m == n;
    float *ahi, *alo = nullptr, *bhi, *blo = nullptr;
    const std::string sfx = tag + std::to_string(c);
    CAP_TRY(ctx->workspace("tf32_ahi" + sfx, (size_t)ldf * m * 4, (void**)&ahi));
    if (passes == 3) CAP_TRY(ctx->workspace("tf32_alo" + sfx, (size_t)ldf * m * 4, (void**)&alo));
    const int gr = (int)std::min<long long>(((long long)k * std::max(m, n) + 255) / 256, (long long)ctx->num_sms * 8);
    to_tf32_kernel<<<gr, 256, 0, st>>>(k, m, ops.A[c], ops.lda, ahi, alo, ldf);
    ctx->counters.kernel_launches++;
    if (same) { bhi = ahi; blo = alo; }
    else {
      CAP_TRY(ctx->workspace("tf32_bhi" + sfx, (size_t)ldf * n * 4, (void**)&bhi));
      if (passes == 3) CAP_TRY(ctx->workspace("tf32_blo" + sfx, (size_t)ldf * n * 4, (void**)&blo));
      to_tf32_kernel<<<gr, 256, 0, st>>>(k, n, ops.B[c], ops.ldb, bhi, blo, ldf);
      ctx->counters.kernel_launches++;
    }
    CAP_CUDA(cudaGetLastError());
    const float* pa[3] = {ahi, ahi, alo};
    const float* pb[3] = {bhi, blo, bhi};
    for (int q = 0; q < passes; q++, np++) {
      CAP_TRY(make_map_f32(ctx, &maps.a[np], pa[q], k, m, ldf, TBM));
      CAP_TRY(make_map_f32(ctx, &maps.b[np], pb[q], k, n, ldf, TBN));
    }
  }
  p.M = (int)m; p.N = (int)n; p.K = (int)k; p.npair = np; p.flags = flags; p.noff = noff;
  p.gm = (int)ceil_div(m, TBM); p.gn = (int)ceil_div(n, TBN);
  p.alpha = alpha; p.beta = beta; p.C = C; p.ldc = ldc; p.err = ctx->d_info;
  dim3 grid((unsigned)p.gm, (unsigned)p.gn, 1);
  const int tli = ctx->tl_begin(st, 9, (double)m, (double)n, (double)k);
  gemm_tn_tf32_kernel<<<grid, T_THREADS, T_SMEM, st>>>(maps, p);
  ctx->tl_end(st, tli);
  CAP_CUDA(cudaGetLastError());
  ctx->counters.kernel_launches++;
  ctx->tf32_launches++;
  ctx->tf32_flops += 2.0 * (double)m * (double)n * (double)k * ops.ncls * passes * ((flags & CAPITAL_GEMM_C_UPPER) ? 0.5 : 1.0);
  return CAPITAL_OK;
}

capital_status_t gemm_tn_tf32(capital_ctx* ctx, cudaStream_t st, int64_t m, int64_t n, int64_t k, double alpha, const double* A, int64_t lda,
                              const double* B, int64_t ldb, double beta, double* C, int64_t ldc, int flags, int passes) {
  GemmOperands ops;
  ops.A[0] = A; ops.B[0] = B; ops.lda = lda; ops.ldb = ldb;
  return gemm_tn_tf32_x(ctx, st, m, n, k, alpha, ops, beta, C, ldc, flags, 0, passes);
}
