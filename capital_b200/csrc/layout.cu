// HBM-bound helpers around the GEMM kernel: window copies / transposes (what serialize<S,D>::invoke does on
// the CPU, serialize.hpp:12-150, reduced to the few that remain once operands are used in place), packed
// upper <-> rect conversion (structure.h:37-39), the reference's generators (structure.hpp:69-129) and the
// validators' Frobenius reductions (util.hpp:25-53).  All kernels are coalesced along the contiguous
// (row) index and sized in multiples of the SM count where the extent allows.
#include "common.cuh"
#include <algorithm>

namespace {

constexpr int TP = 32;

__global__ void transpose_kernel(int rows, int cols, const double* src, long long lds, double* dst,
                                 long long ldd, double scale) {
  __shared__ double tile[TP][TP + 1];
  const int r0 = blockIdx.x * TP, c0 = blockIdx.y * TP;
  for (int j = threadIdx.y; j < TP; j += blockDim.y) {
    const int r = r0 + threadIdx.x, c = c0 + j;
    if (r < rows && c < cols) tile[j][threadIdx.x] = src[(long long)c * lds + r];
  }
  __syncthreads();
  // dst is cols x rows: dst(c, r) = src(r, c)
  for (int j = threadIdx.y; j < TP; j += blockDim.y) {
    const int c = c0 + threadIdx.x, r = r0 + j;
    if (r < rows && c < cols) dst[(long long)r * ldd + c] = scale * tile[threadIdx.x][j];
  }
}

__global__ void copy_kernel(long long rows, long long cols, const double* src, long long lds, double* dst,
                            long long ldd) {
  const long long total = rows * cols;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long c = i / rows, r = i - c * rows;
    dst[c * ldd + r] = src[c * lds + r];
  }
}

__global__ void zero_kernel(long long rows, long long cols, double* dst, long long ldd) {
  const long long total = rows * cols;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long c = i / rows, r = i - c * rows;
    dst[c * ldd + r] = 0.0;
  }
}

// one block per column chunk: column i of the packed triangle is contiguous (i+1 entries at i(i+1)/2); rows [0, skip_top) of the
// columns from skip_top on are neither read nor written
__global__ void pack_upper_kernel(long long c0, long long n, const double* src, long long lds, double* packed,
                                  int zero_diag, long long skip_top) {
  for (long long i = c0 + blockIdx.x; i < n; i += gridDim.x) {
    const double* s = src + i * lds;
    double* d = packed + i * (i + 1) / 2;
    for (long long j = (i >= skip_top ? skip_top : 0) + threadIdx.x; j <= i; j += blockDim.x) d[j] = (zero_diag && j == i) ? 0.0 : s[j];
  }
}
// rows [0, top) of the packed columns [top, n)
__global__ void zero_packed_top_kernel(long long top, long long n, double* packed) {
  for (long long i = top + blockIdx.x; i < n; i += gridDim.x) {
    double* d = packed + i * (i + 1) / 2;
    for (long long j = threadIdx.x; j < top; j += blockDim.x) d[j] = 0.0;
  }
}
__global__ void unpack_upper_kernel(long long n, const double* packed, double* dst, long long ldd) {
  for (long long i = blockIdx.x; i < n; i += gridDim.x) {
    const double* s = packed + i * (i + 1) / 2;
    double* d = dst + i * ldd;
    for (long long j = threadIdx.x; j < n; j += blockDim.x) d[j] = j <= i ? s[j] : 0.0;
  }
}
__global__ void triu_copy_kernel(long long n, const double* src, long long lds, double* dst, long long ldd,
                                 int zero_diag) {
  for (long long i = blockIdx.x; i < n; i += gridDim.x) {
    const double* s = src + i * lds;
    double* d = dst + i * ldd;
    for (long long j = threadIdx.x; j < n; j += blockDim.x) d[j] = (j < i || (j == i && !zero_diag)) ? s[j] : 0.0;
  }
}

// The full local block of a symmetric result of which only the upper half was computed: out(r, c) = U(r, c) where the GLOBAL position
// (y + d r, x + d c) lies on or above the diagonal, else the mirror source S -- read transposed (S(c, r): U itself on one GPU) or as
// it is (on a grid: the transpose partner's upper half, already transposed).  One pass over 32 x 32 tiles; a transposed read is
// staged in shared memory so that it stays coalesced too, and tiles wholly above the diagonal read U only.
__global__ void sym_merge_kernel(int n, const double* U, long long ldu, const double* S, long long lds, int s_trans, double* out,
                                 long long ldo, int x, int y, int d) {
  __shared__ double tile[TP][TP + 1];
  const int r0 = blockIdx.x * TP, c0 = blockIdx.y * TP;
  const bool all_upper = y + (long long)d * (r0 + TP - 1) <= x + (long long)d * c0;  // the tile's bottom-left corner is
  if (s_trans && !all_upper) {
    for (int j = threadIdx.y; j < TP; j += blockDim.y) {
      const int r = r0 + j, c = c0 + threadIdx.x;
      if (r < n && c < n) tile[j][threadIdx.x] = S[(long long)r * lds + c];  // S(c, r)
    }
    __syncthreads();
  }
  for (int j = threadIdx.y; j < TP; j += blockDim.y) {
    const int c = c0 + j, r = r0 + threadIdx.x;
    if (r >= n || c >= n) continue;
    const bool up = y + (long long)d * r <= x + (long long)d * c;
    out[(long long)c * ldo + r] = up ? U[(long long)c * ldu + r] : (s_trans ? tile[threadIdx.x][j] : S[(long long)c * lds + r]);
  }
}

// The operand U^T of sygst's split A = U + U^T (U = triu(A) with its diagonal halved): dst(r, c) = A(r, c) where the GLOBAL position
// (y + d r, x + d c) lies strictly below the diagonal, A(r, c) / 2 on it, 0 above it.  Entries above the global diagonal are never
// read, so whatever they hold (NaN included) cannot reach the result.
__global__ void tril_half_copy_kernel(long long n, const double* src, long long lds, double* dst, long long ldd, int x, int y, int d) {
  for (long long c = blockIdx.x; c < n; c += gridDim.x) {
    const double* s = src + c * lds;
    double* o = dst + c * ldd;
    const long long gc = x + (long long)d * c;
    for (long long r = threadIdx.x; r < n; r += blockDim.x) {
      const long long gr = y + (long long)d * r;
      o[r] = gr > gc ? s[r] : (gr == gc ? 0.5 * s[r] : 0.0);
    }
  }
}

// Copy-in of the batched factor: W_b (nb x nb, ld nb, at W + b nb nb) from the upper triangle of A_b (n x n, ld n, at A + b n n),
// mirrored below the diagonal, and the identity in rows and columns n .. nb.  A's strictly lower triangle is never read.  The mirror
// is a transposed read, staged in shared memory so that it stays coalesced; tiles wholly above the diagonal skip it.
__global__ void sym_pad_batched_kernel(int n, int nb, const double* A, double* W) {
  __shared__ double tile[TP][TP + 1];
  const long long b = blockIdx.z;
  A += b * n * n;
  W += b * nb * nb;
  const int r0 = blockIdx.x * TP, c0 = blockIdx.y * TP;
  if (r0 + TP - 1 > c0) {
    for (int j = threadIdx.y; j < TP; j += blockDim.y) {
      const int r = r0 + j, c = c0 + threadIdx.x;  // A(c, r), the mirror of element (r, c)
      if (r < n && c < r) tile[j][threadIdx.x] = A[(long long)r * n + c];
    }
  }
  __syncthreads();
  for (int j = threadIdx.y; j < TP; j += blockDim.y) {
    const int c = c0 + j, r = r0 + threadIdx.x;
    double v = r == c ? 1.0 : 0.0;
    if (r < n && c < n) v = r <= c ? A[(long long)c * n + r] : tile[threadIdx.x][j];
    W[(long long)c * nb + r] = v;
  }
}

// dst_b (n x n, ld ldd, at dst + b sd) = the upper triangle of the leading n x n block of src_b (ld lds, at src + b ss), exact zeros
// below the diagonal; src's strictly lower triangle is never read.  The copy-out of the batched factor, and the copy-in of a factor
// into the ld-padded workspace of the batched inverse, sygst and products.
__global__ void triu_out_batched_kernel(long long n, long long batch, const double* src, long long lds, long long ss, double* dst,
                                        long long ldd, long long sd) {
  const long long nn = n * n, total = nn * batch;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long b = i / nn, e = i - b * nn, c = e / n, r = e - c * n;
    dst[b * sd + c * ldd + r] = r <= c ? src[b * ss + c * lds + r] : 0.0;
  }
}

// The operand U^T of the batched sygst on matrix blockIdx.z: dst_b (ld ldd, at dst + b sd) = U_b^T with U_b = triu(A_b), its diagonal
// halved, zeros above U^T's diagonal -- tril_half_copy's operand on one GPU, but read from A_b's UPPER triangle (n x n, ld lds, at
// src + b ss; the triangle the batched factor reads), which for a symmetric A holds the same values.  A's strict lower triangle is never
// read.  A transpose of 32 x 32 tiles through shared memory, so that the reads and the writes stay coalesced.
__global__ void tril_half_batched_kernel(int n, const double* src, long long lds, long long ss, double* dst, long long ldd, long long sd) {
  __shared__ double tile[TP][TP + 1];
  src += (long long)blockIdx.z * ss;
  dst += (long long)blockIdx.z * sd;
  const int r0 = blockIdx.x * TP, c0 = blockIdx.y * TP;
  for (int j = threadIdx.y; j < TP; j += blockDim.y) {
    const int r = r0 + threadIdx.x, c = c0 + j;
    if (r < n && c < n) tile[j][threadIdx.x] = r < c ? src[(long long)c * lds + r] : (r == c ? 0.5 * src[(long long)c * lds + r] : 0.0);
  }
  __syncthreads();
  // dst(c, r) = U(r, c)
  for (int j = threadIdx.y; j < TP; j += blockDim.y) {
    const int c = c0 + threadIdx.x, r = r0 + j;
    if (r < n && c < n) dst[(long long)r * ldd + c] = tile[threadIdx.x][j];
  }
}

// sym_merge_kernel (one GPU: S = U read transposed) on matrix blockIdx.z of a batch: out_b(r, c) = U_b(r, c) for r <= c, U_b(c, r)
// below the diagonal.  Only U's upper triangle reaches the output.
__global__ void sym_merge_batched_kernel(int n, const double* U, long long ldu, long long su, double* out, long long ldo, long long so) {
  __shared__ double tile[TP][TP + 1];
  U += (long long)blockIdx.z * su;
  out += (long long)blockIdx.z * so;
  const int r0 = blockIdx.x * TP, c0 = blockIdx.y * TP;
  const bool all_upper = r0 + TP - 1 <= c0;
  if (!all_upper) {
    for (int j = threadIdx.y; j < TP; j += blockDim.y) {
      const int r = r0 + j, c = c0 + threadIdx.x;
      if (r < n && c < n) tile[j][threadIdx.x] = U[(long long)r * ldu + c];  // U(c, r)
    }
    __syncthreads();
  }
  for (int j = threadIdx.y; j < TP; j += blockDim.y) {
    const int c = c0 + j, r = r0 + threadIdx.x;
    if (r >= n || c >= n) continue;
    out[(long long)c * ldo + r] = r <= c ? U[(long long)c * ldu + r] : tile[threadIdx.x][j];
  }
}

// dst_b (rows x cols, ld ldd, at dst + b sd) = src_b (ld lds, at src + b ss): the right-hand-side panels of the batched products
__global__ void copy_batched_kernel(long long rows, long long cols, long long batch, const double* src, long long lds, long long ss,
                                    double* dst, long long ldd, long long sd) {
  const long long per = rows * cols, total = per * batch;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long b = i / per, e = i - b * per, c = e / rows, r = e - c * rows;
    dst[b * sd + c * ldd + r] = src[b * ss + c * lds + r];
  }
}

// drand48: X0 = seed<<16 | 0x330E ; X1 = (a X0 + c) mod 2^48 ; value = X1 / 2^48  (structure.hpp:80-85 re-seeds per element)
__device__ __forceinline__ double drand48_first(unsigned long long seed) {
  const unsigned long long a = 0x5DEECE66DULL, c = 0xBULL, m48 = (1ULL << 48) - 1;
  unsigned long long x = ((seed & 0xFFFFFFFFULL) << 16) | 0x330EULL;
  x = (a * x + c) & m48;  // 64-bit wraparound keeps the low 48 bits exact
  return (double)x * (1.0 / 281474976710656.0);
}

__global__ void gen_symmetric_kernel(double* A, long long ld, long long lrows, long long lcols, long long n, int x, int y,
                                     int d, int diag_dom) {
  const long long total = lrows * lcols;
  for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < total; idx += (long long)gridDim.x * blockDim.x) {
    const long long i = idx / lrows, j = idx - i * lrows;  // local col i, local row j
    const long long gx = x + i * d, gy = y + j * d;
    double v = 0.0;
    if (gx < n && gy < n) {
      const unsigned long long hi = gx > gy ? gx : gy, lo = gx > gy ? gy : gx;
      v = drand48_first(hi + (unsigned long long)n * lo);
      if (diag_dom && gx == gy && i == j) v += (double)n;
    }
    A[i * ld + j] = v;
  }
}

// draw number t (0-based) of the stream after srand48(key): X_{t+1} = a^{t+1} X0 + c (a^{t+1}-1)/(a-1)
__device__ __forceinline__ void lcg_pow(unsigned long long t, unsigned long long& A, unsigned long long& C) {
  const unsigned long long m48 = (1ULL << 48) - 1;
  unsigned long long ca = 0x5DEECE66DULL, cc = 0xBULL;  // current step (a, c) for 2^bit
  A = 1; C = 0;
  while (t) {
    if (t & 1) { A = (A * ca) & m48; C = (C * ca + cc) & m48; }
    cc = (cc * ca + cc) & m48;
    ca = (ca * ca) & m48;
    t >>= 1;
  }
}
__global__ void gen_random_kernel(double* Aout, long long ld, long long lrows, long long lcols, long long pad_rows,
                                  long long pad_cols, long long key) {
  const unsigned long long m48 = (1ULL << 48) - 1;
  const unsigned long long x0 = (((unsigned long long)key & 0xFFFFFFFFULL) << 16) | 0x330EULL;
  const long long total = lrows * lcols;
  for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < total; idx += (long long)gridDim.x * blockDim.x) {
    const long long i = idx / lrows, j = idx - i * lrows;
    double v = 0.0;
    if (i < pad_cols && j < pad_rows) {
      unsigned long long A, C;
      lcg_pow((unsigned long long)(i * pad_rows + j) + 1ULL, A, C);
      const unsigned long long xv = (A * x0 + C) & m48;
      v = (double)xv * (1.0 / 281474976710656.0);
    }
    Aout[i * ld + j] = v;
  }
}

// upper_mode: 0 = all entries, 1 = only entries whose GLOBAL position satisfies row <= col
__global__ void sumsq_kernel(long long rows, long long cols, const double* a, long long ld, int upper_mode, int x, int y,
                             int d, double* out) {
  double s = 0.0;
  const long long total = rows * cols;
  for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < total; idx += (long long)gridDim.x * blockDim.x) {
    const long long i = idx / rows, j = idx - i * rows;
    if (upper_mode && (y + j * d) > (x + i * d)) continue;
    const double v = a[i * ld + j];
    s += v * v;
  }
  for (int o = 16; o; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  __shared__ double ws[32];
  if ((threadIdx.x & 31) == 0) ws[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x < 32) {
    s = threadIdx.x < (blockDim.x >> 5) ? ws[threadIdx.x] : 0.0;
    for (int o = 16; o; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (threadIdx.x == 0) atomicAdd(out, s);
  }
}

__global__ void sub_identity_kernel(long long n, double* a, long long ld) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) a[i * ld + i] -= 1.0;
}

// Shifted CholeskyQR3: the trace of an n x n block in a fixed order -- thread t adds the diagonal entries t, t + SHIFT_T, ... in
// turn, then a fixed shared-memory tree -- the same bits for the same block on every GPU.  One CTA of SHIFT_T threads.
constexpr int SHIFT_T = 256;
__device__ double diag_sum_cta(long long n, const double* a, long long ld) {
  __shared__ double red[SHIFT_T];
  double s = 0.0;
  for (long long i = threadIdx.x; i < n; i += SHIFT_T) s += a[i * ld + i];
  red[threadIdx.x] = s;
  __syncthreads();
  for (int h = SHIFT_T / 2; h; h >>= 1) {
    if (threadIdx.x < h) red[threadIdx.x] += red[threadIdx.x + h];
    __syncthreads();
  }
  return red[0];
}
__global__ void __launch_bounds__(SHIFT_T) gram_shift_kernel(long long n, double* G, long long ld, double coef) {
  const double s = coef * diag_sum_cta(n, G, ld);  // every diagonal read is behind the tree's barriers
  for (long long i = threadIdx.x; i < n; i += SHIFT_T) G[i * ld + i] += s;
}
__global__ void __launch_bounds__(SHIFT_T) gram_diag_partial_kernel(long long n, const double* G, long long ld, double* out) {
  const double s = diag_sum_cta(n, G, ld);
  if (threadIdx.x == 0) *out = s;
}
__global__ void __launch_bounds__(SHIFT_T) gram_shift_by_kernel(long long n, double* G, long long ld, const double* parts, int nparts,
                                                                double coef) {
  double t = 0.0;
  for (int k = 0; k < nparts; k++) {  // system-scope loads: the other partials were stored by peer GPUs' copy engines
    double v;
    asm volatile("ld.relaxed.sys.global.f64 %0, [%1];" : "=d"(v) : "l"(parts + k) : "memory");
    t += v;
  }
  const double s = coef * t;
  for (long long i = threadIdx.x; i < n; i += SHIFT_T) G[i * ld + i] += s;
}

__global__ void __launch_bounds__(SHIFT_T) gram_shift_batched_kernel(long long n, double* G, long long ld, long long sg, double coef) {
  G += (long long)blockIdx.x * sg;
  const double s = coef * diag_sum_cta(n, G, ld);
  for (long long i = threadIdx.x; i < n; i += SHIFT_T) G[i * ld + i] += s;
}

// transpose_kernel on matrix blockIdx.z of a batch
__global__ void transpose_batched_kernel(int rows, int cols, const double* src, long long lds, long long ss, double* dst, long long ldd,
                                         long long sd) {
  __shared__ double tile[TP][TP + 1];
  src += (long long)blockIdx.z * ss;
  dst += (long long)blockIdx.z * sd;
  const int r0 = blockIdx.x * TP, c0 = blockIdx.y * TP;
  for (int j = threadIdx.y; j < TP; j += blockDim.y) {
    const int r = r0 + threadIdx.x, c = c0 + j;
    if (r < rows && c < cols) tile[j][threadIdx.x] = src[(long long)c * lds + r];
  }
  __syncthreads();
  for (int j = threadIdx.y; j < TP; j += blockDim.y) {
    const int c = c0 + threadIdx.x, r = r0 + j;
    if (r < rows && c < cols) dst[(long long)r * ldd + c] = tile[threadIdx.x][j];
  }
}

// zero the band |row - col| <= hw of an n x n matrix: one block per column, contiguous rows
__global__ void zero_band_kernel(long long n, long long hw, double* a, long long ld) {
  for (long long c = blockIdx.x; c < n; c += gridDim.x) {
    const long long r0 = c - hw > 0 ? c - hw : 0, r1 = c + hw < n - 1 ? c + hw : n - 1;
    for (long long r = r0 + threadIdx.x; r <= r1; r += blockDim.x) a[c * ld + r] = 0.0;
  }
}

inline int grid_for(const capital_ctx* ctx, long long total, int threads) {
  long long b = (total + threads - 1) / threads;
  const long long cap = (long long)ctx->num_sms * 8;
  if (b > cap) b = cap;
  if (b < 1) b = 1;
  return (int)b;
}

}  // namespace

#define LAUNCH_CHECK()                      \
  do {                                      \
    ctx->counters.kernel_launches++;        \
    CAP_CUDA(cudaGetLastError());           \
  } while (0)

capital_status_t transpose_block(capital_ctx* ctx, cudaStream_t st, int64_t rows, int64_t cols, const double* src, int64_t lds,
                                 double* dst, int64_t ldd, double scale) {
  if (rows <= 0 || cols <= 0) return CAPITAL_OK;
  dim3 grid((unsigned)ceil_div(rows, TP), (unsigned)ceil_div(cols, TP)), block(TP, 8);
  const int tli = ctx->tl_begin(st, 8, 1, (double)rows, (double)cols);
  transpose_kernel<<<grid, block, 0, st>>>((int)rows, (int)cols, src, lds, dst, ldd, scale);
  ctx->tl_end(st, tli);
  LAUNCH_CHECK();
  return CAPITAL_OK;
}
capital_status_t copy_block(capital_ctx* ctx, cudaStream_t st, int64_t rows, int64_t cols, const double* src, int64_t lds, double* dst,
                            int64_t ldd) {
  if (rows <= 0 || cols <= 0) return CAPITAL_OK;
  if (lds == rows && ldd == rows) {
    const size_t total = (size_t)rows * cols * 8, piece = (size_t)1 << 30;  // pieces of at most 1 GiB (see dist.cu: dma2d)
    for (size_t off = 0; off < total; off += piece)
      CAP_CUDA(cudaMemcpyAsync((char*)dst + off, (const char*)src + off, std::min(piece, total - off), cudaMemcpyDeviceToDevice, st));
    return CAPITAL_OK;
  }
  const int tli = ctx->tl_begin(st, 8, 2, (double)rows, (double)cols);
  copy_kernel<<<grid_for(ctx, rows * cols, 256), 256, 0, st>>>(rows, cols, src, lds, dst, ldd);
  ctx->tl_end(st, tli);
  LAUNCH_CHECK();
  return CAPITAL_OK;
}
capital_status_t zero_block(capital_ctx* ctx, cudaStream_t st, int64_t rows, int64_t cols, double* dst, int64_t ldd) {
  if (rows <= 0 || cols <= 0) return CAPITAL_OK;
  if (ldd == rows) {
    CAP_CUDA(cudaMemsetAsync(dst, 0, (size_t)rows * cols * 8, st));
    return CAPITAL_OK;
  }
  zero_kernel<<<grid_for(ctx, rows * cols, 256), 256, 0, st>>>(rows, cols, dst, ldd);
  LAUNCH_CHECK();
  return CAPITAL_OK;
}
capital_status_t pack_upper(capital_ctx* ctx, cudaStream_t st, int64_t n, const double* src, int64_t lds, double* packed, int zero_diag,
                            int64_t col_begin, int64_t col_end, int64_t skip_top) {
  if (col_end < 0) col_end = n;
  if (skip_top <= 0) skip_top = n;
  const int64_t cols = col_end - col_begin;
  if (cols <= 0) return CAPITAL_OK;
  const int tli = ctx->tl_begin(st, 8, 3, (double)col_begin, (double)col_end);
  pack_upper_kernel<<<(int)(cols < ctx->num_sms * 8 ? cols : ctx->num_sms * 8), 256, 0, st>>>(col_begin, col_end, src, lds, packed, zero_diag,
                                                                                              skip_top);
  ctx->tl_end(st, tli);
  LAUNCH_CHECK();
  return CAPITAL_OK;
}
capital_status_t zero_packed_top(capital_ctx* ctx, cudaStream_t st, int64_t n, double* packed, int64_t top) {
  if (top <= 0 || top >= n) return CAPITAL_OK;
  const int64_t cols = n - top;
  const int tli = ctx->tl_begin(st, 8, 4, (double)top, (double)n);
  zero_packed_top_kernel<<<(int)(cols < ctx->num_sms * 8 ? cols : ctx->num_sms * 8), 256, 0, st>>>(top, n, packed);
  ctx->tl_end(st, tli);
  LAUNCH_CHECK();
  return CAPITAL_OK;
}
capital_status_t unpack_upper(capital_ctx* ctx, cudaStream_t st, int64_t n, const double* packed, double* dst, int64_t ldd) {
  if (n <= 0) return CAPITAL_OK;
  unpack_upper_kernel<<<(int)(n < ctx->num_sms * 8 ? n : ctx->num_sms * 8), 256, 0, st>>>(n, packed, dst, ldd);
  LAUNCH_CHECK();
  return CAPITAL_OK;
}
capital_status_t triu_copy(capital_ctx* ctx, cudaStream_t st, int64_t n, const double* src, int64_t lds, double* dst, int64_t ldd,
                           int zero_diag) {
  if (n <= 0) return CAPITAL_OK;
  triu_copy_kernel<<<(int)(n < ctx->num_sms * 8 ? n : ctx->num_sms * 8), 256, 0, st>>>(n, src, lds, dst, ldd, zero_diag);
  LAUNCH_CHECK();
  return CAPITAL_OK;
}
capital_status_t sym_merge(capital_ctx* ctx, cudaStream_t st, int64_t n, const double* U, int64_t ldu, const double* S, int64_t lds,
                           bool s_trans, double* out, int64_t ldo, int x, int y, int d) {
  if (n <= 0) return CAPITAL_OK;
  dim3 grid((unsigned)ceil_div(n, TP), (unsigned)ceil_div(n, TP)), block(TP, 8);
  sym_merge_kernel<<<grid, block, 0, st>>>((int)n, U, ldu, S, lds, s_trans ? 1 : 0, out, ldo, x, y, d);
  LAUNCH_CHECK();
  return CAPITAL_OK;
}
capital_status_t tril_half_copy(capital_ctx* ctx, cudaStream_t st, int64_t n, const double* src, int64_t lds, double* dst, int64_t ldd,
                                int x, int y, int d) {
  if (n <= 0) return CAPITAL_OK;
  tril_half_copy_kernel<<<(int)(n < ctx->num_sms * 8 ? n : ctx->num_sms * 8), 256, 0, st>>>(n, src, lds, dst, ldd, x, y, d);
  LAUNCH_CHECK();
  return CAPITAL_OK;
}
capital_status_t sym_pad_batched(capital_ctx* ctx, cudaStream_t st, int64_t n, int64_t nb, int64_t batch, const double* A, double* W) {
  if (n <= 0 || batch <= 0) return CAPITAL_OK;
  if (nb < n || nb % TP != 0 || batch > 65535) return CAPITAL_ERR_INVALID;
  dim3 grid((unsigned)(nb / TP), (unsigned)(nb / TP), (unsigned)batch), block(TP, 8);
  sym_pad_batched_kernel<<<grid, block, 0, st>>>((int)n, (int)nb, A, W);
  LAUNCH_CHECK();
  return CAPITAL_OK;
}
capital_status_t triu_out_batched(capital_ctx* ctx, cudaStream_t st, int64_t n, int64_t batch, const double* src, int64_t lds, int64_t ss,
                                  double* dst, int64_t ldd, int64_t sd) {
  if (n <= 0 || batch <= 0) return CAPITAL_OK;
  triu_out_batched_kernel<<<grid_for(ctx, n * n * batch, 256), 256, 0, st>>>(n, batch, src, lds, ss, dst, ldd, sd);
  LAUNCH_CHECK();
  return CAPITAL_OK;
}
capital_status_t tril_half_batched(capital_ctx* ctx, cudaStream_t st, int64_t n, int64_t batch, const double* src, int64_t lds, int64_t ss,
                                   double* dst, int64_t ldd, int64_t sd) {
  if (n <= 0 || batch <= 0) return CAPITAL_OK;
  if (batch > 65535) return CAPITAL_ERR_INVALID;
  dim3 grid((unsigned)ceil_div(n, TP), (unsigned)ceil_div(n, TP), (unsigned)batch), block(TP, 8);
  tril_half_batched_kernel<<<grid, block, 0, st>>>((int)n, src, lds, ss, dst, ldd, sd);
  LAUNCH_CHECK();
  return CAPITAL_OK;
}
capital_status_t sym_merge_batched(capital_ctx* ctx, cudaStream_t st, int64_t n, int64_t batch, const double* U, int64_t ldu, int64_t su,
                                   double* out, int64_t ldo, int64_t so) {
  if (n <= 0 || batch <= 0) return CAPITAL_OK;
  if (batch > 65535) return CAPITAL_ERR_INVALID;
  dim3 grid((unsigned)ceil_div(n, TP), (unsigned)ceil_div(n, TP), (unsigned)batch), block(TP, 8);
  sym_merge_batched_kernel<<<grid, block, 0, st>>>((int)n, U, ldu, su, out, ldo, so);
  LAUNCH_CHECK();
  return CAPITAL_OK;
}
capital_status_t copy_batched(capital_ctx* ctx, cudaStream_t st, int64_t rows, int64_t cols, int64_t batch, const double* src, int64_t lds,
                              int64_t ss, double* dst, int64_t ldd, int64_t sd) {
  if (rows <= 0 || cols <= 0 || batch <= 0) return CAPITAL_OK;
  copy_batched_kernel<<<grid_for(ctx, rows * cols * batch, 256), 256, 0, st>>>(rows, cols, batch, src, lds, ss, dst, ldd, sd);
  LAUNCH_CHECK();
  return CAPITAL_OK;
}
capital_status_t gen_symmetric(capital_ctx* ctx, cudaStream_t st, double* A, int64_t ld, int64_t lrows, int64_t lcols, int64_t n_global,
                               int x, int y, int d, int diag_dom) {
  gen_symmetric_kernel<<<grid_for(ctx, lrows * lcols, 256), 256, 0, st>>>(A, ld, lrows, lcols, n_global, x, y, d, diag_dom);
  LAUNCH_CHECK();
  return CAPITAL_OK;
}
capital_status_t gen_random(capital_ctx* ctx, cudaStream_t st, double* A, int64_t ld, int64_t lrows, int64_t lcols, int64_t pad_rows,
                            int64_t pad_cols, int64_t key) {
  gen_random_kernel<<<grid_for(ctx, lrows * lcols, 256), 256, 0, st>>>(A, ld, lrows, lcols, pad_rows, pad_cols, key);
  LAUNCH_CHECK();
  return CAPITAL_OK;
}
capital_status_t sumsq_block(capital_ctx* ctx, cudaStream_t st, int64_t rows, int64_t cols, const double* a, int64_t ld, int upper_mode,
                             int x, int y, int d, double* out) {
  if (rows <= 0 || cols <= 0) return CAPITAL_OK;
  sumsq_kernel<<<grid_for(ctx, rows * cols, 256), 256, 0, st>>>(rows, cols, a, ld, upper_mode, x, y, d, out);
  LAUNCH_CHECK();
  return CAPITAL_OK;
}
capital_status_t sub_identity_local(capital_ctx* ctx, cudaStream_t st, int64_t n, double* a, int64_t ld) {
  sub_identity_kernel<<<grid_for(ctx, n, 256), 256, 0, st>>>(n, a, ld);
  LAUNCH_CHECK();
  return CAPITAL_OK;
}
capital_status_t gram_shift(capital_ctx* ctx, cudaStream_t st, int64_t n, double* G, int64_t ld, double coef) {
  if (n <= 0) return CAPITAL_OK;
  gram_shift_kernel<<<1, SHIFT_T, 0, st>>>(n, G, ld, coef);
  LAUNCH_CHECK();
  return CAPITAL_OK;
}
capital_status_t gram_shift_batched(capital_ctx* ctx, cudaStream_t st, int64_t n, int64_t batch, double* G, int64_t ld, int64_t sg,
                                    double coef) {
  if (n <= 0 || batch <= 0) return CAPITAL_OK;
  if (batch > 65535) return CAPITAL_ERR_INVALID;
  gram_shift_batched_kernel<<<(unsigned)batch, SHIFT_T, 0, st>>>(n, G, ld, sg, coef);
  LAUNCH_CHECK();
  return CAPITAL_OK;
}
capital_status_t transpose_batched(capital_ctx* ctx, cudaStream_t st, int64_t rows, int64_t cols, int64_t batch, const double* src,
                                   int64_t lds, int64_t ss, double* dst, int64_t ldd, int64_t sd) {
  if (rows <= 0 || cols <= 0 || batch <= 0) return CAPITAL_OK;
  if (batch > 65535 || ceil_div(cols, TP) > 65535) return CAPITAL_ERR_INVALID;
  dim3 grid((unsigned)ceil_div(rows, TP), (unsigned)ceil_div(cols, TP), (unsigned)batch), block(TP, 8);
  transpose_batched_kernel<<<grid, block, 0, st>>>((int)rows, (int)cols, src, lds, ss, dst, ldd, sd);
  LAUNCH_CHECK();
  return CAPITAL_OK;
}
capital_status_t gram_diag_partial(capital_ctx* ctx, cudaStream_t st, int64_t n, const double* G, int64_t ld, double* out) {
  gram_diag_partial_kernel<<<1, SHIFT_T, 0, st>>>(n, G, ld, out);
  LAUNCH_CHECK();
  return CAPITAL_OK;
}
capital_status_t gram_shift_by(capital_ctx* ctx, cudaStream_t st, int64_t n, double* G, int64_t ld, const double* parts, int nparts,
                               double coef) {
  if (n <= 0) return CAPITAL_OK;
  gram_shift_by_kernel<<<1, SHIFT_T, 0, st>>>(n, G, ld, parts, nparts, coef);
  LAUNCH_CHECK();
  return CAPITAL_OK;
}

// The triangular products read whole diagonal GEMM tiles (<= 128 wide) of Rinv / Rinv^T, including entries on the other side of
// the diagonal that no kernel writes; everything farther than one tile from the diagonal is either written before it is read
// or never read.  Zeroing the band |row - col| <= 256 therefore replaces a memset of the whole n x n buffer.
capital_status_t zero_band(capital_ctx* ctx, cudaStream_t st, int64_t n, double* a, int64_t ld) {
  if (n <= 0) return CAPITAL_OK;
  const int64_t hw = 256;
  if (n <= 4 * hw) {
    CAP_CUDA(cudaMemsetAsync(a, 0, (size_t)ld * n * 8, st));
    return CAPITAL_OK;
  }
  const int tli = ctx->tl_begin(st, 8, 5, (double)n, (double)hw);
  zero_band_kernel<<<(int)(n < ctx->num_sms * 8 ? n : ctx->num_sms * 8), 256, 0, st>>>(n, hw, a, ld);
  ctx->tl_end(st, tli);
  LAUNCH_CHECK();
  return CAPITAL_OK;
}
