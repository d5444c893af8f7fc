// Batched symmetric eigensolver (capital_syevj_batched_f64): parallel cyclic Jacobi for many small matrices, n <= 512.
//
//   n <= 64   syevj_small_kernel: one CTA per matrix, A and V in shared memory, circle-method Jacobi steps of n/2 disjoint
//             rotations, then the sort.  No host synchronisation.
//   n > 64    block Jacobi over Np = roundup(n, 64) in global memory, N = Np / 32 blocks of 32 columns.  Per outer step the blocks
//             are paired by the circle method; every (matrix, pair (I, J)) diagonalises its 64 x 64 subproblem
//             S = [A_II A_IJ; A_JI A_JJ] with the n <= 64 routine (syevj_pair_kernel), then A_PP' <- Q_P^T A_PP' Q_P' and
//             V[:, P] <- V[:, P] Q_P run as 64 x 64 x 64 DMMA tile products (syevj_update_kernel).  A matrix has converged after an
//             outer sweep in which no subproblem rotated; its CTAs exit at once from then on.  The host reads one counter per sweep.
//
// Threshold: rotation (p, q) is skipped iff |a_pq| <= max(u sqrt|a_pp| sqrt|a_qq|, u ||A||_F), u = 2^-53, ||A||_F of the input.
// The first term is the Demmel-Veselic relative criterion.  The floor keeps singular and graded matrices from rotating forever:
// every rotation of a row holding an O(||A||) entry leaves rounding noise of order u ||A|| in its other entries, so a floor below
// that level (u ||A||_F / n was tried) chases noise, and graded matrices (eigenvalues 1e-15 .. 1) at n = 512 did not converge in 30
// sweeps.  Dropping the entries below the floor moves an eigenvalue by at most ||E||_2 <= ||E||_F <= n u ||A||_F.  Every formula is exact under a
// scaling of A by 4^k (sqrt|a_pp| sqrt|a_qq| rather than sqrt|a_pp a_qq|, a norm summed at the scale of the largest entry), so a
// matrix scaled by 4^k gets 2^2k times the bits of the unscaled one as long as nothing underflows.
//
// Padding: pad rows and columns are exactly zero off the diagonal (zero on it), so every rotation that would couple a pad index with
// a real one sees a_pq = 0 and is skipped, and every product keeps those couplings exactly zero.  The finish drops pad indices by
// position.
#include "common.cuh"
#include "tile64.cuh"
#include <algorithm>
#include <cfloat>

namespace {
// Bound on the (outer) sweeps.  Cyclic Jacobi converges quadratically: FP64 matrices take 6 to 10 sweeps, and a sweep in which
// nothing rotated ends the iteration.  A matrix that has not converged after 30 reports info = 1 with its last iterate.
constexpr int SYEVJ_SWEEPS = 30;
constexpr double SYEVJ_U = 0x1p-53;
constexpr int LDJ = 65;        // the Jacobi arrays: A and V of up to 64 x 64, element (i, j) at [i + j LDJ]
constexpr int JT = 256;        // threads of every kernel here

struct JacobiScratch {
  double c[32], s[32], t[32];
  int p[32], q[32], fire[32];
};
constexpr int JACOBI_SMEM = 2 * 64 * LDJ * (int)sizeof(double) + (int)sizeof(JacobiScratch) + JT * (int)sizeof(double);
constexpr int UPDATE_SMEM = 4 * TILE_DOUBLES * (int)sizeof(double);

// Circle-method ("round-robin") pairing of m (even) players: step s in [0, m - 1), pair k in [0, m / 2).  Pair 0 is (s, m - 1), pair k
// ((s + k) mod (m - 1), (s - k) mod (m - 1)); every unordered pair comes up exactly once in the m - 1 steps.  Returns p < q.
__device__ __forceinline__ void circle_pair(int m, int s, int k, int& p, int& q) {
  int a, b;
  if (k == 0) {
    a = s; b = m - 1;
  } else {
    a = (s + k) % (m - 1);
    b = (s - k + m - 1) % (m - 1);
  }
  p = min(a, b); q = max(a, b);
}

// ||M||_F of the m x m matrix get(i, j), summed at the scale 2^e of its largest entry (exact under power-of-two scaling), in a fixed
// order (deterministic).  +Inf when an entry is NaN or infinite.  All JT threads call; red: JT doubles of shared scratch.
template <class Get>
__device__ double block_fro(int m, Get get, double* red) {
  const int tid = threadIdx.x, mm = m * m;
  double mx = 0.0;
  int bad = 0;
  for (int idx = tid; idx < mm; idx += JT) {
    const double x = fabs(get(idx % m, idx / m));
    bad |= !(x <= DBL_MAX);
    mx = fmax(mx, x);
  }
  bad = __syncthreads_or(bad);
  red[tid] = mx;
  __syncthreads();
  for (int h = JT / 2; h > 0; h >>= 1) {
    if (tid < h) red[tid] = fmax(red[tid], red[tid + h]);
    __syncthreads();
  }
  mx = red[0];
  __syncthreads();
  if (bad) return INFINITY;
  if (mx == 0.0) return 0.0;
  const int e = ilogb(mx);
  const double sc = ldexp(1.0, -e);
  double s = 0.0;
  for (int idx = tid; idx < mm; idx += JT) {
    const double x = get(idx % m, idx / m) * sc;
    s = fma(x, x, s);
  }
  red[tid] = s;
  __syncthreads();
  for (int h = JT / 2; h > 0; h >>= 1) {
    if (tid < h) red[tid] += red[tid + h];
    __syncthreads();
  }
  s = red[0];
  __syncthreads();
  return ldexp(sqrt(s), e);
}

// Cyclic Jacobi on the symmetric np x np matrix a (np even, <= 64), accumulating the rotations into v (a @ [i + j LDJ], exactly
// symmetric throughout).  Each step rotates the np / 2 pairs of one circle-method round at once: every thread owns whole 2 x 2
// blocks of pair x pair (and their mirrors), applies the column rotation and then the row rotation, and writes both halves from the
// same registers.  Returns true when a sweep rotated nothing within SYEVJ_SWEEPS; *first: whether the first sweep rotated.
__device__ bool jacobi64(double* __restrict__ a, double* __restrict__ v, int np, double floor_, JacobiScratch* js, bool* first) {
  const int tid = threadIdx.x, h = np >> 1;
  for (int sweep = 0; sweep < SYEVJ_SWEEPS; sweep++) {
    int rotated = 0;
    for (int step = 0; step < np - 1; step++) {
      int fire = 0;
      if (tid < h) {
        int p, q;
        circle_pair(np, step, tid, p, q);
        const double app = a[p + p * LDJ], aqq = a[q + q * LDJ], apq = a[p + q * LDJ];
        const double thr = fmax(SYEVJ_U * (sqrt(fabs(app)) * sqrt(fabs(aqq))), floor_);
        fire = !(fabs(apq) <= thr);
        double c = 1.0, s = 0.0, t = 0.0;
        if (fire) {
          // Rutishauser: tan of the smaller angle that zeroes a_pq; for |tau| > 2^60, sqrt(1 + tau^2) = |tau| and t = 1 / (2 tau)
          const double tau = (aqq - app) / (2.0 * apq);
          t = fabs(tau) > 0x1p60 ? 0.5 / tau : copysign(1.0, tau) / (fabs(tau) + sqrt(fma(tau, tau, 1.0)));
          c = 1.0 / sqrt(fma(t, t, 1.0));
          s = t * c;
        }
        js->p[tid] = p; js->q[tid] = q; js->c[tid] = c; js->s[tid] = s; js->t[tid] = t; js->fire[tid] = fire;
      }
      if (!__syncthreads_or(fire)) continue;
      rotated = 1;
      for (int idx = tid; idx < 32 * 32; idx += JT) {  // 2 x 2 blocks (pair k rows, pair k2 columns), k <= k2
        const int k = idx >> 5, k2 = idx & 31;
        if (k2 >= h || k > k2) continue;
        const int fk = js->fire[k], fk2 = js->fire[k2];
        if (!fk && !fk2) continue;
        const int p = js->p[k], q = js->q[k];
        if (k == k2) {
          const double t = js->t[k], apq = a[p + q * LDJ];
          a[p + p * LDJ] -= t * apq;
          a[q + q * LDJ] += t * apq;
          a[p + q * LDJ] = 0.0;
          a[q + p * LDJ] = 0.0;
          continue;
        }
        const int p2 = js->p[k2], q2 = js->q[k2];
        const double c = js->c[k], s = js->s[k], c2 = js->c[k2], s2 = js->s[k2];
        const double x00 = a[p + p2 * LDJ], x01 = a[p + q2 * LDJ], x10 = a[q + p2 * LDJ], x11 = a[q + q2 * LDJ];
        // columns (p2, q2) by pair k2, then rows (p, q) by pair k
        const double y00 = c2 * x00 - s2 * x01, y01 = s2 * x00 + c2 * x01;
        const double y10 = c2 * x10 - s2 * x11, y11 = s2 * x10 + c2 * x11;
        const double z00 = c * y00 - s * y10, z10 = s * y00 + c * y10;
        const double z01 = c * y01 - s * y11, z11 = s * y01 + c * y11;
        a[p + p2 * LDJ] = z00; a[p + q2 * LDJ] = z01; a[q + p2 * LDJ] = z10; a[q + q2 * LDJ] = z11;
        a[p2 + p * LDJ] = z00; a[q2 + p * LDJ] = z01; a[p2 + q * LDJ] = z10; a[q2 + q * LDJ] = z11;
      }
      for (int idx = tid; idx < h * 64; idx += JT) {  // V[:, (p, q)] by pair k
        const int k = idx >> 6, i = idx & 63;
        if (i >= np || !js->fire[k]) continue;
        const int p = js->p[k], q = js->q[k];
        const double c = js->c[k], s = js->s[k], vp = v[i + p * LDJ], vq = v[i + q * LDJ];
        v[i + p * LDJ] = c * vp - s * vq;
        v[i + q * LDJ] = s * vp + c * vq;
      }
      __syncthreads();
    }
    if (sweep == 0) *first = rotated;
    if (!rotated) return true;
  }
  return false;
}

__device__ __forceinline__ void jacobi_smem(double*& a, double*& v, JacobiScratch*& js, double*& red) {
  extern __shared__ __align__(16) double sm[];
  a = sm;
  v = sm + 64 * LDJ;
  js = reinterpret_cast<JacobiScratch*>(sm + 2 * 64 * LDJ);
  red = reinterpret_cast<double*>(js + 1);
}

// n <= 64: one CTA per matrix, everything in shared memory.  Matrix b: A + b n n (upper triangle read), w + b n, V + b n n.
__global__ void __launch_bounds__(JT) syevj_small_kernel(int n, const double* __restrict__ A, double* __restrict__ w,
                                                         double* __restrict__ V, int* __restrict__ info) {
  double *a, *v, *red;
  JacobiScratch* js;
  jacobi_smem(a, v, js, red);
  __shared__ int rank[64];
  const long long b = blockIdx.x, nn = (long long)n * n;
  A += b * nn; V += b * nn; w += b * n;
  const int np = n + (n & 1), tid = threadIdx.x;
  for (int idx = tid; idx < np * np; idx += JT) {
    const int i = idx % np, j = idx / np;
    a[i + j * LDJ] = (i < n && j < n) ? A[min(i, j) + (long long)max(i, j) * n] : 0.0;
    v[i + j * LDJ] = i == j ? 1.0 : 0.0;
  }
  __syncthreads();
  const double fro = block_fro(np, [&](int i, int j) { return a[i + j * LDJ]; }, red);
  const bool finite = fro <= DBL_MAX;
  bool first = false, conv = false;
  if (finite) conv = jacobi64(a, v, np, SYEVJ_U * fro, js, &first);
  // ascending order by rank counting: rank_i = #{j : w_j < w_i or (w_j = w_i and j < i)}
  if (tid < n) {
    const double wi = a[tid + tid * LDJ];
    int r = 0;
    for (int j = 0; j < n; j++) {
      const double wj = a[j + j * LDJ];
      r += (wj < wi) || (wj == wi && j < tid);
    }
    rank[tid] = r;
    w[rank[tid]] = finite ? wi : NAN;
  }
  __syncthreads();
  for (int idx = tid; idx < n * n; idx += JT) {
    const int i = idx % n, j = idx / n;
    V[i + (long long)rank[j] * n] = finite ? v[i + j * LDJ] : NAN;
  }
  if (tid == 0) info[b] = conv ? 0 : 1;
}

// ---- n > 64: block Jacobi -------------------------------------------------------------------------------------------------------------
// Per matrix b of the chunk: Aw, Vt (Np x Np, ld Np; Vt = V^T, so that V[:, P] <- V[:, P] Q_P is Vt[P, :] <- Q_P^T Vt[P, :]),
// Q (h = N / 2 tiles of 64 x 64, ld 64), quiet[h], floor, state (1 iterating, 0 converged, 2 non-finite input), dirty (some
// subproblem rotated in this sweep).
struct BlockJacobi {
  int n, Np;
  double *Aw, *Vt, *Q, *floor_;
  int *quiet, *state, *dirty, *active;
};

__global__ void __launch_bounds__(JT) syevj_init_kernel(BlockJacobi bj, const double* __restrict__ A) {
  __shared__ double red[JT];
  const long long b = blockIdx.x, nn = (long long)bj.n * bj.n, NN = (long long)bj.Np * bj.Np;
  const int n = bj.n, Np = bj.Np;
  A += b * nn;
  double* Aw = bj.Aw + b * NN;
  double* Vt = bj.Vt + b * NN;
  for (long long idx = threadIdx.x; idx < NN; idx += JT) {
    const int i = (int)(idx % Np), j = (int)(idx / Np);
    Aw[idx] = (i < n && j < n) ? A[min(i, j) + (long long)max(i, j) * n] : 0.0;
    Vt[idx] = i == j ? 1.0 : 0.0;
  }
  const double fro = block_fro(n, [&](int i, int j) { return A[min(i, j) + (long long)max(i, j) * n]; }, red);
  if (threadIdx.x == 0) {
    bj.floor_[b] = SYEVJ_U * fro;
    bj.state[b] = fro <= DBL_MAX ? 1 : 2;
    bj.dirty[b] = 0;
  }
}

// global row of row r of a pair tile whose 32-row halves start at rI and rJ
__device__ __forceinline__ int pair_row(int r, int rI, int rJ) { return r < 32 ? rI + r : rJ + r - 32; }

// Subproblem of pair blockIdx.x: S from the four 32 x 32 quarters of A in place, diagonalised; Q_P, quiet_P, and when something
// rotated, the rotated S back into A (it is this pair's diagonal tile, which no other CTA of the step touches).
__global__ void __launch_bounds__(JT) syevj_pair_kernel(BlockJacobi bj, int step) {
  const long long b = blockIdx.y;
  if (bj.state[b] != 1) return;
  double *a, *v, *red;
  JacobiScratch* js;
  jacobi_smem(a, v, js, red);
  const int Np = bj.Np, N = Np / 32, h = N / 2, k = blockIdx.x;
  int I, J;
  circle_pair(N, step, k, I, J);
  const int rI = 32 * I, rJ = 32 * J;
  double* Aw = bj.Aw + b * Np * Np;
  for (int idx = threadIdx.x; idx < 64 * 64; idx += JT) {
    const int i = idx & 63, j = idx >> 6;
    a[i + j * LDJ] = Aw[pair_row(i, rI, rJ) + (long long)pair_row(j, rI, rJ) * Np];
    v[i + j * LDJ] = i == j ? 1.0 : 0.0;
  }
  __syncthreads();
  bool first = false;
  jacobi64(a, v, 64, bj.floor_[b], js, &first);
  double* Q = bj.Q + (b * h + k) * 4096;
  for (int idx = threadIdx.x; idx < 64 * 64; idx += JT) {
    const int i = idx & 63, j = idx >> 6;
    Q[idx] = v[i + j * LDJ];
    if (first) Aw[pair_row(i, rI, rJ) + (long long)pair_row(j, rI, rJ) * Np] = a[i + j * LDJ];
  }
  if (threadIdx.x == 0) {
    bj.quiet[b * h + k] = !first;
    if (first) bj.dirty[b] = 1;
  }
}

// a 64 x 64 tile whose rows (k) come in two contiguous 32-row halves at rI, rJ and whose columns come in two 32-column halves at cI,
// cJ, into a padded [col][k] tile: tile_load's mapping with the pair gather
__device__ __forceinline__ void pair_tile_load(double* __restrict__ dst, const double* src, long long ld, int rI, int rJ, int cI, int cJ) {
  const int k2 = (threadIdx.x & 31) * 2, c0 = threadIdx.x >> 5, row = pair_row(k2, rI, rJ);
  double2 v[8];
#pragma unroll
  for (int r = 0; r < 8; r++)
    v[r] = __ldcg(reinterpret_cast<const double2*>(src + row + (long long)pair_row(c0 + 8 * r, cI, cJ) * ld));
#pragma unroll
  for (int r = 0; r < 8; r++) *reinterpret_cast<double2*>(dst + (c0 + 8 * r) * TLD + k2) = v[r];
}
// and back: the [col][row] shared tile sC into the scattered halves
__device__ __forceinline__ void pair_tile_store(double* dst, long long ld, const double* sC, int rI, int rJ, int cI, int cJ) {
  const int r2 = (threadIdx.x & 31) * 2, c0 = threadIdx.x >> 5, row = pair_row(r2, rI, rJ);
#pragma unroll
  for (int r = 0; r < 8; r++) {
    const int c = c0 + 8 * r;
    *reinterpret_cast<double2*>(dst + row + (long long)pair_row(c, cI, cJ) * ld) = *reinterpret_cast<const double2*>(sC + c * TLD + r2);
  }
}

// Task blockIdx.x < h (h - 1) / 2: the upper pair tile (P, P2), P < P2: A_PP2 <- Q_P^T A_PP2 Q_P2, written with its mirror A_P2P from
// the same registers (A stays exactly symmetric); skipped when both pairs were quiet (both Q are exactly I).  The other tasks:
// column tile R of Vt and pair P, Vt[P, R] <- Q_P^T Vt[P, R], skipped for a quiet pair.
__global__ void __launch_bounds__(JT, 1) syevj_update_kernel(BlockJacobi bj, int step) {
  const long long b = blockIdx.y;
  if (bj.state[b] != 1) return;
  extern __shared__ __align__(16) double sm[];
  double *s0 = sm, *s1 = sm + TILE_DOUBLES, *s2 = sm + 2 * TILE_DOUBLES, *s3 = sm + 3 * TILE_DOUBLES;
  const int Np = bj.Np, N = Np / 32, h = N / 2, nA = h * (h - 1) / 2;
  const int* quiet = bj.quiet + b * h;
  const double* Q = bj.Q + b * h * 4096;
  double acc[4][2][2];
  int t = blockIdx.x;
  if (t < nA) {
    int P = 0;
    while (t >= h - 1 - P) { t -= h - 1 - P; P++; }
    const int P2 = P + 1 + t;
    if (quiet[P] && quiet[P2]) return;
    int I, J, I2, J2;
    circle_pair(N, step, P, I, J);
    circle_pair(N, step, P2, I2, J2);
    double* Aw = bj.Aw + b * Np * Np;
    tile_load(s0, Q + P * 4096, 64);
    tile_load(s1, Q + P2 * 4096, 64);
    pair_tile_load(s2, Aw, Np, 32 * I, 32 * J, 32 * I2, 32 * J2);
    __syncthreads();
    acc_zero(acc);
    tile_mma(acc, s0, s2);               // T = Q_P^T A_PP2
    acc_to_smem_rowmajor(acc, s3, 1.0);  // s3[i][k] = T(i, k): the B operand of T^T
    __syncthreads();
    acc_zero(acc);
    tile_mma(acc, s1, s3);               // acc(i, j) = (Q_P2^T T^T)(i, j) = A'_P2P(i, j) = A'_PP2(j, i)
    __syncthreads();
    acc_to_smem_colmajor(acc, s0, 1.0);  // [col j][row i] of A'_P2P
    acc_to_smem_rowmajor(acc, s2, 1.0);  // [col i][row j] of A'_PP2
    __syncthreads();
    pair_tile_store(Aw, Np, s0, 32 * I2, 32 * J2, 32 * I, 32 * J);
    pair_tile_store(Aw, Np, s2, 32 * I, 32 * J, 32 * I2, 32 * J2);
  } else {
    t -= nA;
    const int R = t / h, P = t % h;
    if (quiet[P]) return;
    int I, J;
    circle_pair(N, step, P, I, J);
    double* Vt = bj.Vt + b * Np * Np;
    tile_load(s0, Q + P * 4096, 64);
    pair_tile_load(s1, Vt, Np, 32 * I, 32 * J, 64 * R, 64 * R + 32);
    __syncthreads();
    acc_zero(acc);
    tile_mma(acc, s0, s1);
    acc_to_smem_colmajor(acc, s2, 1.0);
    __syncthreads();
    pair_tile_store(Vt, Np, s2, 32 * I, 32 * J, 64 * R, 64 * R + 32);
  }
}

// End of an outer sweep: a matrix none of whose subproblems rotated has converged.  *active = matrices still iterating.
__global__ void __launch_bounds__(1024) syevj_sweep_end_kernel(BlockJacobi bj, int cnt) {
  int c = 0;
  for (int b = threadIdx.x; b < cnt; b += 1024) {
    if (bj.state[b] == 1 && !bj.dirty[b]) bj.state[b] = 0;
    bj.dirty[b] = 0;
    c += bj.state[b] == 1;
  }
  __shared__ int part[1024];
  part[threadIdx.x] = c;
  __syncthreads();
  for (int s = 512; s > 0; s >>= 1) {
    if (threadIdx.x < s) part[threadIdx.x] += part[threadIdx.x + s];
    __syncthreads();
  }
  if (threadIdx.x == 0) *bj.active = part[0];
}

// w = diag(A) over the real indices, sorted by rank counting; V's columns permuted alike; info = 0 converged, 1 otherwise.
__global__ void __launch_bounds__(JT) syevj_finish_kernel(BlockJacobi bj, double* __restrict__ w, double* __restrict__ V,
                                                          int* __restrict__ info) {
  __shared__ double wv[BASECASE_MAX];
  __shared__ int rank[BASECASE_MAX];
  const long long b = blockIdx.x;
  const int n = bj.n, Np = bj.Np;
  const double* Aw = bj.Aw + b * Np * Np;
  const double* Vt = bj.Vt + b * Np * Np;
  w += b * n; V += b * n * n;
  const int state = bj.state[b];
  for (int i = threadIdx.x; i < n; i += JT) wv[i] = Aw[i + (long long)i * Np];
  __syncthreads();
  for (int i = threadIdx.x; i < n; i += JT) {
    const double wi = wv[i];
    int r = 0;
    for (int j = 0; j < n; j++) r += (wv[j] < wi) || (wv[j] == wi && j < i);
    rank[i] = r;
    w[rank[i]] = state == 2 ? NAN : wi;
  }
  __syncthreads();
  for (long long idx = threadIdx.x; idx < (long long)n * n; idx += JT) {
    const int j = (int)(idx % n), r = (int)(idx / n);  // V(r, rank_j) = Vt(j, r): coalesced reads
    V[r + (long long)rank[j] * n] = state == 2 ? NAN : Vt[j + (long long)r * Np];
  }
  if (threadIdx.x == 0) info[b] = state == 0 ? 0 : 1;
}
}  // namespace

#define SYEVJ_LAUNCHED()                   \
  do {                                     \
    ctx->counters.kernel_launches++;       \
    CAP_CUDA(cudaGetLastError());          \
  } while (0)

capital_status_t syevj_init(capital_ctx* ctx) {
  CAP_CUDA(cudaFuncSetAttribute(syevj_small_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, JACOBI_SMEM));
  CAP_CUDA(cudaFuncSetAttribute(syevj_pair_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, JACOBI_SMEM));
  CAP_CUDA(cudaFuncSetAttribute(syevj_update_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, UPDATE_SMEM));
  return CAPITAL_OK;
}

int64_t syevj_chunk(int64_t n, int64_t batch) {
  if (n <= 64) return std::min<int64_t>(batch, 65535);
  const int64_t Np = round_up(n, 64), h = Np / 64;
  return std::min<int64_t>({batch, 65535, (int64_t)(BATCHED_WORKSPACE_CAP / ((2 * Np * Np + h * 4096) * 8))});
}

capital_status_t syevj_batched(capital_ctx* ctx, cudaStream_t st, int64_t n, int64_t batch, const double* A, double* w, double* V, int* info) {
  const int64_t nn = n * n, chunk = syevj_chunk(n, batch);
  if (n <= 64) {
    for (int64_t b0 = 0; b0 < batch; b0 += chunk) {
      const int64_t cnt = std::min(chunk, batch - b0);
      syevj_small_kernel<<<(unsigned)cnt, JT, JACOBI_SMEM, st>>>((int)n, A + b0 * nn, w + b0 * n, V + b0 * nn, info + b0);
      SYEVJ_LAUNCHED();
    }
    return CAPITAL_OK;
  }
  const int64_t Np = round_up(n, 64), N = Np / 32, h = N / 2, NN = Np * Np;
  BlockJacobi bj{(int)n, (int)Np};
  CAP_TRY(ctx->workspace("syevj_A", (size_t)(chunk * NN) * 8, (void**)&bj.Aw));
  CAP_TRY(ctx->workspace("syevj_V", (size_t)(chunk * NN) * 8, (void**)&bj.Vt));
  CAP_TRY(ctx->workspace("syevj_Q", (size_t)(chunk * h * 4096) * 8, (void**)&bj.Q));
  double* fl;
  CAP_TRY(ctx->workspace("syevj_floor", (size_t)chunk * 8, (void**)&fl));
  bj.floor_ = fl;
  int* flags;
  CAP_TRY(ctx->workspace("syevj_flags", (size_t)(chunk * (h + 2) + 1) * sizeof(int), (void**)&flags));
  bj.quiet = flags;
  bj.state = flags + chunk * h;
  bj.dirty = bj.state + chunk;
  bj.active = bj.dirty + chunk;
  const unsigned ntasks = (unsigned)(h * (h - 1) / 2 + (Np / 64) * h);
  for (int64_t b0 = 0; b0 < batch; b0 += chunk) {
    const int64_t cnt = std::min(chunk, batch - b0);
    syevj_init_kernel<<<(unsigned)cnt, JT, 0, st>>>(bj, A + b0 * nn);
    SYEVJ_LAUNCHED();
    for (int sweep = 0; sweep < SYEVJ_SWEEPS; sweep++) {
      for (int step = 0; step < N - 1; step++) {
        syevj_pair_kernel<<<dim3((unsigned)h, (unsigned)cnt), JT, JACOBI_SMEM, st>>>(bj, step);
        SYEVJ_LAUNCHED();
        syevj_update_kernel<<<dim3(ntasks, (unsigned)cnt), JT, UPDATE_SMEM, st>>>(bj, step);
        SYEVJ_LAUNCHED();
      }
      syevj_sweep_end_kernel<<<1, 1024, 0, st>>>(bj, (int)cnt);
      SYEVJ_LAUNCHED();
      int active = 0;  // the one host synchronisation per outer sweep: stop once every matrix of the chunk has converged
      CAP_CUDA(cudaMemcpyAsync(&active, bj.active, sizeof(int), cudaMemcpyDeviceToHost, st));
      CAP_CUDA(cudaStreamSynchronize(st));
      if (active == 0) break;
    }
    syevj_finish_kernel<<<(unsigned)cnt, JT, 0, st>>>(bj, w + b0 * n, V + b0 * nn, info + b0);
    SYEVJ_LAUNCHED();
  }
  return CAPITAL_OK;
}
