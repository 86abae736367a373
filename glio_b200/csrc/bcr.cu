// bcr.cu — the band solve by block cyclic reduction (glio_band_solve_bcr, GLIO_FACTOR_BCR in the device minimizer).
//
// With blocks of b >= hb rows a band matrix is block tridiagonal.  b = 32 * ceil(max(hb, 1) / 32) (bcr_block_size): a multiple
// of the 32 x 32 tiles every kernel below works on, so no tile is partial.  Block i covers rows [i b, (i+1) b); m = ceil(n / b)
// blocks, the rows past n padded with an identity diagonal and a zero right-hand side.  D_i is the diagonal block, E_i the coupling
// A[block i+1, block i], r_i the right-hand side.
//
// The workspace keeps every level in the original block numbering: level l holds the blocks k = 0, s, 2s, ... < m with s = 2^l,
// and "odd" means k / s odd.  Each level eliminates its odd blocks, every one independently:
//   D_k = L L^T                     (k_bcr_potrf, in place in D[k])
//   Ut = E_(k-s)^T L^-T             (U_k^T, k_bcr_trsm, into U[k])
//   Vt = E_k L^-T                   (V_k^T, in place in E[k]; only when block k+s exists)
//   w  = L^-1 r_k                   (in place in r[k])
// and then updates each even block j (k_bcr_update), left neighbour j-s first, right neighbour j+s second:
//   D_j -= Vt_(j-s) Vt_(j-s)^T,  D_j -= Ut_(j+s) Ut_(j+s)^T,  r_j -= Vt_(j-s) w_(j-s),  r_j -= Ut_(j+s) w_(j+s),
//   E_j = -Vt_(j+s) Ut_(j+s)^T     (the new coupling of j and j+2s, when j+2s exists).
// Each original block index is eliminated at exactly one level, so U[k], E[k], D[k] and r[k] of an eliminated block stay for the
// back-substitution.  When one block is left it is factored and solved; then, level by level in reverse (k_bcr_back),
//   x_k = L^-T (w_k - Ut_k^T x_(k-s) - Vt_k^T x_(k+s)).
//
// Summation order (tests/band_bcr_reference.py restates the block order; the dense work inside a block is held to a tolerance):
// every product sum runs over ascending k as a chain of fused multiply-adds into one accumulator, and the accumulator is then
// subtracted once; an even block takes its left neighbour's update before its right neighbour's.  No floating-point atomics and
// no data-dependent scheduling: the result is the same bit for bit from run to run and on every context.
//
// Failure: a pivot that is not positive and finite in any block Cholesky sets flag[0] = 1, and so does a non-finite x
// (k_bcr_finish).  The kernels then run on to the end on whatever values they hold; no control flow depends on a value.
#include "common.cuh"

namespace glio {

namespace {

constexpr int kT = 32;          // tile edge
constexpr int kP = kT + 1;      // padded smem row of a tile: conflict-free column access
constexpr int kThreads = 256;

__device__ __forceinline__ bool bad_pivot(double d) { return !(d > 0.0) || !isfinite(d); }

// Gather D, E and r from the band (entry (i, j), i-hb <= j <= i, at band[i*(hb+1) + (j-i+hb)]).  v != nullptr: the device
// minimizer's shifted matrix, diagonal entry band_ii + v_i * v_i (k_band_shift's rounding).  Reads only slots with j >= 0.
__global__ void k_bcr_gather(const double* __restrict__ band, const double* __restrict__ v, const double* __restrict__ rhs, int n, int hb,
                             int b, int m, double* __restrict__ D, double* __restrict__ E, double* __restrict__ R) {
  const int64_t bb = (int64_t)b * b, nd = (int64_t)m * bb, total = 2 * nd + (int64_t)m * b;
  for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (int64_t)gridDim.x * blockDim.x) {
    if (e < nd) {                                   // D[k][p][q]: rows and columns of block k
      const int64_t k = e / bb; const int p = (int)(e % bb) / b, q = (int)(e % bb) % b;
      const int64_t i = k * b + p, j = k * b + q;
      double val = 0.0;
      if (i >= n) val = p == q ? 1.0 : 0.0;
      else if (q <= p && i - j <= hb) {
        val = band[i * (hb + 1) + (j - i + hb)];
        if (v && p == q) val = __dadd_rn(val, __dmul_rn(v[i], v[i]));
      }
      D[e] = val;
    } else if (e < 2 * nd) {                        // E[k][p][q] = A[(k+1) b + p, k b + q]
      const int64_t f = e - nd, k = f / bb; const int p = (int)(f % bb) / b, q = (int)(f % bb) % b;
      const int64_t i = (k + 1) * b + p, j = k * b + q;
      E[f] = (k + 1 < m && i < n && i - j <= hb) ? band[i * (hb + 1) + (j - i + hb)] : 0.0;
    } else {
      const int64_t i = e - 2 * nd;
      R[i] = i < n ? rhs[i] : 0.0;
    }
  }
}

// One CTA per block k = first + blockIdx.x * step: D[k] = L L^T in place (lower triangle), right-looking over 32-column panels.
// The panel (rows 32J .. b-1 of tile column J) is staged in shared memory: warp 0 factors its diagonal tile, every thread solves
// one row of the tiles below, the panel is written back, and the trailing lower tiles take the panel's product from global memory.
__global__ void __launch_bounds__(kThreads) k_bcr_potrf(double* __restrict__ D, int b, int first, int step, int* __restrict__ flag) {
  extern __shared__ double P[];                     // [b][kP]
  const int k = first + blockIdx.x * step, tid = threadIdx.x, nb = b / kT;
  double* A = D + (size_t)k * b * b;
  for (int J = 0; J < nb; ++J) {
    const int r0 = kT * J, rows = b - r0;
    for (int e = tid; e < rows * kT; e += kThreads) P[(e >> 5) * kP + (e & 31)] = A[(size_t)(r0 + (e >> 5)) * b + r0 + (e & 31)];
    __syncthreads();
    if (tid < kT) {                                 // the diagonal tile, lane = row
      const int lane = tid;
      for (int c = 0; c < kT; ++c) {
        const double d = P[c * kP + c];
        if (lane == 0 && bad_pivot(d)) flag[0] = 1;
        const double l = sqrt(d);
        __syncwarp();
        if (lane > c) P[lane * kP + c] = P[lane * kP + c] / l;
        else if (lane == c) P[c * kP + c] = l;
        __syncwarp();
        if (lane > c) {
          const double lc = P[lane * kP + c];
          for (int u = c + 1; u <= lane; ++u) P[lane * kP + u] = fma(-lc, P[u * kP + c], P[lane * kP + u]);
        }
        __syncwarp();
      }
    }
    __syncthreads();
    if (kT + tid < rows) {                          // the tiles below: y L_JJ^T = a, one row per thread
      double* row = P + (kT + tid) * kP;
      for (int c = 0; c < kT; ++c) {
        double s = 0.0;
        for (int q = 0; q < c; ++q) s = fma(row[q], P[c * kP + q], s);
        row[c] = (row[c] - s) / P[c * kP + c];
      }
    }
    __syncthreads();
    for (int e = tid; e < rows * kT; e += kThreads) A[(size_t)(r0 + (e >> 5)) * b + r0 + (e & 31)] = P[(e >> 5) * kP + (e & 31)];
    // trailing tiles (I, K), J < K <= I < nb: A_IK -= P_I P_K^T.  Each warp covers one row of one tile.
    const int t = nb - J - 1;
    for (int e = tid; e < t * t * kT * kT; e += kThreads) {
      const int tile = e >> 10, I = tile / t, K = tile % t;
      if (K > I) continue;
      const int i = (e >> 5) & 31, kk = e & 31;
      const double* pi = P + (kT * (I + 1) + i) * kP;
      const double* pk = P + (kT * (K + 1) + kk) * kP;
      double s = 0.0;
      for (int c = 0; c < kT; ++c) s = fma(pi[c], pk[c], s);
      double* a = A + (size_t)(r0 + kT * (I + 1) + i) * b + r0 + kT * (K + 1) + kk;
      *a = *a - s;
    }
    __syncthreads();
  }
}

// The row solves y L^T = a of the blocks k = first + (y0 + blockIdx.y) * step.  Rows [0, b): Ut from E[k-s] transposed (when k >= s),
// into U[k]; rows [b, 2b): Vt from E[k] (when k+s < m), in place; row 2b: w from r[k], in place.  blockIdx.x picks 32 rows.
__global__ void __launch_bounds__(kThreads) k_bcr_trsm(const double* __restrict__ D, double* __restrict__ E, double* __restrict__ U,
                                                       double* __restrict__ R, int m, int b, int s, int first, int step, int y0) {
  extern __shared__ double sm[];
  const int k = first + (y0 + (int)blockIdx.y) * step, tid = threadIdx.x, nb = b / kT, c0 = kT * blockIdx.x;
  const int kind = c0 < b ? 0 : c0 < 2 * b ? 1 : 2;
  if ((kind == 0 && k < s) || (kind == 1 && k + s >= m)) return;
  const int YW = b + 1;                             // odd row stride: conflict-free
  double* Y = sm;                                   // [32][YW]
  double* sL = Y + kT * YW;                         // [32][kP]
  const size_t bb = (size_t)b * b;
  const double* L = D + k * bb;
  const int nrows = kind == 2 ? 1 : kT;
  if (kind == 0) {
    const double* Ek = E + (size_t)(k - s) * bb;    // Y[r][q] = E_(k-s)[q][c0 + r]
    for (int e = tid; e < kT * b; e += kThreads) { const int q = e >> 5, r = e & 31; Y[r * YW + q] = Ek[(size_t)q * b + c0 + r]; }
  } else if (kind == 1) {
    const double* Ek = E + k * bb + (size_t)(c0 - b) * b;
    for (int e = tid; e < kT * b; e += kThreads) { const int r = e / b, q = e % b; Y[r * YW + q] = Ek[(size_t)r * b + q]; }
  } else {
    for (int q = tid; q < b; q += kThreads) Y[q] = R[(size_t)k * b + q];
  }
  for (int J = 0; J < nb; ++J) {
    // Y_J -= sum_(K < J) Y_K L_JK^T; thread (ty, tx) owns rows ty + 8 u of column tx
    const int ty = tid >> 5, tx = tid & 31;
    double acc[4] = {0.0, 0.0, 0.0, 0.0};
    for (int K = 0; K < J; ++K) {
      __syncthreads();
      for (int e = tid; e < kT * kT; e += kThreads) sL[(e >> 5) * kP + (e & 31)] = L[(size_t)(kT * J + (e >> 5)) * b + kT * K + (e & 31)];
      __syncthreads();
      for (int u = 0; u < 4; ++u) {
        const double* y = Y + (ty + 8 * u) * YW + kT * K;
        for (int q = 0; q < kT; ++q) acc[u] = fma(y[q], sL[tx * kP + q], acc[u]);
      }
    }
    __syncthreads();
    for (int u = 0; u < 4; ++u) { double& y = Y[(ty + 8 * u) * YW + kT * J + tx]; y = y - acc[u]; }
    for (int e = tid; e < kT * kT; e += kThreads) sL[(e >> 5) * kP + (e & 31)] = L[(size_t)(kT * J + (e >> 5)) * b + kT * J + (e & 31)];
    __syncthreads();
    if (tid < nrows) {                              // the diagonal tile, one row per thread
      double* y = Y + tid * YW + kT * J;
      for (int c = 0; c < kT; ++c) {
        double sum = 0.0;
        for (int q = 0; q < c; ++q) sum = fma(y[q], sL[c * kP + q], sum);
        y[c] = (y[c] - sum) / sL[c * kP + c];
      }
    }
  }
  __syncthreads();
  if (kind == 2) {
    for (int q = tid; q < b; q += kThreads) R[(size_t)k * b + q] = Y[q];
  } else {
    double* out = kind == 0 ? U + k * bb + (size_t)c0 * b : E + k * bb + (size_t)(c0 - b) * b;
    for (int e = tid; e < kT * b; e += kThreads) { const int r = e / b, q = e % b; out[(size_t)r * b + q] = Y[r * YW + q]; }
  }
}

// acc[u] = sum_q X[32 I + ty + 8u][q] Y[32 K + tx][q], q ascending; X and Y are b x b row-major
__device__ __forceinline__ void tile_xyt(const double* __restrict__ X, const double* __restrict__ Yb, int b, int I, int K, double* sX,
                                         double* sY, double acc[4]) {
  const int tid = threadIdx.x, ty = tid >> 5, tx = tid & 31;
  for (int u = 0; u < 4; ++u) acc[u] = 0.0;
  for (int q0 = 0; q0 < b; q0 += kT) {
    __syncthreads();
    for (int e = tid; e < kT * kT; e += kThreads) {
      const int r = e >> 5, c = e & 31;
      sX[r * kP + c] = X[(size_t)(kT * I + r) * b + q0 + c];
      sY[r * kP + c] = Yb[(size_t)(kT * K + r) * b + q0 + c];
    }
    __syncthreads();
    for (int u = 0; u < 4; ++u) {
      const double* x = sX + (ty + 8 * u) * kP;
      for (int q = 0; q < kT; ++q) acc[u] = fma(x[q], sY[tx * kP + q], acc[u]);
    }
  }
}

// The even blocks j = (y0 + blockIdx.y) * 2s of one level.  blockIdx.x: the lower tiles of D_j, then the tiles of the new E_j, then the
// 32-row tiles of r_j.
__global__ void __launch_bounds__(kThreads) k_bcr_update(double* __restrict__ D, double* __restrict__ E, const double* __restrict__ U,
                                                         double* __restrict__ R, int m, int b, int s, int y0) {
  __shared__ double sX[kT * kP], sY[kT * kP];
  const int j = (y0 + (int)blockIdx.y) * 2 * s, nb = b / kT, nd = nb * (nb + 1) / 2, tid = threadIdx.x, ty = tid >> 5, tx = tid & 31;
  const int lft = j >= s ? j - s : -1, rgt = j + s < m ? j + s : -1;
  const size_t bb = (size_t)b * b;
  int t = blockIdx.x;
  double acc[4];
  if (t < nd) {                                     // D tile (I, K), K <= I
    int I = 0;
    while (t > I) { t -= I + 1; ++I; }
    const int K = t;
    double* out = D + j * bb + (size_t)(kT * I) * b + kT * K;
    double o[4];
    for (int u = 0; u < 4; ++u) o[u] = out[(size_t)(ty + 8 * u) * b + tx];
    if (lft >= 0) {
      tile_xyt(E + lft * bb, E + lft * bb, b, I, K, sX, sY, acc);
      for (int u = 0; u < 4; ++u) o[u] = o[u] - acc[u];
    }
    if (rgt >= 0) {
      tile_xyt(U + rgt * bb, U + rgt * bb, b, I, K, sX, sY, acc);
      for (int u = 0; u < 4; ++u) o[u] = o[u] - acc[u];
    }
    for (int u = 0; u < 4; ++u) out[(size_t)(ty + 8 * u) * b + tx] = o[u];
    return;
  }
  t -= nd;
  if (t < nb * nb) {                                // E tile (I, K) of the coupling j -> j + 2s
    if (j + 2 * s >= m) return;
    const int I = t / nb, K = t % nb;
    tile_xyt(E + rgt * bb, U + rgt * bb, b, I, K, sX, sY, acc);
    double* out = E + j * bb + (size_t)(kT * I) * b + kT * K;
    for (int u = 0; u < 4; ++u) out[(size_t)(ty + 8 * u) * b + tx] = -acc[u];
    return;
  }
  t -= nb * nb;                                     // r rows 32 t .. 32 t + 31, one per thread of warp 0
  if (tid >= kT) return;
  const int p = kT * t + tid;
  double o = R[(size_t)j * b + p];
  if (lft >= 0) {
    const double* x = E + lft * bb + (size_t)p * b; const double* w = R + (size_t)lft * b;
    double a = 0.0;
    for (int q = 0; q < b; ++q) a = fma(x[q], w[q], a);
    o = o - a;
  }
  if (rgt >= 0) {
    const double* x = U + rgt * bb + (size_t)p * b; const double* w = R + (size_t)rgt * b;
    double a = 0.0;
    for (int q = 0; q < b; ++q) a = fma(x[q], w[q], a);
    o = o - a;
  }
  R[(size_t)j * b + p] = o;
}

// x_k = L^-T (w_k - Ut_k^T x_(k-s) - Vt_k^T x_(k+s)) for k = first + blockIdx.x * step: the neighbour products one column per
// thread, then the backward solve over tiles, last first (warp 0 solves the diagonal tile, the block updates the rows above).
__global__ void __launch_bounds__(kThreads) k_bcr_back(const double* __restrict__ D, const double* __restrict__ E, const double* __restrict__ U,
                                                       const double* __restrict__ R, double* __restrict__ X, int m, int b, int s, int first, int step) {
  __shared__ double t[kThreads], sL[kT * kP];
  const int k = first + blockIdx.x * step, tid = threadIdx.x, nb = b / kT;
  const int lft = k >= s ? k - s : -1, rgt = k + s < m ? k + s : -1;
  const size_t bb = (size_t)b * b;
  const double* L = D + k * bb;
  if (tid < b) {
    double o = R[(size_t)k * b + tid];
    if (lft >= 0) {
      const double* ut = U + k * bb; const double* x = X + (size_t)lft * b;
      double a = 0.0;
      for (int p = 0; p < b; ++p) a = fma(ut[(size_t)p * b + tid], x[p], a);
      o = o - a;
    }
    if (rgt >= 0) {
      const double* vt = E + k * bb; const double* x = X + (size_t)rgt * b;
      double a = 0.0;
      for (int p = 0; p < b; ++p) a = fma(vt[(size_t)p * b + tid], x[p], a);
      o = o - a;
    }
    t[tid] = o;
  }
  for (int J = nb - 1; J >= 0; --J) {
    __syncthreads();
    for (int e = tid; e < kT * kT; e += kThreads) sL[(e >> 5) * kP + (e & 31)] = L[(size_t)(kT * J + (e >> 5)) * b + kT * J + (e & 31)];
    __syncthreads();
    if (tid < kT) {                                 // L_JJ^T x_J = t_J, lane = row
      double tv = t[kT * J + tid];
      for (int q = kT - 1; q >= 0; --q) {
        if (tid == q) tv = tv / sL[q * kP + q];
        const double xq = __shfl_sync(0xffffffffu, tv, q);
        if (tid < q) tv = fma(-sL[q * kP + tid], xq, tv);
      }
      t[kT * J + tid] = tv;
    }
    __syncthreads();
    if (tid < kT * J) {                             // t_p -= sum_c L[32J + c][p] x_(32J + c)
      double a = 0.0;
      for (int c = 0; c < kT; ++c) a = fma(L[(size_t)(kT * J + c) * b + tid], t[kT * J + c], a);
      t[tid] = t[tid] - a;
    }
  }
  __syncthreads();
  if (tid < b) X[(size_t)k * b + tid] = t[tid];
}

// x[i] = X[i] for i < n; a non-finite entry sets flag[0]
__global__ void k_bcr_finish(const double* __restrict__ X, double* __restrict__ x, int n, int* __restrict__ flag) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const double v = X[i];
  x[i] = v;
  if (!isfinite(v)) flag[0] = 1;
}

// gridDim.y is at most 65 535: launches over more blocks than that go in chunks, each told its first y (one launch below the limit)
constexpr int kMaxGridY = 65535;

size_t potrf_smem(int b) { return (size_t)b * kP * sizeof(double); }
size_t trsm_smem(int b) { return ((size_t)kT * (b + 1) + kT * kP) * sizeof(double); }

}  // namespace

int bcr_block_size(int hb) { return kT * ((std::max(hb, 1) + kT - 1) / kT); }

void BcrWork::reserve(int n, int hb) {
  const size_t b = (size_t)bcr_block_size(hb), m = ((size_t)n + b - 1) / b;
  D.reserve(m * b * b); E.reserve(m * b * b); U.reserve(m * b * b); R.reserve(m * b); X.reserve(m * b); flag.reserve(1);
}

void bcr_solve_run(BcrWork& w, const double* d_band, const double* d_v, const double* d_b, double* d_x, int n, int hb, cudaStream_t st,
                   LaunchCounter& lc) {
  const int b = bcr_block_size(hb), m = (n + b - 1) / b, nb = b / kT;
  w.reserve(n, hb);
  GLIO_CUDA_TRY(cudaFuncSetAttribute(k_bcr_potrf, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)potrf_smem(b)));
  GLIO_CUDA_TRY(cudaFuncSetAttribute(k_bcr_trsm, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)trsm_smem(b)));
  GLIO_CUDA_TRY(cudaMemsetAsync(w.flag.p, 0, sizeof(int), st));
  const int64_t total = 2 * (int64_t)m * b * b + (int64_t)m * b;
  lc.begin("k_bcr_gather", st);
  k_bcr_gather<<<(unsigned)std::min<int64_t>((total + 255) / 256, 64 * kNumSMs), 256, 0, st>>>(d_band, d_v, d_b, n, hb, b, m, w.D.p, w.E.p, w.R.p);
  lc.end(st);
  auto eliminate = [&](int s, int first, int step, int count) {
    lc.begin("k_bcr_potrf", st);
    k_bcr_potrf<<<count, kThreads, potrf_smem(b), st>>>(w.D.p, b, first, step, w.flag.p);
    lc.end(st);
    for (int y0 = 0; y0 < count; y0 += kMaxGridY) {
      lc.begin("k_bcr_trsm", st);
      k_bcr_trsm<<<dim3(2 * nb + 1, std::min(count - y0, kMaxGridY)), kThreads, trsm_smem(b), st>>>(w.D.p, w.E.p, w.U.p, w.R.p, m, b, s,
                                                                                                   first, step, y0);
      lc.end(st);
    }
  };
  int s = 1;
  for (; s < m; s *= 2) {                           // level with blocks 0, s, 2s, ... < m: at least two
    const int ml = (m + s - 1) / s;
    eliminate(s, s, 2 * s, ml / 2);
    const int even = (ml + 1) / 2;
    for (int y0 = 0; y0 < even; y0 += kMaxGridY) {
      lc.begin("k_bcr_update", st);
      k_bcr_update<<<dim3(nb * (nb + 1) / 2 + nb * nb + nb, std::min(even - y0, kMaxGridY)), kThreads, 0, st>>>(w.D.p, w.E.p, w.U.p, w.R.p,
                                                                                                             m, b, s, y0);
      lc.end(st);
    }
  }
  eliminate(s, 0, 1, 1);                            // the one block left: k = 0, s >= m, no neighbours
  for (; s >= 1; s /= 2) {
    const int ml = (m + s - 1) / s;
    const bool top = s >= m;
    lc.begin("k_bcr_back", st);
    k_bcr_back<<<top ? 1 : ml / 2, kThreads, 0, st>>>(w.D.p, w.E.p, w.U.p, w.R.p, w.X.p, m, b, s, top ? 0 : s, 2 * s);
    lc.end(st);
  }
  lc.begin("k_bcr_finish", st);
  k_bcr_finish<<<(n + 255) / 256, 256, 0, st>>>(w.X.p, d_x, n, w.flag.p);
  lc.end(st);
  GLIO_CUDA_TRY(cudaGetLastError());
}

}  // namespace glio
