// band.cu — K4: the band Cholesky factor-and-solve of the normal equations on the device.
//
// Band layout (BandMat, glio_host_factors_band_fn): entry (i, j), i - hb <= j <= i, at a[i*(hb+1) + (j - i + hb)].
//
// k_band_chol_solve factors A = L L^T in place and solves L L^T x = b with ONE thread block, which keeps a sliding window of
// the band's rows in shared memory.  The factorisation is right-looking, in the operation order of detail::cholesky_solve_scalar
// (solver.cpp), so L and the forward half are bit-identical to the scalar host path:
//   column j:  l = sqrt(a_jj), linv = 1.0 / l (one division per column), L_(j+t, j) = a_(j+t, j) * linv,
//              a_(j+t, j+1+u) = a_(j+t, j+1+u) - L_(j+t, j) * L_(j+1+u, j) for 0 <= u < t <= min(hb, n-1-j),
//   so every entry receives its updates in ascending column order, each as one rounded product and one rounded difference
//   (this file is built with -fmad=false: no contraction).  The forward substitution is fused column by column into the sweep:
//   y_j = s_j / l, then s_(j+t) = s_(j+t) - L_(j+t, j) * y_j, which is the scalar forward solve's order (s_i = b_i minus its
//   terms in ascending column order).
// The backward substitution is in axpy form, descending rows: x_i = s_i / L_ii, then s_k = s_k - L_(i, k) * x_i for
// k = i-1 down to i-hb, with s starting at y.  Its sums therefore run in descending row order, where the host's dot form runs in
// ascending order: x differs from the host's by rounding.  tests/band_solve_reference.py restates exactly this order.
//
// Failure (the host's `false`, which drives the dogleg's mu escalation): a pivot that is not positive or not finite stops the
// sweep; a non-finite x is reported after the backward pass.  On failure the band and x hold partial results.
//
// Rows reach shared memory by cp.async kBandPrefetch steps before the sweep needs them, so the loads stay off the column
// chain.  The n column steps are one dependent chain of sqrt and divide on one SM: that is the price of the host's order.
#include <cuda_pipeline.h>

#include "common.cuh"

namespace glio {

namespace {

constexpr int kBandThreads = 512;
constexpr int kBandPrefetch = 8;   // steps between a row's load and its first use

struct BandSmem {
  int R, W;            // ring rows (hb + 1 + kBandPrefetch), row width (hb + 1)
  double* win;         // [R][W]: the band rows of the window, row r in slot r % R
  double* s;           // [R]: right-hand side of row r in slot r % R (forward: b -> y; backward: y -> x)
  double* col;         // [W]: the scaled column of the current step, col[t] = L_(j+t, j)
};

__device__ __forceinline__ void load_row_async(const BandSmem& m, const double* __restrict__ band, const double* __restrict__ rhs,
                                               int64_t r) {
  const int slot = (int)(r % m.R);
  double* dst = m.win + (size_t)slot * m.W;
  const double* src = band + (size_t)r * m.W;
  for (int e = threadIdx.x; e < m.W; e += blockDim.x) __pipeline_memcpy_async(dst + e, src + e, sizeof(double));
  if (rhs && threadIdx.x == 0) __pipeline_memcpy_async(m.s + slot, rhs + r, sizeof(double));
}

__device__ __forceinline__ bool bad_pivot(double d) { return !(d > 0.0) || !isfinite(d); }

// One block.  band[n*(hb+1)]: in A, out L.  b[n] in.  x[n] out (y after the forward half, then x).  flag[0] = 1 on success.
__global__ void __launch_bounds__(kBandThreads) k_band_chol_solve(double* __restrict__ band, const double* __restrict__ b,
                                                                   double* __restrict__ x, int n, int hb, int* __restrict__ flag) {
  extern __shared__ double smem[];
  BandSmem m;
  m.W = hb + 1; m.R = hb + 1 + kBandPrefetch;
  m.win = smem; m.s = m.win + (size_t)m.R * m.W; m.col = m.s + m.R;
  const int tid = threadIdx.x;

  // ---- factorisation with the fused forward substitution
  for (int r = 0; r < m.R - 1 && r < n; ++r) load_row_async(m, band, b, r);
  __pipeline_commit();
  for (int k = 0; k < kBandPrefetch - 1; ++k) __pipeline_commit();   // empty groups: the wait below then always covers the rows due
  bool ok = true;
  for (int j = 0; j < n; ++j) {
    __pipeline_wait_prior(kBandPrefetch - 1);   // rows up to j + hb are here (issued at step j - kBandPrefetch or before)
    __syncthreads();
    double* rowj = m.win + (size_t)(j % m.R) * m.W;
    const double d = rowj[hb];
    if (bad_pivot(d)) { ok = false; break; }    // every thread reads the same d: a uniform exit
    const double l = __dsqrt_rn(d);
    const double linv = 1.0 / l;
    const double yj = m.s[j % m.R] / l;
    const int mm = min(hb, n - 1 - j);
    if (tid == 0) x[j] = yj;
    // phase A: scale column j and carry y_j into the rows below
    for (int t = 1 + tid; t <= mm; t += blockDim.x) {
      double* e = m.win + (size_t)((j + t) % m.R) * m.W + (hb - t);   // (j+t, j)
      const double v = __dmul_rn(*e, linv);
      *e = v; m.col[t] = v;
      double& st = m.s[(j + t) % m.R];
      st = __dsub_rn(st, __dmul_rn(v, yj));
    }
    __syncthreads();
    // phase B: the rank-1 update of the trailing triangle, (t, u) with 0 <= u < t <= mm, folded into a ceil(mm/2) x (mm+1)
    // rectangle (row pair t = r + 1 and t = mm - r) so the threads stay busy
    const int cols = mm + 1, rows = (mm + 1) / 2;
    for (int e = tid; e < rows * cols; e += blockDim.x) {
      const int r = e / cols, c = e - r * cols;
      int t, u;
      if (c <= r) { t = r + 1; u = c; }
      else { t = mm - r; u = c - (r + 1); if (t == r + 1) continue; }
      double* a = m.win + (size_t)((j + t) % m.R) * m.W + (hb + 1 + u - t);   // (j+t, j+1+u)
      *a = __dsub_rn(*a, __dmul_rn(m.col[t], m.col[1 + u]));
    }
    // row j is final (its diagonal is l): write it back.  Row j-1's slot was written back a step ago: load row j-1+R into it.
    for (int e = tid; e < m.W; e += blockDim.x) band[(size_t)j * m.W + e] = e == hb ? l : rowj[e];
    if (j - 1 + m.R < n) load_row_async(m, band, b, (int64_t)j - 1 + m.R);   // j = 0: slot R-1, still unused
    __pipeline_commit();
  }
  __pipeline_wait_prior(0);
  __syncthreads();
  if (!ok) { if (tid == 0) flag[0] = 0; return; }

  // ---- backward substitution, axpy form, descending rows.  Step i needs L row i (slot i % R) and s_k for k in [i-hb, i]
  // (slot k % R); both are loaded kBandPrefetch steps ahead: row i-P and y_(i-P-hb).
  auto issue = [&](int i) {
    if (i >= 0) load_row_async(m, band, nullptr, i);
    const int k = i - hb;
    if (k >= 0 && tid == 0) __pipeline_memcpy_async(m.s + (k % m.R), x + k, sizeof(double));
  };
  // the first P steps' rows and y values; y_k with k > n-1-hb is first needed at step n-1 as well
  for (int k = n - 1; k >= 0 && k > n - 1 - hb; --k) if (tid == 0) __pipeline_memcpy_async(m.s + (k % m.R), x + k, sizeof(double));
  for (int i = n - 1; i > n - 1 - kBandPrefetch && i >= 0; --i) issue(i);
  __pipeline_commit();
  for (int k = 0; k < kBandPrefetch - 1; ++k) __pipeline_commit();
  bool finite = true;
  for (int i = n - 1; i >= 0; --i) {
    __pipeline_wait_prior(kBandPrefetch - 1);
    __syncthreads();
    const double* rowi = m.win + (size_t)(i % m.R) * m.W;
    const double xi = m.s[i % m.R] / rowi[hb];
    if (tid == 0) { x[i] = xi; finite = finite && isfinite(xi); }
    const int mm = min(hb, i);
    for (int t = 1 + tid; t <= mm; t += blockDim.x) {
      double& sk = m.s[(i - t) % m.R];
      sk = __dsub_rn(sk, __dmul_rn(rowi[hb - t], xi));
    }
    issue(i - kBandPrefetch);
    __pipeline_commit();
  }
  __pipeline_wait_prior(0);
  if (tid == 0) flag[0] = finite ? 1 : 0;
}

// K4 assembly: one thread per entry (p, q) of a planned nt x nt block (ka, kb), ka >= kb (q <= p on the diagonal).  The entry
// already holds the host callback's value (or 0); its contributions are added in plan order, which is the host path's order
// (K x 28 diagonal blocks, off-diagonal 6-column blocks in `off` order, IMU diagonal blocks, IMU pair blocks).
__global__ void k_band_assemble(double* __restrict__ H, int hb, int nt, const BandBlock* __restrict__ blocks, int n_blocks,
                                const BandContrib* __restrict__ contrib, const double* __restrict__ diag6, const double* __restrict__ off6,
                                const double* __restrict__ imu_diag, const double* __restrict__ imu_off) {
  const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int per = nt * nt;
  if (e >= (int64_t)n_blocks * per) return;
  const BandBlock bk = blocks[e / per];
  const int p = (int)(e % per) / nt, q = (int)(e % per) % nt;
  if (bk.ka == bk.kb && q > p) return;
  const int64_t i = (int64_t)nt * bk.ka + p, j = (int64_t)nt * bk.kb + q;
  double* h = H + i * (hb + 1) + (j - i + hb);
  double v = *h;
  const bool six = p < 6 && q < 6;
  for (int c = bk.c0; c < bk.c1; ++c) {
    const BandContrib cb = contrib[c];
    switch (cb.kind) {
      case BAND_DIAG6: if (six) v = __dadd_rn(v, diag6[(size_t)cb.idx * GLIO_NACC + (q * (13 - q)) / 2 + (p - q)]); break;
      case BAND_OFF6: if (six) v = __dadd_rn(v, off6[(size_t)cb.idx * 36 + 6 * p + q]); break;
      case BAND_OFF6_T: if (six) v = __dadd_rn(v, off6[(size_t)cb.idx * 36 + 6 * q + p]); break;
      case BAND_IMU_DIAG: v = __dadd_rn(v, imu_diag[(size_t)cb.idx * GLIO_NACC_IMU_KF + 15 * p + q]); break;
      default: v = __dadd_rn(v, imu_off[(size_t)cb.idx * 225 + 15 * q + p]); break;   // BAND_IMU_OFF_T
    }
  }
  *h = v;
}

// g entry i = nt k + p: the callback's value (or 0), then the keyframe's 6-column g, then its IMU g (the host path's order)
__global__ void k_band_assemble_g(double* __restrict__ g, int n, int nt, const double* __restrict__ diag6, const double* __restrict__ imu_diag) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int k = i / nt, p = i % nt;
  double v = g[i];
  if (p < 6) v = __dadd_rn(v, diag6[(size_t)k * GLIO_NACC + 21 + p]);
  if (imu_diag) v = __dadd_rn(v, imu_diag[(size_t)k * GLIO_NACC_IMU_KF + 225 + p]);
  g[i] = v;
}

// Hs = S H S (each entry (H_ij * s_i) * s_j, the host's order) and diag(Hs)
__global__ void k_band_scale(const double* __restrict__ H, double* __restrict__ Hs, const double* __restrict__ s, int n, int hb,
                             double* __restrict__ hs_diag) {
  const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= (int64_t)n * (hb + 1)) return;
  const int64_t i = e / (hb + 1), j = i - hb + e % (hb + 1);
  if (j < 0) return;
  const double v = __dmul_rn(__dmul_rn(H[e], s[i]), s[j]);
  Hs[e] = v;
  if (j == i) hs_diag[i] = v;
}

// A = Hs + diag(v * v)
__global__ void k_band_shift(const double* __restrict__ Hs, double* __restrict__ A, const double* __restrict__ v, int n, int hb) {
  const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= (int64_t)n * (hb + 1)) return;
  const int64_t i = e / (hb + 1), k = e % (hb + 1);
  A[e] = k == hb ? __dadd_rn(Hs[e], __dmul_rn(v[i], v[i])) : Hs[e];
}

// y = Hs x for the symmetric band: one thread per row, columns ascending, each term one rounded product and one rounded sum
__global__ void k_band_symv(const double* __restrict__ Hs, const double* __restrict__ x, double* __restrict__ y, int n, int hb) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const size_t w = (size_t)hb + 1;
  double s = 0.0;
  for (int j = max(0, i - hb); j <= i; ++j) s = __dadd_rn(s, __dmul_rn(Hs[(size_t)i * w + (j - i + hb)], x[j]));
  for (int j = i + 1; j <= min(n - 1, i + hb); ++j) s = __dadd_rn(s, __dmul_rn(Hs[(size_t)j * w + (i - j + hb)], x[j]));
  y[i] = s;
}

}  // namespace

void band_assemble_run(double* d_H, int hb, int nt, const BandBlock* d_blocks, int n_blocks, const BandContrib* d_contrib,
                       const double* d_diag6, const double* d_off6, const double* d_imu_diag, const double* d_imu_off, double* d_g, int n,
                       cudaStream_t st, LaunchCounter& lc) {
  const int64_t work = (int64_t)n_blocks * nt * nt;
  lc.begin("k_band_assemble", st);
  k_band_assemble<<<(unsigned)((work + 255) / 256), 256, 0, st>>>(d_H, hb, nt, d_blocks, n_blocks, d_contrib, d_diag6, d_off6, d_imu_diag, d_imu_off);
  lc.end(st);
  lc.begin("k_band_assemble_g", st);
  k_band_assemble_g<<<(n + 255) / 256, 256, 0, st>>>(d_g, n, nt, d_diag6, d_imu_diag);
  lc.end(st);
}

void band_scale_run(const double* d_H, double* d_Hs, const double* d_s, int n, int hb, double* d_hs_diag, cudaStream_t st, LaunchCounter& lc) {
  const int64_t work = (int64_t)n * (hb + 1);
  lc.begin("k_band_scale", st);
  k_band_scale<<<(unsigned)((work + 255) / 256), 256, 0, st>>>(d_H, d_Hs, d_s, n, hb, d_hs_diag);
  lc.end(st);
}

void band_shift_run(const double* d_Hs, double* d_A, const double* d_v, int n, int hb, cudaStream_t st, LaunchCounter& lc) {
  const int64_t work = (int64_t)n * (hb + 1);
  lc.begin("k_band_shift", st);
  k_band_shift<<<(unsigned)((work + 255) / 256), 256, 0, st>>>(d_Hs, d_A, d_v, n, hb);
  lc.end(st);
}

void band_symv_run(const double* d_Hs, const double* d_x, double* d_y, int n, int hb, cudaStream_t st, LaunchCounter& lc) {
  lc.begin("k_band_symv", st);
  k_band_symv<<<(n + 127) / 128, 128, 0, st>>>(d_Hs, d_x, d_y, n, hb);
  lc.end(st);
}

size_t band_chol_smem_bytes(int hb) {
  const size_t W = (size_t)hb + 1, R = W + kBandPrefetch;
  return (R * W + R + W) * sizeof(double);
}

void band_chol_solve_run(double* d_band, const double* d_b, double* d_x, int n, int hb, int* d_flag, cudaStream_t st, LaunchCounter& lc) {
  const size_t smem = band_chol_smem_bytes(hb);
  GLIO_CUDA_TRY(cudaFuncSetAttribute(k_band_chol_solve, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  lc.begin("k_band_chol_solve", st);
  k_band_chol_solve<<<1, kBandThreads, smem, st>>>(d_band, d_b, d_x, n, hb, d_flag);
  lc.end(st);
  GLIO_CUDA_TRY(cudaGetLastError());
}

}  // namespace glio
