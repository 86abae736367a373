// loop.cu — loop-closure registration (SURVEY 8 f-7): pcl::IterativeClosestPoint<PointXYZI, PointXYZI> as the Estimator's
// performLoopClosure configures it (GLIO/src/Estimator.cpp:5183-5273), restated from PCL 1.8's registration/impl/icp.hpp,
// transformation_estimation_svd.hpp (pcl::umeyama), correspondence_estimation.hpp and default_convergence_criteria.hpp, plus
// getFitnessScore (registration/impl/registration.hpp) and the host pose arithmetic of the accepted loop.
//
// One registration = set-up (pack the source, K0 grid of the target, cell order of the source) + up to max_iterations ICP
// iterations + one fitness pass.  The ICP state lives on the device (IcpState); iterations are launched in batches of
// 8, 16, 32, 32, ... and a `done` flag set by the one-thread kernels makes every later kernel of the batch return at once, so
// the host synchronises once per batch (plus once inside the grid build and once for the result): 3 host synchronisations for a
// registration that converges within 8 iterations.
//
// Kernels (glio_profile_get names), per iteration:
//   k_lc_nn        exact 1-NN of every source point on the K0 grid: (distance, index) key, FLANN L2_Simple<float> distances,
//                  ties by index; box growth face by face until the best distance is proven, or the box covers the gate (the
//                  correspondence distance) or the whole grid (the fitness pass has no gate); queries in cell order
//   k_scan_block / k_scan_add   exclusive scan of the correspondence flags (grid.cu)
//   k_lc_compact   correspondences in source order: (query, match, float squared distance)
//   k_lc_sum0 / k_lc_sum1       deterministic sums, see "Summation order" below
//   k_lc_means     correspondence count test (< 3: NO_CORRESPONDENCES), the two means, the MSE
//   k_lc_solve     sigma, Eigen 3.3 JacobiSVD<Matrix3f>, R, t, final = transformation * final, convergence test
//   k_lc_transform the in-place transform of the source cloud by this iteration's transformation (PCL's order)
// set-up k_lc_load, k_lc_qhist, k_lc_qscatter, k_lc_init (+ the K0 kernels of grid.cu); fitness pass k_lc_final, k_lc_nn,
// k_lc_sum0, k_lc_sum1, k_lc_fitness.
//
// Summation order (fixed, so that a sequential restatement reproduces every bit): the terms of a sum are taken in list order (the compacted
// correspondence list, or the source order for the fitness); level 0 sums runs of LC_RUN = 64 consecutive terms, level 1 sums
// runs of 64 consecutive level-0 results, and the result is the sum of the level-1 results in order; every run is a
// left-to-right sum that starts from zero.  Float sums: the six coordinate sums of the two means and the nine entries of
// dst_demean * src_demean^T; double sums: the MSE and the fitness.  Eigen's packet reductions and GEMM use another order
// (DESIGN 2: unpinned).
//
// Compiled with -fmad=false: every float / double operation rounds as written (baseline x86-64, no FMA contraction).
#include <cfloat>

#include "common.cuh"
#include "devmath.cuh"
#include "hostmath.h"
#include "knn_common.cuh"

namespace glio {

constexpr int LC_RUN = 64;
constexpr int LC_T = 128;

// ---------------------------------------------------------------------------------------------------------------------
// set-up
// ---------------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_lc_load(const float* __restrict__ xyz, int stride, int64_t n, float4* __restrict__ a,
                                                 float4* __restrict__ b) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const float4 p = make_float4(xyz[i * stride], xyz[i * stride + 1], xyz[i * stride + 2], 0.f);
    a[i] = p; b[i] = p;
  }
}

__global__ void __launch_bounds__(256) k_lc_qhist(GridDesc g, const float4* __restrict__ pts, int64_t n, int* __restrict__ count) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const float4 p = pts[i];
    atomicAdd(&count[cell_of_clamped(g, p.x, p.y, p.z)], 1);
  }
}

__global__ void __launch_bounds__(256) k_lc_qscatter(GridDesc g, const float4* __restrict__ pts, int64_t n, const int* __restrict__ start,
                                                     int* __restrict__ fill, int* __restrict__ perm) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const float4 p = pts[i];
    const int c = cell_of_clamped(g, p.x, p.y, p.z);
    perm[start[c] + atomicAdd(&fill[c], 1)] = (int)i;   // the order inside a cell only affects speed, never a result
  }
}

__global__ void k_lc_init(IcpState* s) {
  if (threadIdx.x != 0) return;
  IcpState z;
  memset(&z, 0, sizeof(z));
  for (int k = 0; k < 16; ++k) { z.transformation[k] = (k % 5 == 0) ? 1.f : 0.f; z.final_T[k] = z.transformation[k]; }
  z.prev_mse = DBL_MAX;
  z.fitness = DBL_MAX;
  *s = z;
}

// ---------------------------------------------------------------------------------------------------------------------
// exact 1-NN on the K0 grid
// ---------------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ void nn_range(const float4* __restrict__ pts, int s, int e, float qx, float qy, float qz, unsigned long long& best, float& bd) {
  for (int k = s; k < e; ++k) {
    const float4 p = __ldg(&pts[k]);
    const float d = l2_simple(qx, qy, qz, p.x, p.y, p.z);
    if (d <= bd) {
      const unsigned long long key = make_key(d, __float_as_int(p.w));
      if (key < best) { best = key; bd = d; }
    }
  }
}

__device__ __forceinline__ void nn_rows(const GridDesc& g, int x0, int x1, int y0, int y1, int z0, int z1, float qx, float qy, float qz,
                                        unsigned long long& best, float& bd) {
  x0 = max(x0, 0); x1 = min(x1, g.nx - 1); y0 = max(y0, 0); y1 = min(y1, g.ny - 1); z0 = max(z0, 0); z1 = min(z1, g.nz - 1);
  if (x0 > x1) return;
  const int* __restrict__ cs = g.cell_start;
  for (int z = z0; z <= z1; ++z)
    for (int y = y0; y <= y1; ++y) {
      const int row = (z * g.ny + y) * g.nx;
      nn_range(g.pts, __ldg(&cs[row + x0]), __ldg(&cs[row + x1 + 1]), qx, qy, qz, best, bd);
    }
}

// can a point nearer than the current best (or, with no best yet, within the gate) hide beyond face f of the searched box?
// Faces at the grid border hide nothing; the margins are those of the K1 box search (box_face_open).
__device__ __forceinline__ bool nn_face_open(const GridDesc& g, int f, float qx, float qy, float qz, float gate_r, const int (&lo)[3],
                                             const int (&hi)[3], float bd) {
  const int ax = f >> 1;
  const bool up = (f & 1) != 0;
  const int n = ax == 0 ? g.nx : (ax == 1 ? g.ny : g.nz);
  const float qa = ax == 0 ? qx : (ax == 1 ? qy : qz), oa = ax == 0 ? g.ox : (ax == 1 ? g.oy : g.oz);
  if (up ? (hi[ax] >= n - 1) : (lo[ax] <= 0)) return false;
  const float b = up ? (oa + (float)(hi[ax] + 1) * g.cell) - qa : qa - (oa + (float)lo[ax] * g.cell);
  const float bs = b * 0.999f - g.slack;
  if (bs >= gate_r) return false;
  if (bs > 0.f && bd <= bs * bs) return false;
  return true;
}

// one query: the start box is the 3x3x3 cells around its (clamped) cell; faces are pushed out one cell layer at a time while
// they are open.  Every unscanned point lies beyond some closed face, so the result is the exact (distance, index) minimum
// among the points within the gate (gate_r = +inf: among all points).
__device__ __forceinline__ unsigned long long nn_search(const GridDesc& g, float qx, float qy, float qz, float gate_r) {
  unsigned long long best = KEY_EMPTY;
  float bd = __int_as_float(0x7f800000);
  const int cx = clampi(cell_coord(qx, g.ox, g.inv_cell), 0, g.nx - 1);
  const int cy = clampi(cell_coord(qy, g.oy, g.inv_cell), 0, g.ny - 1);
  const int cz = clampi(cell_coord(qz, g.oz, g.inv_cell), 0, g.nz - 1);
  int lo[3] = {cx - 1, cy - 1, cz - 1}, hi[3] = {cx + 1, cy + 1, cz + 1};
  nn_rows(g, lo[0], hi[0], lo[1], hi[1], lo[2], hi[2], qx, qy, qz, best, bd);
  const int rounds = g.nx + g.ny + g.nz + 3;
  for (int r = 0; r < rounds; ++r) {
    bool any = false;
#pragma unroll 1
    for (int f = 0; f < 6; ++f) {
      if (!nn_face_open(g, f, qx, qy, qz, gate_r, lo, hi, bd)) continue;
      const int ax = f >> 1;
      const bool up = (f & 1) != 0;
      const int nc = up ? hi[ax] + 1 : lo[ax] - 1;
      int b0[3] = {lo[0], lo[1], lo[2]}, b1[3] = {hi[0], hi[1], hi[2]};
      b0[ax] = b1[ax] = nc;
      if (up) hi[ax] = nc; else lo[ax] = nc;
      nn_rows(g, b0[0], b1[0], b0[1], b1[1], b0[2], b1[2], qx, qy, qz, best, bd);
      any = true;
    }
    if (!any) break;
  }
  return best;
}

// GATED: ICP correspondences (flag = float distance <= max_dist_sqr, PCL's `distance[0] > max_dist_sqr` rejection); returns at once
// when the registration is done.  Otherwise the fitness pass (no gate, every point counts).
template <bool GATED>
__global__ void __launch_bounds__(LC_T) k_lc_nn(GridDesc g, const float4* __restrict__ pts, const int* __restrict__ perm, int64_t n,
                                                double max_dist_sqr, float gate_r, const IcpState* __restrict__ st, int* __restrict__ nn_idx,
                                                float* __restrict__ nn_d, int* __restrict__ flags) {
  if (GATED && st->done) return;
  const int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= n) return;
  const int i = perm[p];
  const float4 q = pts[i];
  const unsigned long long k = nn_search(g, q.x, q.y, q.z, gate_r);
  const float d = key_dist(k);
  nn_idx[i] = key_idx(k);
  nn_d[i] = d;
  if (GATED) flags[i] = ((double)d <= max_dist_sqr) ? 1 : 0;
}

__global__ void __launch_bounds__(256) k_lc_compact(const IcpState* __restrict__ st, const int* __restrict__ flags, const int* __restrict__ pos,
                                                    int64_t n, const int* __restrict__ nn_idx, const float* __restrict__ nn_d,
                                                    int* __restrict__ cq, int* __restrict__ cm, float* __restrict__ cd) {
  if (st->done) return;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    if (!flags[i]) continue;
    const int o = pos[i];
    cq[o] = (int)i; cm[o] = nn_idx[i]; cd[o] = nn_d[i];
  }
}

// ---------------------------------------------------------------------------------------------------------------------
// deterministic sums (order: see the file header).  A partial record is 9 floats + 1 double, stored structure-of-arrays with
// row stride `ld`.
// ---------------------------------------------------------------------------------------------------------------------
enum { LC_SUM_MEANS = 0, LC_SUM_SIGMA = 1, LC_SUM_FIT = 2 };

__device__ __forceinline__ int64_t lc_count(int mode, const int* d_cnt, int64_t n) { return mode == LC_SUM_FIT ? n : (int64_t)*d_cnt; }

template <int MODE>
__global__ void __launch_bounds__(LC_T) k_lc_sum0(const IcpState* __restrict__ st, const int* __restrict__ d_cnt, int64_t n,
                                                  const float4* __restrict__ cur, const float4* __restrict__ tgt, const int* __restrict__ cq,
                                                  const int* __restrict__ cm, const float* __restrict__ dist, float* __restrict__ pf,
                                                  double* __restrict__ pd, int64_t ld) {
  if (MODE != LC_SUM_FIT && st->done) return;
  const int64_t cnt = lc_count(MODE, d_cnt, n);
  const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (r * LC_RUN >= cnt) return;
  const int64_t e = min(cnt, (r + 1) * LC_RUN);
  float acc[9];
#pragma unroll
  for (int k = 0; k < 9; ++k) acc[k] = 0.f;
  double ad = 0.0;
  float sm[3] = {0.f, 0.f, 0.f}, tm[3] = {0.f, 0.f, 0.f};
  if (MODE == LC_SUM_SIGMA) for (int k = 0; k < 3; ++k) { sm[k] = st->smean[k]; tm[k] = st->tmean[k]; }
  for (int64_t j = r * LC_RUN; j < e; ++j) {
    if (MODE == LC_SUM_FIT) { ad = ad + (double)dist[j]; continue; }
    const float4 s = cur[cq[j]], t = tgt[cm[j]];
    if (MODE == LC_SUM_MEANS) {
      acc[0] = acc[0] + s.x; acc[1] = acc[1] + s.y; acc[2] = acc[2] + s.z;
      acc[3] = acc[3] + t.x; acc[4] = acc[4] + t.y; acc[5] = acc[5] + t.z;
      ad = ad + (double)dist[j];
    } else {
      const float sd[3] = {s.x - sm[0], s.y - sm[1], s.z - sm[2]}, td[3] = {t.x - tm[0], t.y - tm[1], t.z - tm[2]};
#pragma unroll
      for (int a = 0; a < 3; ++a)
#pragma unroll
        for (int b = 0; b < 3; ++b) acc[3 * a + b] = acc[3 * a + b] + td[a] * sd[b];     // (dst_demean * src_demean^T)(a, b)
    }
  }
#pragma unroll
  for (int k = 0; k < 9; ++k) pf[k * ld + r] = acc[k];
  pd[r] = ad;
}

template <int MODE>
__global__ void __launch_bounds__(LC_T) k_lc_sum1(const IcpState* __restrict__ st, const int* __restrict__ d_cnt, int64_t n,
                                                  const float* __restrict__ pf0, const double* __restrict__ pd0, int64_t ld0,
                                                  float* __restrict__ pf1, double* __restrict__ pd1, int64_t ld1) {
  if (MODE != LC_SUM_FIT && st->done) return;
  const int64_t c0 = (lc_count(MODE, d_cnt, n) + LC_RUN - 1) / LC_RUN;
  const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (r * LC_RUN >= c0) return;
  const int64_t e = min(c0, (r + 1) * LC_RUN);
  float acc[9];
#pragma unroll
  for (int k = 0; k < 9; ++k) acc[k] = 0.f;
  double ad = 0.0;
  for (int64_t j = r * LC_RUN; j < e; ++j) {
#pragma unroll
    for (int k = 0; k < 9; ++k) acc[k] = acc[k] + pf0[k * ld0 + j];
    ad = ad + pd0[j];
  }
#pragma unroll
  for (int k = 0; k < 9; ++k) pf1[k * ld1 + r] = acc[k];
  pd1[r] = ad;
}

// level 2: the level-1 results in order (one thread)
__device__ __forceinline__ void lc_sum2(int64_t cnt, const float* pf1, const double* pd1, int64_t ld1, float (&s)[9], double& sd) {
  const int64_t c1 = ((cnt + LC_RUN - 1) / LC_RUN + LC_RUN - 1) / LC_RUN;
  for (int k = 0; k < 9; ++k) s[k] = 0.f;
  sd = 0.0;
  for (int64_t j = 0; j < c1; ++j) {
    for (int k = 0; k < 9; ++k) s[k] = s[k] + pf1[k * ld1 + j];
    sd = sd + pd1[j];
  }
}

__global__ void k_lc_means(IcpState* __restrict__ st, const int* __restrict__ d_cnt, const float* __restrict__ pf1, const double* __restrict__ pd1,
                           int64_t ld1) {
  if (threadIdx.x != 0 || st->done) return;
  const int cnt = *d_cnt;
  st->n_corr = cnt;
  if (cnt < 3) {                     // icp.hpp: "Not enough correspondences found", CONVERGENCE_CRITERIA_NO_CORRESPONDENCES
    st->converged = 0; st->state = GLIO_ICP_NO_CORRESPONDENCES; st->done = 1;
    return;
  }
  float s[9]; double sd;
  lc_sum2(cnt, pf1, pd1, ld1, s, sd);
  const float one_over_n = 1.f / (float)cnt;                       // umeyama: 1 / RealScalar(n)
  for (int k = 0; k < 3; ++k) { st->smean[k] = s[k] * one_over_n; st->tmean[k] = s[3 + k] * one_over_n; }
  st->mse = sd / (double)cnt;                                      // DefaultConvergenceCriteria::calculateMSE
}

// ---------------------------------------------------------------------------------------------------------------------
// Eigen 3.3 JacobiSVD<Matrix3f>(ComputeFullU | ComputeFullV) (Eigen/src/SVD/JacobiSVD.h compute, RealSvd2x2.h, Jacobi/Jacobi.h):
// square input, so no QR preconditioner; scaled by the largest |coefficient|; sweeps over (p,q) = (1,0), (2,0), (2,1) while an
// off-diagonal entry exceeds max(FLT_MIN, 2 eps maxDiagEntry); then signs made positive (U's columns flipped) and the values
// sorted descending (first maximum wins).  a is row-major.
// ---------------------------------------------------------------------------------------------------------------------
// apply_rotation_in_the_plane(x, y, (c, s)): x' = c x + s y, y' = -s x + c y; skipped for (1, 0)
__device__ __forceinline__ void lc_plane(float* x, float* y, int inc, float c, float s) {
  if (c == 1.f && s == 0.f) return;
  for (int i = 0; i < 3; ++i) {
    const float xi = x[i * inc], yi = y[i * inc];
    x[i * inc] = c * xi + s * yi;
    y[i * inc] = -s * xi + c * yi;
  }
}

__device__ void lc_svd3(const float a[9], float U[9], float sv[3], float V[9]) {
  float W[9];
  float scale = 0.f;
  for (int k = 0; k < 9; ++k) scale = fmaxf(scale, fabsf(a[k]));
  if (scale == 0.f) scale = 1.f;
  for (int k = 0; k < 9; ++k) { W[k] = a[k] / scale; U[k] = (k % 4 == 0) ? 1.f : 0.f; V[k] = U[k]; }
  float maxDiag = fabsf(W[0]);
  if (fabsf(W[4]) > maxDiag) maxDiag = fabsf(W[4]);
  if (fabsf(W[8]) > maxDiag) maxDiag = fabsf(W[8]);
  const float precision = 2.f * FLT_EPSILON;
  bool finished = false;
  for (int sweep = 0; !finished && sweep < 256; ++sweep) {
    finished = true;
    for (int p = 1; p < 3; ++p)
      for (int q = 0; q < p; ++q) {
        const float thr = fmaxf(FLT_MIN, precision * maxDiag);
        if (!(fabsf(W[3 * p + q]) > thr || fabsf(W[3 * q + p]) > thr)) continue;
        finished = false;
        // real_2x2_jacobi_svd
        float m00 = W[3 * p + p], m01 = W[3 * p + q], m10 = W[3 * q + p], m11 = W[3 * q + q];
        const float t = m00 + m11, d = m10 - m01;
        float rc, rs;
        if (fabsf(d) < FLT_MIN) { rs = 0.f; rc = 1.f; }
        else { const float u = t / d; const float tmp = sqrtf(1.f + u * u); rs = 1.f / tmp; rc = u / tmp; }
        if (!(rc == 1.f && rs == 0.f)) {
          const float a0 = m00, a1 = m01, b0 = m10, b1 = m11;
          m00 = rc * a0 + rs * b0; m01 = rc * a1 + rs * b1;
          m10 = -rs * a0 + rc * b0; m11 = -rs * a1 + rc * b1;
        }
        (void)m10;
        // j_right.makeJacobi(m, 0, 1)
        float jrc = 1.f, jrs = 0.f;
        const float deno = 2.f * fabsf(m01);
        if (!(deno < FLT_MIN)) {
          const float tau = (m00 - m11) / deno;
          const float w = sqrtf(tau * tau + 1.f);
          const float tt = tau > 0.f ? 1.f / (tau + w) : 1.f / (tau - w);
          const float sign_t = tt > 0.f ? 1.f : -1.f;
          const float nn = 1.f / sqrtf(tt * tt + 1.f);
          jrs = ((-sign_t * (m01 / fabsf(m01))) * fabsf(tt)) * nn;
          jrc = nn;
        }
        // j_left = rot1 * j_right.transpose()
        const float jlc = rc * jrc - rs * (-jrs);
        const float jls = rc * (-jrs) + rs * jrc;
        lc_plane(W + 3 * p, W + 3 * q, 1, jlc, jls);          // m_workMatrix.applyOnTheLeft(p, q, j_left): rows
        lc_plane(U + p, U + q, 3, jlc, jls);                  // m_matrixU.applyOnTheRight(p, q, j_left.transpose()): columns
        lc_plane(W + p, W + q, 3, jrc, -jrs);                 // m_workMatrix.applyOnTheRight(p, q, j_right)
        lc_plane(V + p, V + q, 3, jrc, -jrs);                 // m_matrixV.applyOnTheRight(p, q, j_right)
        const float dm = fmaxf(fabsf(W[3 * p + p]), fabsf(W[3 * q + q]));
        if (maxDiag < dm) maxDiag = dm;
      }
  }
  for (int i = 0; i < 3; ++i) {
    const float a_ii = W[4 * i];
    sv[i] = fabsf(a_ii);
    if (a_ii < 0.f) for (int r = 0; r < 3; ++r) U[3 * r + i] = -U[3 * r + i];
  }
  for (int i = 0; i < 3; ++i) sv[i] = sv[i] * scale;
  for (int i = 0; i < 3; ++i) {
    int pos = i;
    for (int j = i + 1; j < 3; ++j) if (sv[j] > sv[pos]) pos = j;
    if (sv[pos] == 0.f) break;
    if (pos != i) {
      float tmp = sv[i]; sv[i] = sv[pos]; sv[pos] = tmp;
      for (int r = 0; r < 3; ++r) {
        tmp = U[3 * r + i]; U[3 * r + i] = U[3 * r + pos]; U[3 * r + pos] = tmp;
        tmp = V[3 * r + i]; V[3 * r + i] = V[3 * r + pos]; V[3 * r + pos] = tmp;
      }
    }
  }
}

// Eigen determinant_impl<3>: bruteforce_det3_helper(m,0,1,2) - (m,1,0,2) + (m,2,0,1), m(0,a) * (m(1,b) m(2,c) - m(1,c) m(2,b))
__device__ __forceinline__ float lc_det3(const float m[9]) {
  auto h = [&](int a, int b, int c) { return m[a] * (m[3 + b] * m[6 + c] - m[3 + c] * m[6 + b]); };
  return h(0, 1, 2) - h(1, 0, 2) + h(2, 0, 1);
}

// sigma, SVD, transformation (pcl::umeyama without scaling), final = transformation * final, ++nr_iterations, the convergence test
__global__ void k_lc_solve(IcpState* __restrict__ st, const int* __restrict__ d_cnt, const float* __restrict__ pf1, const double* __restrict__ pd1,
                           int64_t ld1, IcpConvergence cc, glio_icp_iteration* __restrict__ log) {
  if (threadIdx.x != 0 || st->done) return;
  const int cnt = *d_cnt;
  float s[9]; double sd;
  lc_sum2(cnt, pf1, pd1, ld1, s, sd);
  const float one_over_n = 1.f / (float)cnt;
  float sigma[9];
  for (int k = 0; k < 9; ++k) sigma[k] = one_over_n * s[k];
  float U[9], sv[3], V[9];
  lc_svd3(sigma, U, sv, V);
  const float S2 = (lc_det3(U) * lc_det3(V) < 0.f) ? -1.f : 1.f;
  float T[16];
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j)                                   // (U S) V^T, coefficient-based, k in order
      T[4 * i + j] = ((U[3 * i] * 1.f) * V[3 * j] + (U[3 * i + 1] * 1.f) * V[3 * j + 1]) + (U[3 * i + 2] * S2) * V[3 * j + 2];
  for (int i = 0; i < 3; ++i)                                     // t = dst_mean; t -= R src_mean (column-major GEMV order)
    T[4 * i + 3] = ((st->tmean[i] - T[4 * i] * st->smean[0]) - T[4 * i + 1] * st->smean[1]) - T[4 * i + 2] * st->smean[2];
  T[12] = 0.f; T[13] = 0.f; T[14] = 0.f; T[15] = 1.f;
  float F[16];
  for (int i = 0; i < 4; ++i)
    for (int j = 0; j < 4; ++j)
      F[4 * i + j] = ((T[4 * i] * st->final_T[j] + T[4 * i + 1] * st->final_T[4 + j]) + T[4 * i + 2] * st->final_T[8 + j]) + T[4 * i + 3] * st->final_T[12 + j];
  for (int k = 0; k < 16; ++k) { st->transformation[k] = T[k]; st->final_T[k] = F[k]; }
  const int it = st->nr_iter;
  st->nr_iter = it + 1;
  if (log && it < cc.log_cap) {
    for (int k = 0; k < 16; ++k) log[it].transformation[k] = T[k];
    log[it].n_corr = cnt; log[it].mse = st->mse;
  }
  // DefaultConvergenceCriteria::hasConverged (max_iterations_similar_transforms_ = 0, failure_after_max_iter_ = false)
  if (it + 1 >= cc.max_iterations) { st->converged = 1; st->state = GLIO_ICP_ITERATIONS; st->done = 1; return; }
  const double cos_angle = 0.5 * (double)(((T[0] + T[5]) + T[10]) - 1.f);
  const double translation_sqr = (double)((T[3] * T[3] + T[7] * T[7]) + T[11] * T[11]);
  if (cos_angle >= cc.rotation_threshold && translation_sqr <= cc.translation_threshold) {
    st->converged = 1; st->state = GLIO_ICP_TRANSFORM; st->done = 1; return;
  }
  const double mse = st->mse, prev = st->prev_mse;
  if (fabs(mse - prev) < cc.mse_threshold_absolute) { st->converged = 1; st->state = GLIO_ICP_ABS_MSE; st->done = 1; return; }
  if (fabs(mse - prev) / prev < cc.mse_threshold_relative) { st->converged = 1; st->state = GLIO_ICP_REL_MSE; st->done = 1; return; }
  st->prev_mse = mse;
}

// IterativeClosestPoint::transformCloud: pt_t = tr * (x, y, z, 1) in float, ((t0 x + t1 y) + t2 z) + t3
__device__ __forceinline__ float4 lc_apply(const float* T, float4 p) {
  return make_float4(((T[0] * p.x + T[1] * p.y) + T[2] * p.z) + T[3], ((T[4] * p.x + T[5] * p.y) + T[6] * p.z) + T[7],
                     ((T[8] * p.x + T[9] * p.y) + T[10] * p.z) + T[11], p.w);
}

// in place, only when iteration `it` ran its estimation (the device iteration counter moved to it + 1)
__global__ void __launch_bounds__(256) k_lc_transform(const IcpState* __restrict__ st, int it, float4* __restrict__ cur, int64_t n) {
  __shared__ float T[16];
  __shared__ int go;
  if (threadIdx.x == 0) go = st->nr_iter == it + 1;
  if (threadIdx.x < 16) T[threadIdx.x] = st->transformation[threadIdx.x];
  __syncthreads();
  if (!go) return;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) cur[i] = lc_apply(T, cur[i]);
}

// the aligned cloud: the INPUT transformed by final (recomputed, not the accumulated cloud)
__global__ void __launch_bounds__(256) k_lc_final(const IcpState* __restrict__ st, const float4* __restrict__ src, float4* __restrict__ out, int64_t n) {
  __shared__ float T[16];
  if (threadIdx.x < 16) T[threadIdx.x] = st->final_T[threadIdx.x];
  __syncthreads();
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) out[i] = lc_apply(T, src[i]);
}

__global__ void k_lc_fitness(IcpState* __restrict__ st, int64_t n, const float* __restrict__ pf1, const double* __restrict__ pd1, int64_t ld1) {
  if (threadIdx.x != 0) return;
  float s[9]; double sd;
  lc_sum2(n, pf1, pd1, ld1, s, sd);
  st->nr_fit = (int)n;
  st->fitness = n > 0 ? sd / (double)n : DBL_MAX;
}

// ---------------------------------------------------------------------------------------------------------------------
// host driver
// ---------------------------------------------------------------------------------------------------------------------
static unsigned lc_blocks(int64_t n, int t) { return (unsigned)std::max<int64_t>(1, (n + t - 1) / t); }

void icp_run(IcpWork& w, const float* d_src, int src_stride, int64_t n_src, const float* d_tgt, int tgt_stride, int64_t n_tgt,
             const glio_icp_options& o, int log_cap, float pts_per_cell, cudaStream_t st, LaunchCounter& lc, IcpState* out, int* host_syncs) {
  GLIO_REQUIRE(n_src >= 0 && n_src < ((int64_t)1 << 30) && n_tgt >= 0 && n_tgt < ((int64_t)1 << 30), GLIO_ERR_ARG, "icp: cloud size out of range");
  int syncs = 0;
  w.n_src = n_src; w.n_tgt = n_tgt;
  w.state.reserve(1);
  lc.begin("k_lc_init", st); k_lc_init<<<1, 32, 0, st>>>(w.state.p); lc.end(st);
  if (n_src == 0 || n_tgt == 0) {
    // nothing to search with or against: no correspondence, the aligned cloud is the input under the identity, and
    // getFitnessScore counts no point
    if (n_src > 0) {
      w.src0.reserve(n_src); w.cur.reserve(n_src); w.fit.reserve(n_src);
      const int nb = (int)std::min<int64_t>((n_src + 255) / 256, kNumSMs * 8);
      lc.begin("k_lc_load", st); k_lc_load<<<nb, 256, 0, st>>>(d_src, src_stride, n_src, w.src0.p, w.cur.p); lc.end(st);
      lc.begin("k_lc_final", st); k_lc_final<<<nb, 256, 0, st>>>(w.state.p, w.src0.p, w.fit.p, n_src); lc.end(st);
    }
    IcpState h;
    GLIO_CUDA_TRY(cudaMemcpyAsync(&h, w.state.p, sizeof(h), cudaMemcpyDeviceToHost, st));
    GLIO_CUDA_TRY(cudaStreamSynchronize(st)); ++syncs;
    h.converged = 0; h.state = GLIO_ICP_NO_CORRESPONDENCES; h.done = 1; h.n_corr = 0;
    *out = h; w.last = h;
    if (host_syncs) *host_syncs = syncs;
    return;
  }
  const int64_t n = n_src;
  const int64_t r0 = (n + LC_RUN - 1) / LC_RUN, r1 = (r0 + LC_RUN - 1) / LC_RUN;
  w.src0.reserve(n); w.cur.reserve(n); w.fit.reserve(n);
  w.nn_idx.reserve(n); w.nn_d.reserve(n); w.flags.reserve(n + 1); w.pos.reserve(n + 1); w.perm.reserve(n);
  w.cq.reserve(n); w.cm.reserve(n); w.cd.reserve(n);
  w.pf0.reserve(9 * r0); w.pd0.reserve(r0); w.pf1.reserve(9 * r1); w.pd1.reserve(r1);
  w.log.reserve(std::max(1, log_cap));
  const int nb = (int)std::min<int64_t>((n + 255) / 256, kNumSMs * 8);
  lc.begin("k_lc_load", st); k_lc_load<<<nb, 256, 0, st>>>(d_src, src_stride, n, w.src0.p, w.cur.p); lc.end(st);
  // the target stays fixed over the iterations: one K0 grid (kd_tree->setInputCloud (target_), Registration::initCompute)
  grid_build(w.grid, d_tgt, tgt_stride, n_tgt, nullptr, nullptr, 0.f, pts_per_cell, st, lc); ++syncs;
  const GridDesc g = w.grid.desc;
  // cell order of the source, once: the cloud moves little from one iteration to the next, warps keep their locality
  const int64_t ncell = (int64_t)g.nx * g.ny * g.nz;
  w.qcount.reserve(ncell + 2); w.qstart.reserve(ncell + 2);
  GLIO_CUDA_TRY(cudaMemsetAsync(w.qcount.p, 0, (size_t)(ncell + 1) * sizeof(int), st));
  lc.begin("k_lc_qhist", st); k_lc_qhist<<<nb, 256, 0, st>>>(g, w.src0.p, n, w.qcount.p); lc.end(st);
  exclusive_scan_i32(w.qcount.p, w.qstart.p, ncell + 1, w.scan_tmp, st, lc);
  GLIO_CUDA_TRY(cudaMemsetAsync(w.qcount.p, 0, (size_t)(ncell + 1) * sizeof(int), st));
  lc.begin("k_lc_qscatter", st); k_lc_qscatter<<<nb, 256, 0, st>>>(g, w.src0.p, n, w.qstart.p, w.qcount.p, w.perm.p); lc.end(st);
  GLIO_CUDA_TRY(cudaMemsetAsync(w.flags.p, 0, (size_t)(n + 1) * sizeof(int), st));   // flags[n] = 0: pos[n] = count
  const double max_dist_sqr = o.max_correspondence_distance * o.max_correspondence_distance;
  const float gate_r = (float)std::sqrt(max_dist_sqr) + g.slack;
  IcpConvergence cc;
  cc.max_iterations = o.max_iterations;
  cc.translation_threshold = o.transformation_epsilon;              // icp.hpp: setTranslationThreshold (transformation_epsilon_)
  cc.rotation_threshold = 1.0 - o.transformation_epsilon;           //           setRotationThreshold (1.0 - transformation_epsilon_)
  cc.mse_threshold_relative = o.euclidean_fitness_epsilon;          //           setRelativeMSE (euclidean_fitness_epsilon_)
  cc.mse_threshold_absolute = 1e-12;                                // DefaultConvergenceCriteria's default
  cc.log_cap = log_cap;
  const int* d_cnt = w.pos.p + n;
  const unsigned nbq = lc_blocks(n, LC_T), nb0 = lc_blocks(r0, LC_T), nb1 = lc_blocks(r1, LC_T);
  IcpState h;
  int it = 0, batch = 8;
  bool done = o.max_iterations <= 0;
  while (!done) {
    const int nit = std::min(batch, o.max_iterations - it);
    for (int k = 0; k < nit; ++k, ++it) {
      lc.begin("k_lc_nn", st);
      k_lc_nn<true><<<nbq, LC_T, 0, st>>>(g, w.cur.p, w.perm.p, n, max_dist_sqr, gate_r, w.state.p, w.nn_idx.p, w.nn_d.p, w.flags.p);
      lc.end(st);
      exclusive_scan_i32(w.flags.p, w.pos.p, n + 1, w.scan_tmp, st, lc);
      lc.begin("k_lc_compact", st);
      k_lc_compact<<<nb, 256, 0, st>>>(w.state.p, w.flags.p, w.pos.p, n, w.nn_idx.p, w.nn_d.p, w.cq.p, w.cm.p, w.cd.p);
      lc.end(st);
      lc.begin("k_lc_sum0", st);
      k_lc_sum0<LC_SUM_MEANS><<<nb0, LC_T, 0, st>>>(w.state.p, d_cnt, n, w.cur.p, w.grid.tmp4.p, w.cq.p, w.cm.p, w.cd.p, w.pf0.p, w.pd0.p, r0);
      lc.end(st);
      lc.begin("k_lc_sum1", st);
      k_lc_sum1<LC_SUM_MEANS><<<nb1, LC_T, 0, st>>>(w.state.p, d_cnt, n, w.pf0.p, w.pd0.p, r0, w.pf1.p, w.pd1.p, r1);
      lc.end(st);
      lc.begin("k_lc_means", st); k_lc_means<<<1, 32, 0, st>>>(w.state.p, d_cnt, w.pf1.p, w.pd1.p, r1); lc.end(st);
      lc.begin("k_lc_sum0", st);
      k_lc_sum0<LC_SUM_SIGMA><<<nb0, LC_T, 0, st>>>(w.state.p, d_cnt, n, w.cur.p, w.grid.tmp4.p, w.cq.p, w.cm.p, w.cd.p, w.pf0.p, w.pd0.p, r0);
      lc.end(st);
      lc.begin("k_lc_sum1", st);
      k_lc_sum1<LC_SUM_SIGMA><<<nb1, LC_T, 0, st>>>(w.state.p, d_cnt, n, w.pf0.p, w.pd0.p, r0, w.pf1.p, w.pd1.p, r1);
      lc.end(st);
      lc.begin("k_lc_solve", st); k_lc_solve<<<1, 32, 0, st>>>(w.state.p, d_cnt, w.pf1.p, w.pd1.p, r1, cc, log_cap > 0 ? w.log.p : nullptr); lc.end(st);
      lc.begin("k_lc_transform", st); k_lc_transform<<<nb, 256, 0, st>>>(w.state.p, it, w.cur.p, n); lc.end(st);
    }
    GLIO_CUDA_TRY(cudaMemcpyAsync(&h, w.state.p, sizeof(h), cudaMemcpyDeviceToHost, st));
    GLIO_CUDA_TRY(cudaStreamSynchronize(st)); ++syncs;
    done = h.done || it >= o.max_iterations;
    batch = std::min(batch * 2, 32);
  }
  // getFitnessScore (): the input transformed by final, 1-NN without gate, double mean
  lc.begin("k_lc_final", st); k_lc_final<<<nb, 256, 0, st>>>(w.state.p, w.src0.p, w.fit.p, n); lc.end(st);
  lc.begin("k_lc_nn", st);
  k_lc_nn<false><<<nbq, LC_T, 0, st>>>(g, w.fit.p, w.perm.p, n, 0.0, INFINITY, w.state.p, w.nn_idx.p, w.nn_d.p, nullptr);
  lc.end(st);
  lc.begin("k_lc_sum0", st);
  k_lc_sum0<LC_SUM_FIT><<<nb0, LC_T, 0, st>>>(w.state.p, nullptr, n, nullptr, nullptr, nullptr, nullptr, w.nn_d.p, w.pf0.p, w.pd0.p, r0);
  lc.end(st);
  lc.begin("k_lc_sum1", st);
  k_lc_sum1<LC_SUM_FIT><<<nb1, LC_T, 0, st>>>(w.state.p, nullptr, n, w.pf0.p, w.pd0.p, r0, w.pf1.p, w.pd1.p, r1);
  lc.end(st);
  lc.begin("k_lc_fitness", st); k_lc_fitness<<<1, 32, 0, st>>>(w.state.p, n, w.pf1.p, w.pd1.p, r1); lc.end(st);
  GLIO_CUDA_TRY(cudaGetLastError());
  GLIO_CUDA_TRY(cudaMemcpyAsync(&h, w.state.p, sizeof(h), cudaMemcpyDeviceToHost, st));
  GLIO_CUDA_TRY(cudaStreamSynchronize(st)); ++syncs;
  *out = h; w.last = h;
  if (host_syncs) *host_syncs = syncs;
}

// ---------------------------------------------------------------------------------------------------------------------
// save_pcd's global map (Estimator.cpp:5324-5349): transformCloud(transformCloud(surf_frames[i], &Tbl), &pose_info_keyframe[i]), two
// float roundings per point; one launch over every segment (blockIdx.y strides the segments)
// ---------------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_gm_transform(const GlobalMapSeg* __restrict__ segs, int nseg, PoseD first, float4* __restrict__ out) {
  for (int s = blockIdx.y; s < nseg; s += gridDim.y) {
    const GlobalMapSeg g = segs[s];
    PoseD pose;
    for (int k = 0; k < 3; ++k) pose.t[k] = g.t[k];
    for (int k = 0; k < 4; ++k) pose.q[k] = g.q[k];
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < g.n; i += (int64_t)gridDim.x * blockDim.x) {
      float p[3] = {g.xyz[3 * i], g.xyz[3 * i + 1], g.xyz[3 * i + 2]};
      transform_point_f(first, p, p);
      transform_point_f(pose, p, p);
      out[g.off + i] = make_float4(p[0], p[1], p[2], 0.f);
    }
  }
}

void loop_global_map_cloud(const GlobalMapSeg* d_segs, int nseg, int64_t n_max, const double t_first[3], const double q_first[4], float4* out,
                           cudaStream_t st, LaunchCounter& lc) {
  if (nseg <= 0 || n_max <= 0) return;
  PoseD first;
  for (int k = 0; k < 3; ++k) first.t[k] = t_first[k];
  for (int k = 0; k < 4; ++k) first.q[k] = q_first[k];
  const dim3 grid((unsigned)std::min<int64_t>((n_max + 255) / 256, 64), (unsigned)std::min(nseg, 65535));
  lc.begin("k_gm_transform", st); k_gm_transform<<<grid, 256, 0, st>>>(d_segs, nseg, first, out); lc.end(st);
  GLIO_CUDA_TRY(cudaGetLastError());
}

// ---------------------------------------------------------------------------------------------------------------------
// host pose arithmetic of performLoopClosure (scalar double, Eigen's operation order, no FMA: this unit is -fmad=false and
// the host compiler targets baseline x86-64)
// ---------------------------------------------------------------------------------------------------------------------
// Eigen quaternion_assign_impl<Other, 3, 3>: rotation matrix -> quaternion (w, x, y, z)
void loop_quat_from_R(const double R[9], double q[4]) {
  double t = (R[0] + R[4]) + R[8];
  if (t > 0.0) {
    t = std::sqrt(t + 1.0);
    q[0] = 0.5 * t;
    t = 0.5 / t;
    q[1] = (R[7] - R[5]) * t;
    q[2] = (R[2] - R[6]) * t;
    q[3] = (R[3] - R[1]) * t;
  } else {
    int i = 0;
    if (R[4] > R[0]) i = 1;
    if (R[8] > R[3 * i + i]) i = 2;
    const int j = (i + 1) % 3, k = (j + 1) % 3;
    t = std::sqrt(((R[3 * i + i] - R[3 * j + j]) - R[3 * k + k]) + 1.0);
    double c[3];
    c[i] = 0.5 * t;
    t = 0.5 / t;
    q[0] = (R[3 * k + j] - R[3 * j + k]) * t;
    c[j] = (R[3 * j + i] + R[3 * i + j]) * t;
    c[k] = (R[3 * k + i] + R[3 * i + k]) * t;
    q[1] = c[0]; q[2] = c[1]; q[3] = c[2];
  }
}

// q_bl = q_lb.inverse(), t_bl = -(q_bl * t_lb)   (Estimator.cpp:873-877)
void loop_extrinsic_bl(const double q_lb[4], const double t_lb[3], double q_bl[4], double t_bl[3]) {
  odom_quat_inverse(q_lb, q_bl);
  double r[3]; h_qrot(q_bl, t_lb, r);
  t_bl[0] = -r[0]; t_bl[1] = -r[1]; t_bl[2] = -r[2];
}

// q_tmp = q_po * q_bl, t_tmp = q_po * t_bl + t_po   (Estimator.cpp:5140-5141); pose = t, q
void loop_world_of_cloud(const double pose[7], const double q_bl[4], const double t_bl[3], double t[3], double q[4]) {
  h_qmul(pose + 3, q_bl, q);
  double r[3]; h_qrot(pose + 3, t_bl, r);
  t[0] = r[0] + pose[0]; t[1] = r[1] + pose[1]; t[2] = r[2] + pose[2];
}

// quaternionIncre (R of final), quaternionCorrected = qIncre * q_latest, transitionCorrected = qIncre * t_latest + tIncre (:5228-5242)
void loop_pose_from(const float F[16], const double latest[7], double out[7]) {
  const double R[9] = {(double)F[0], (double)F[1], (double)F[2], (double)F[4], (double)F[5], (double)F[6], (double)F[8], (double)F[9], (double)F[10]};
  double qi[4]; loop_quat_from_R(R, qi);
  double q[4]; h_qmul(qi, latest + 3, q);
  double r[3]; h_qrot(qi, latest, r);
  out[0] = r[0] + (double)F[3]; out[1] = r[1] + (double)F[7]; out[2] = r[2] + (double)F[11];
  out[3] = q[0]; out[4] = q[1]; out[5] = q[2]; out[6] = q[3];
}

}  // namespace glio
