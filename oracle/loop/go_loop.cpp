/*
 * go_loop.cpp — CPU oracle of the loop-closure registration (SURVEY 8 f-7): detectLoopClosure's candidate search and
 * performLoopClosure's pcl::IterativeClosestPoint + getFitnessScore (GLIO/src/Estimator.cpp:5101-5273), sequential.
 *
 * TEST INFRASTRUCTURE ONLY.  Nothing under glio_b200/ may include, link or call this.
 *
 * Restated from the published sources of the reference's dependencies, none of which is in the image:
 *   PCL 1.8   registration/impl/icp.hpp (computeTransformation, transformCloud), correspondence_estimation.hpp
 *             (determineCorrespondences), transformation_estimation_svd.hpp + common/impl/eigen.hpp (pcl::umeyama, no scaling),
 *             default_convergence_criteria.hpp (hasConverged, calculateMSE), registration.hpp (getFitnessScore);
 *   Eigen 3.3 JacobiSVD (SVD/JacobiSVD.h compute, SVD/RealSvd2x2.h, Jacobi/Jacobi.h makeJacobi / apply_rotation_in_the_plane),
 *             determinant_impl<3>;
 *   FLANN     L2_Simple<float> (((0 + dx^2) + dy^2) + dz^2 in float), radius search kept when dist < float(r^2), sorted by
 *             (distance, index); exact 1-NN, ties by index.
 *
 * PARITY UNPINNED (stated, not hidden):
 *   - PCL's ICP and convergence code itself (PCL is absent): the state machine above is restated from its source;
 *   - Eigen's JacobiSVD, umeyama and GEMM order: the SVD is restated operation by operation; the products U S V^T,
 *     R * src_mean and transformation * final use the coefficient-based / column-major GEMV orders written below;
 *   - Eigen's packet reductions (rowwise().sum(), the sigma GEMM): replaced by the device's documented order, runs of 64
 *     summed left to right from zero, twice, then the run results in order (glio_b200/csrc/loop.cu);
 *   - PCL's sequential double MSE / fitness order: the same hierarchical order in double;
 *   - FLANN's radius-search boundary (strict <) and tie order (by index);
 *   - the VoxelGrid points of DESIGN 2 (the clouds are assembled by oracle/pyoracle_loop.py on the existing voxel filter).
 * tests/test_loop_closure.py checks the SVD against LAPACK, umeyama on exact data, every convergence exit, the detection against
 * numpy, the ICP against an independent float64 Kabsch ICP and the 1-NN against OpenCV's FLANN.
 *
 * Floating point: -ffp-contract=off, SSE2 float / double, so every operation rounds as written.
 */
#include <stdint.h>

#include <algorithm>
#include <cfloat>
#include <cmath>
#include <cstring>
#include <memory>
#include <utility>
#include <vector>

extern "C" {

enum { GO_ICP_NOT_CONVERGED = 0, GO_ICP_ITERATIONS = 1, GO_ICP_TRANSFORM = 2, GO_ICP_ABS_MSE = 3, GO_ICP_REL_MSE = 4, GO_ICP_NO_CORRESPONDENCES = 5 };

typedef struct {
  int32_t converged, state, iterations, pad;
  int64_t n_corr;
  float final_T[16];
  double fitness;
} go_icp_result;

typedef struct {
  float transformation[16];
  int64_t n_corr;
  double mse;
} go_icp_iteration;
}

namespace {

constexpr int RUN = 64;

// the device's summation order: runs of 64 from zero, twice, then the run results in order
template <class T>
T hsum(const std::vector<T>& v) {
  std::vector<T> l0, l1;
  for (size_t r = 0; r < v.size(); r += RUN) { T a = 0; for (size_t j = r; j < std::min(v.size(), r + RUN); ++j) a = a + v[j]; l0.push_back(a); }
  for (size_t r = 0; r < l0.size(); r += RUN) { T a = 0; for (size_t j = r; j < std::min(l0.size(), r + RUN); ++j) a = a + l0[j]; l1.push_back(a); }
  T a = 0;
  for (T x : l1) a = a + x;
  return a;
}

inline float l2_simple(const float* a, const float* b) {
  float r = 0.f;
  const float d0 = a[0] - b[0], d1 = a[1] - b[1], d2 = a[2] - b[2];
  r = r + d0 * d0; r = r + d1 * d1; r = r + d2 * d2;
  return r;
}

// exact 1-NN by (float distance, index): a median-split kd-tree; a subtree is skipped only when the float square of the distance to
// its splitting plane (a lower bound of every float L2_Simple distance inside, by monotone rounding) exceeds the best distance
struct Tree {
  std::vector<float> p;      // 3 per point, original order
  std::vector<int> idx;
  struct Node { int lo, hi, dim, left, right; float split; };
  std::vector<Node> nodes;
  int build(int lo, int hi) {
    Node nd{lo, hi, -1, -1, -1, 0.f};
    const int id = (int)nodes.size();
    nodes.push_back(nd);
    if (hi - lo <= 16) return id;
    float mn[3] = {FLT_MAX, FLT_MAX, FLT_MAX}, mx[3] = {-FLT_MAX, -FLT_MAX, -FLT_MAX};
    for (int k = lo; k < hi; ++k) for (int d = 0; d < 3; ++d) { mn[d] = std::min(mn[d], p[3 * idx[k] + d]); mx[d] = std::max(mx[d], p[3 * idx[k] + d]); }
    int dim = 0;
    for (int d = 1; d < 3; ++d) if (mx[d] - mn[d] > mx[dim] - mn[dim]) dim = d;
    if (!(mx[dim] > mn[dim])) return id;                   // all points equal: one leaf
    const int mid = (lo + hi) / 2;
    std::nth_element(idx.begin() + lo, idx.begin() + mid, idx.begin() + hi, [&](int a, int b) { return p[3 * a + dim] < p[3 * b + dim]; });
    const float split = p[3 * idx[mid] + dim];
    const int l = build(lo, mid), r = build(mid, hi);
    nodes[id].dim = dim; nodes[id].split = split; nodes[id].left = l; nodes[id].right = r;
    return id;
  }
  void search(int id, const float* q, float& bd, int& bi) const {
    const Node& nd = nodes[id];
    if (nd.dim < 0) {
      for (int k = nd.lo; k < nd.hi; ++k) {
        const int i = idx[k];
        const float d = l2_simple(q, &p[3 * i]);
        if (d < bd || (d == bd && i < bi)) { bd = d; bi = i; }
      }
      return;
    }
    const float diff = q[nd.dim] - nd.split;
    const int near = diff < 0.f ? nd.left : nd.right, far = diff < 0.f ? nd.right : nd.left;
    search(near, q, bd, bi);
    const float lb = diff * diff;
    if (!(lb > bd)) search(far, q, bd, bi);
  }
};

std::unique_ptr<Tree> make_tree(const float* xyz, int64_t m, int stride) {
  std::unique_ptr<Tree> t(new Tree());
  t->p.resize((size_t)m * 3);
  for (int64_t i = 0; i < m; ++i) for (int d = 0; d < 3; ++d) t->p[3 * i + d] = xyz[i * stride + d];
  t->idx.resize((size_t)m);
  for (int64_t i = 0; i < m; ++i) t->idx[i] = (int)i;
  if (m > 0) t->build(0, (int)m);
  return t;
}

// apply_rotation_in_the_plane(x, y, (c, s)) on 3-vectors at stride inc
void plane(float* x, float* y, int inc, float c, float s) {
  if (c == 1.f && s == 0.f) return;
  for (int i = 0; i < 3; ++i) {
    const float xi = x[i * inc], yi = y[i * inc];
    x[i * inc] = c * xi + s * yi;
    y[i * inc] = -s * xi + c * yi;
  }
}

// Eigen 3.3 JacobiSVD<Matrix3f>(a, ComputeFullU | ComputeFullV), a row-major
void svd3(const float a[9], float U[9], float sv[3], float V[9]) {
  float W[9];
  float scale = 0.f;
  for (int k = 0; k < 9; ++k) scale = std::max(scale, std::fabs(a[k]));
  if (scale == 0.f) scale = 1.f;
  for (int k = 0; k < 9; ++k) { W[k] = a[k] / scale; U[k] = (k % 4 == 0) ? 1.f : 0.f; V[k] = U[k]; }
  float maxDiag = std::max(std::max(std::fabs(W[0]), std::fabs(W[4])), std::fabs(W[8]));
  const float precision = 2.f * FLT_EPSILON, considerAsZero = FLT_MIN;
  bool finished = false;
  for (int sweep = 0; !finished && sweep < 256; ++sweep) {
    finished = true;
    for (int p = 1; p < 3; ++p)
      for (int q = 0; q < p; ++q) {
        const float threshold = std::max(considerAsZero, precision * maxDiag);
        if (!(std::fabs(W[3 * p + q]) > threshold || std::fabs(W[3 * q + p]) > threshold)) continue;
        finished = false;
        // real_2x2_jacobi_svd: rot1 makes the 2x2 block symmetric, makeJacobi diagonalises it
        float m[4] = {W[3 * p + p], W[3 * p + q], W[3 * q + p], W[3 * q + q]};   // row-major 2x2
        const float t = m[0] + m[3], d = m[2] - m[1];
        float c1, s1;
        if (std::fabs(d) < considerAsZero) { s1 = 0.f; c1 = 1.f; }
        else { const float u = t / d; const float tmp = std::sqrt(1.f + u * u); s1 = 1.f / tmp; c1 = u / tmp; }
        if (!(c1 == 1.f && s1 == 0.f))       // m.applyOnTheLeft(0, 1, rot1)
          for (int col = 0; col < 2; ++col) { const float xi = m[col], yi = m[2 + col]; m[col] = c1 * xi + s1 * yi; m[2 + col] = -s1 * xi + c1 * yi; }
        float jc = 1.f, js = 0.f;             // makeJacobi(m(0,0), m(0,1), m(1,1))
        const float x = m[0], y = m[1], z = m[3];
        const float deno = 2.f * std::fabs(y);
        if (!(deno < considerAsZero)) {
          const float tau = (x - z) / deno;
          const float w = std::sqrt(tau * tau + 1.f);
          const float tt = tau > 0.f ? 1.f / (tau + w) : 1.f / (tau - w);
          const float sign_t = tt > 0.f ? 1.f : -1.f;
          const float n = 1.f / std::sqrt(tt * tt + 1.f);
          js = ((-sign_t * (y / std::fabs(y))) * std::fabs(tt)) * n;
          jc = n;
        }
        // j_left = rot1 * j_right.transpose()
        const float lc = c1 * jc - s1 * (-js);
        const float ls = c1 * (-js) + s1 * jc;
        plane(W + 3 * p, W + 3 * q, 1, lc, ls);   // work.applyOnTheLeft(p, q, j_left)
        plane(U + p, U + q, 3, lc, ls);           // U.applyOnTheRight(p, q, j_left.transpose())
        plane(W + p, W + q, 3, jc, -js);          // work.applyOnTheRight(p, q, j_right)
        plane(V + p, V + q, 3, jc, -js);          // V.applyOnTheRight(p, q, j_right)
        maxDiag = std::max(maxDiag, std::max(std::fabs(W[3 * p + p]), std::fabs(W[3 * q + q])));
      }
  }
  for (int i = 0; i < 3; ++i) {
    const float a_ii = W[4 * i];
    sv[i] = std::fabs(a_ii);
    if (a_ii < 0.f) for (int r = 0; r < 3; ++r) U[3 * r + i] = -U[3 * r + i];
  }
  for (int i = 0; i < 3; ++i) sv[i] = sv[i] * scale;
  for (int i = 0; i < 3; ++i) {
    int pos = i;
    for (int j = i + 1; j < 3; ++j) if (sv[j] > sv[pos]) pos = j;
    if (sv[pos] == 0.f) break;
    if (pos != i) {
      std::swap(sv[i], sv[pos]);
      for (int r = 0; r < 3; ++r) { std::swap(U[3 * r + i], U[3 * r + pos]); std::swap(V[3 * r + i], V[3 * r + pos]); }
    }
  }
}

float det3(const float m[9]) {
  auto h = [&](int a, int b, int c) { return m[a] * (m[3 + b] * m[6 + c] - m[3 + c] * m[6 + b]); };
  return h(0, 1, 2) - h(1, 0, 2) + h(2, 0, 1);
}

// pcl::umeyama(src, dst, false) over the correspondence list (src_k = cur[q_k], dst_k = tgt[m_k]); T row-major 4x4
void umeyama(const std::vector<float>& s, const std::vector<float>& d, float T[16]) {
  const size_t n = s.size() / 3;
  const float one_over_n = 1.f / (float)n;
  float sm[3], dm[3];
  std::vector<float> col(n);
  for (int a = 0; a < 3; ++a) {
    for (size_t k = 0; k < n; ++k) col[k] = s[3 * k + a];
    sm[a] = hsum(col) * one_over_n;
    for (size_t k = 0; k < n; ++k) col[k] = d[3 * k + a];
    dm[a] = hsum(col) * one_over_n;
  }
  float sigma[9];
  for (int a = 0; a < 3; ++a)
    for (int b = 0; b < 3; ++b) {
      for (size_t k = 0; k < n; ++k) col[k] = (d[3 * k + a] - dm[a]) * (s[3 * k + b] - sm[b]);
      sigma[3 * a + b] = one_over_n * hsum(col);
    }
  float U[9], sv[3], V[9];
  svd3(sigma, U, sv, V);
  const float S2 = (det3(U) * det3(V) < 0.f) ? -1.f : 1.f;
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) T[4 * i + j] = ((U[3 * i] * 1.f) * V[3 * j] + (U[3 * i + 1] * 1.f) * V[3 * j + 1]) + (U[3 * i + 2] * S2) * V[3 * j + 2];
  for (int i = 0; i < 3; ++i) T[4 * i + 3] = ((dm[i] - T[4 * i] * sm[0]) - T[4 * i + 1] * sm[1]) - T[4 * i + 2] * sm[2];
  T[12] = 0.f; T[13] = 0.f; T[14] = 0.f; T[15] = 1.f;
}

inline void apply(const float T[16], const float* p, float* o) {
  const float x = p[0], y = p[1], z = p[2];
  o[0] = ((T[0] * x + T[1] * y) + T[2] * z) + T[3];
  o[1] = ((T[4] * x + T[5] * y) + T[6] * z) + T[7];
  o[2] = ((T[8] * x + T[9] * y) + T[10] * z) + T[11];
}

}  // namespace

extern "C" {

void go_lc_svd3(const float a[9], float U[9], float sv[3], float V[9]) { svd3(a, U, sv, V); }

/* pcl::umeyama(src, dst, false): src / dst n x 3 row-major (correspondence k = row k); T row-major 4x4 */
void go_lc_umeyama(const float* src, const float* dst, int64_t n, float T[16]) {
  std::vector<float> s(src, src + 3 * n), d(dst, dst + 3 * n);
  umeyama(s, d, T);
}

/* exact 1-NN (float L2_Simple, ties by index) of every query; idx -1 / dist +inf for an empty target */
void go_lc_nn(const float* tgt, int64_t m, const float* qry, int64_t nq, int32_t* idx, float* dist) {
  auto t = make_tree(tgt, m, 3);
  for (int64_t i = 0; i < nq; ++i) {
    float bd = INFINITY; int bi = -1;
    if (m > 0) t->search(0, qry + 3 * i, bd, bi);
    idx[i] = bi; dist[i] = bd;
  }
}

/* The hierarchical sums, exposed for the tests */
float go_lc_hsum_f(const float* v, int64_t n) { return hsum(std::vector<float>(v, v + n)); }
double go_lc_hsum_d(const double* v, int64_t n) { return hsum(std::vector<double>(v, v + n)); }

/* IterativeClosestPoint::align (identity guess) + getFitnessScore.  src n x 3, tgt m x 3.  aligned[3n], log[log_cap],
 * corr_q/m/d[corr_cap] (the last correspondence estimation) may be NULL. */
void go_lc_icp(const float* src, int64_t n, const float* tgt, int64_t m, int max_iterations, double max_corr_dist, double trans_eps,
               double fit_eps, go_icp_result* res, float* aligned, go_icp_iteration* log, int log_cap, int32_t* corr_q, int32_t* corr_m,
               float* corr_d, int64_t corr_cap) {
  go_icp_result R;
  std::memset(&R, 0, sizeof(R));
  float F[16] = {1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1};
  R.fitness = DBL_MAX;
  std::vector<float> cur(src, src + 3 * n);
  if (n == 0 || m == 0) {
    R.state = GO_ICP_NO_CORRESPONDENCES;
  } else {
    auto tree = make_tree(tgt, m, 3);
    const double max_dist_sqr = max_corr_dist * max_corr_dist;
    const double translation_threshold = trans_eps, rotation_threshold = 1.0 - trans_eps, mse_rel = fit_eps, mse_abs = 1e-12;
    double prev_mse = DBL_MAX;
    std::vector<int32_t> cq, cm; std::vector<float> cd;
    for (;;) {
      // determineCorrespondences: source order, 1-NN, rejected when distance > max_dist_sqr
      cq.clear(); cm.clear(); cd.clear();
      for (int64_t i = 0; i < n; ++i) {
        float bd = INFINITY; int bi = -1;
        tree->search(0, &cur[3 * i], bd, bi);
        if ((double)bd > max_dist_sqr) continue;
        cq.push_back((int32_t)i); cm.push_back(bi); cd.push_back(bd);
      }
      R.n_corr = (int64_t)cq.size();
      if (cq.size() < 3) { R.converged = 0; R.state = GO_ICP_NO_CORRESPONDENCES; break; }
      std::vector<float> s(3 * cq.size()), d(3 * cq.size());
      for (size_t k = 0; k < cq.size(); ++k) for (int a = 0; a < 3; ++a) { s[3 * k + a] = cur[3 * cq[k] + a]; d[3 * k + a] = tgt[3 * cm[k] + a]; }
      float T[16];
      umeyama(s, d, T);
      for (int64_t i = 0; i < n; ++i) { float o[3]; apply(T, &cur[3 * i], o); cur[3 * i] = o[0]; cur[3 * i + 1] = o[1]; cur[3 * i + 2] = o[2]; }
      float G[16];
      for (int i = 0; i < 4; ++i)
        for (int j = 0; j < 4; ++j) G[4 * i + j] = ((T[4 * i] * F[j] + T[4 * i + 1] * F[4 + j]) + T[4 * i + 2] * F[8 + j]) + T[4 * i + 3] * F[12 + j];
      std::memcpy(F, G, sizeof(F));
      const int it = R.iterations++;
      std::vector<double> dd(cd.begin(), cd.end());
      const double mse = hsum(dd) / (double)cd.size();
      if (log && it < log_cap) { std::memcpy(log[it].transformation, T, sizeof(T)); log[it].n_corr = (int64_t)cq.size(); log[it].mse = mse; }
      if (R.iterations >= max_iterations) { R.converged = 1; R.state = GO_ICP_ITERATIONS; break; }
      const double cos_angle = 0.5 * (double)(((T[0] + T[5]) + T[10]) - 1.f);
      const double translation_sqr = (double)((T[3] * T[3] + T[7] * T[7]) + T[11] * T[11]);
      if (cos_angle >= rotation_threshold && translation_sqr <= translation_threshold) { R.converged = 1; R.state = GO_ICP_TRANSFORM; break; }
      if (std::fabs(mse - prev_mse) < mse_abs) { R.converged = 1; R.state = GO_ICP_ABS_MSE; break; }
      if (std::fabs(mse - prev_mse) / prev_mse < mse_rel) { R.converged = 1; R.state = GO_ICP_REL_MSE; break; }
      prev_mse = mse;
    }
    const int64_t nc = std::min<int64_t>(corr_cap, (int64_t)cq.size());
    for (int64_t k = 0; k < nc; ++k) {
      if (corr_q) corr_q[k] = cq[k];
      if (corr_m) corr_m[k] = cm[k];
      if (corr_d) corr_d[k] = cd[k];
    }
    // getFitnessScore: the input transformed by final, 1-NN without gate, every point counts
    std::vector<double> fd((size_t)n);
    for (int64_t i = 0; i < n; ++i) {
      float o[3]; apply(F, src + 3 * i, o);
      float bd = INFINITY; int bi = -1;
      tree->search(0, o, bd, bi);
      fd[i] = (double)bd;
    }
    R.fitness = hsum(fd) / (double)n;
  }
  std::memcpy(R.final_T, F, sizeof(F));
  if (aligned) for (int64_t i = 0; i < n; ++i) apply(F, src + 3 * i, aligned + 3 * i);
  *res = R;
}

/* detectLoopClosure's candidate search (Estimator.cpp:5108-5127): pos[3K] float, times[K].  order[K] receives the radius-search result
 * (indices, by float distance then index), *n_found its length; returns closest_his_idx (-1: none passes the time test).  The 0.2 s
 * rule on time_last_loop is the caller's. */
int go_lc_detect(const float* pos, const double* times, int K, const float sel[3], double time_new_odom, double radius, double time_thres,
                 int32_t* order, int32_t* n_found) {
  const float r2 = (float)(radius * radius);
  std::vector<std::pair<float, int>> hits;
  for (int k = 0; k < K; ++k) {
    const float d = l2_simple(sel, pos + 3 * k);
    if (d < r2) hits.emplace_back(d, k);
  }
  std::sort(hits.begin(), hits.end());
  *n_found = (int32_t)hits.size();
  for (size_t i = 0; i < hits.size(); ++i) if (order) order[i] = hits[i].second;
  for (auto& h : hits) if (std::fabs(times[h.second] - time_new_odom) > time_thres) return h.second;
  return -1;
}

}  // extern "C"
