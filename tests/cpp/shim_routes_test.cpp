// shim_routes_test.cpp — the LiDAR routes of the Ceres-API shim beyond LidarPlaneNormFactor: LidarEdgeFactor blocks added the
// way Estimator.cpp:2091-2248 adds its LiDAR blocks ((t, q), HuberLoss), and LidarPlaneNormIncreFactor blocks added the way the
// front end's scan matcher does (LidarOdometry.cpp:499-530: (q, t), HuberLoss(0.1), LEVENBERG_MARQUARDT).  Used by
// tests/test_shim_routes.py and scripts/bench_shim_routes.py:
//   shim_routes_test host   [--repeat R] problem.bin...   every block evaluated on the host (no GPU needed)
//   shim_routes_test evaluate problem.bin...               Problem::Evaluate (host): cost and tangent gradient
//   shim_routes_test device [--repeat R] [--use-edges] [--preload-edges N] problem.bin...
//       the described blocks are routed to the GPU; all problems are solved in turn on ONE context (created with the first
//       problem's parameters), after glio_window_use_edges(ctx, 1) if asked.  One problem per call is a fresh context.
//       --preload-edges N first leaves what a direct (Level-2) caller would: N edges in every slot of the first problem through
//       glio_set_edges, sub-sampled by glio_select_random_edges, and prints their cost at that problem's poses (preload_cost).
// For each problem it prints the iterations, poses and costs (%.17g), the device block counts and the K2e launches of that solve.
// With --repeat R each problem is rebuilt from its file and solved R times, and each solve's wall time is printed.
//
// The functors are Eigen-free restatements of the two factors from their formulas (SURVEY a-6):
//   edge : r = s |(p - a) x (p - b)| / |a - b|,   p = q * (q_lb^-1 * (cp - t_lb)) + t
//   incre: r = n . (q * cp + t) + d
#include <algorithm>
#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <string>
#include <vector>

#include "ceres/ceres.h"
#include "ceres/rotation.h"
#include "shim_driver.h"

template <typename T> static void Rotate(const T q[4], const T v[3], T o[3]) {   // q v q^-1 for any q: v + 2w (u x v) + 2 u x (u x v)
  T uv[3] = {q[2] * v[2] - q[3] * v[1], q[3] * v[0] - q[1] * v[2], q[1] * v[1] - q[2] * v[0]};
  for (int k = 0; k < 3; ++k) uv[k] = uv[k] + uv[k];
  T uuv[3] = {q[2] * uv[2] - q[3] * uv[1], q[3] * uv[0] - q[1] * uv[2], q[1] * uv[1] - q[2] * uv[0]};
  for (int k = 0; k < 3; ++k) o[k] = v[k] + q[0] * uv[k] + uuv[k];
}
template <typename T> static T Norm3(const T v[3]) { return ceres::sqrt(v[0] * v[0] + v[1] * v[1] + v[2] * v[2]); }

struct LidarEdgeFactor {
  template <typename T> bool operator()(const T* t, const T* q, T* residual) const {
    const double n2 = qlb[0] * qlb[0] + qlb[1] * qlb[1] + qlb[2] * qlb[2] + qlb[3] * qlb[3];
    const T qi[4] = {T(qlb[0] / n2), T(-qlb[1] / n2), T(-qlb[2] / n2), T(-qlb[3] / n2)};
    T d[3], pl[3], p[3];
    for (int k = 0; k < 3; ++k) d[k] = T(curr_point[k]) - T(tlb[k]);
    Rotate(qi, d, pl); Rotate(q, pl, p);
    T pa[3], pb[3], ab[3];
    for (int k = 0; k < 3; ++k) { p[k] = p[k] + t[k]; pa[k] = p[k] - T(last_point_a[k]); pb[k] = p[k] - T(last_point_b[k]); ab[k] = T(last_point_a[k]) - T(last_point_b[k]); }
    const T c[3] = {pa[1] * pb[2] - pa[2] * pb[1], pa[2] * pb[0] - pa[0] * pb[2], pa[0] * pb[1] - pa[1] * pb[0]};
    residual[0] = Norm3(c) / Norm3(ab) * T(s);
    return true;
  }
  double curr_point[3], last_point_a[3], last_point_b[3], qlb[4], tlb[3], s;
};

struct LidarPlaneNormIncreFactor {
  template <typename T> bool operator()(const T* q, const T* t, T* residual) const {
    const T cp[3] = {T(curr_point[0]), T(curr_point[1]), T(curr_point[2])};
    T pw[3];
    Rotate(q, cp, pw);
    residual[0] = T(plane_unit_norm[0]) * (pw[0] + t[0]) + T(plane_unit_norm[1]) * (pw[1] + t[1]) + T(plane_unit_norm[2]) * (pw[2] + t[2]) +
                  T(negative_OA_dot_norm);
    return true;
  }
  double curr_point[3], plane_unit_norm[3], negative_OA_dot_norm;
};

// the unary plane factor of tests/cpp/shim_test.cpp, so one problem can hold all three unary kinds
struct LidarPlaneNormFactor {
  template <typename T> bool operator()(const T* t, const T* q, T* residual) const {
    const double n2 = qlb[0] * qlb[0] + qlb[1] * qlb[1] + qlb[2] * qlb[2] + qlb[3] * qlb[3];
    const T qi[4] = {T(qlb[0] / n2), T(-qlb[1] / n2), T(-qlb[2] / n2), T(-qlb[3] / n2)};
    T d[3], pl[3], pw[3];
    for (int k = 0; k < 3; ++k) d[k] = T(curr_point[k]) - T(tlb[k]);
    Rotate(qi, d, pl); Rotate(q, pl, pw);
    residual[0] = T(score) * (T(plane_unit_norm[0]) * (pw[0] + t[0]) + T(plane_unit_norm[1]) * (pw[1] + t[1]) + T(plane_unit_norm[2]) * (pw[2] + t[2]) +
                              T(negative_OA_dot_norm));
    return true;
  }
  double curr_point[3], plane_unit_norm[3], qlb[4], tlb[3], negative_OA_dot_norm, score;
};

// and its binary plane factor, so the problems of tests/test_shim.py can be rebuilt here
struct BinaryLidarPlaneNormFactor {
  template <typename T> bool operator()(const T* t1, const T* q1, const T* t2, const T* q2, T* residual) const {
    const T cp[3] = {T(curr_point[0]), T(curr_point[1]), T(curr_point[2])};
    const T nl[3] = {T(planet_norm_cent[0]), T(planet_norm_cent[1]), T(planet_norm_cent[2])}, cl[3] = {T(planet_norm_cent[3]), T(planet_norm_cent[4]), T(planet_norm_cent[5])};
    T pw[3], no[3], co[3];
    Rotate(q1, cp, pw); Rotate(q2, nl, no); Rotate(q2, cl, co);
    for (int k = 0; k < 3; ++k) { pw[k] = pw[k] + t1[k]; co[k] = co[k] + t2[k]; }
    residual[0] = T(score) * (no[0] * (pw[0] - co[0]) + no[1] * (pw[1] - co[1]) + no[2] * (pw[2] - co[2]));
    return true;
  }
  double curr_point[3], planet_norm_cent[6], score;
};

// what a maintainer adds next to the reference's functors (INTEGRATION.md, Level 1)
namespace glio {
template <> struct DeviceFactorTraits<LidarEdgeFactor> {
  static bool describe(const LidarEdgeFactor& f, FactorDesc* d) {
    d->kind = FACTOR_EDGE_UNARY;
    for (int k = 0; k < 3; ++k) { d->cp[k] = f.curr_point[k]; d->pa[k] = f.last_point_a[k]; d->pb[k] = f.last_point_b[k]; d->t_lb[k] = f.tlb[k]; }
    for (int k = 0; k < 4; ++k) d->q_lb[k] = f.qlb[k];
    d->score = f.s;
    return true;
  }
};
template <> struct DeviceFactorTraits<LidarPlaneNormIncreFactor> {
  static bool describe(const LidarPlaneNormIncreFactor& f, FactorDesc* d) {
    d->kind = FACTOR_PLANE_INCRE;
    for (int k = 0; k < 3; ++k) { d->cp[k] = f.curr_point[k]; d->n[k] = f.plane_unit_norm[k]; }
    d->d = f.negative_OA_dot_norm;
    return true;
  }
};
template <> struct DeviceFactorTraits<BinaryLidarPlaneNormFactor> {
  static bool describe(const BinaryLidarPlaneNormFactor& f, FactorDesc* d) {
    d->kind = FACTOR_PLANE_BINARY;
    for (int k = 0; k < 3; ++k) d->cp[k] = f.curr_point[k];
    for (int k = 0; k < 6; ++k) d->nc[k] = f.planet_norm_cent[k];
    d->score = f.score;
    return true;
  }
};
template <> struct DeviceFactorTraits<LidarPlaneNormFactor> {
  static bool describe(const LidarPlaneNormFactor& f, FactorDesc* d) {
    d->kind = FACTOR_PLANE_UNARY;
    for (int k = 0; k < 3; ++k) { d->cp[k] = f.curr_point[k]; d->n[k] = f.plane_unit_norm[k]; d->t_lb[k] = f.tlb[k]; }
    for (int k = 0; k < 4; ++k) d->q_lb[k] = f.qlb[k];
    d->d = f.negative_OA_dot_norm; d->score = f.score;
    return true;
  }
};
}  // namespace glio

// stand-ins for the host factors, the same functions as tests/cpp/shim_test.cpp's
struct PriorF {
  double t0[3], q0[4], sb0[9], sw[15];
  template <typename T> bool operator()(const T* t, const T* q, const T* sb, T* r) const {
    for (int k = 0; k < 3; ++k) r[k] = T(sw[k]) * (t[k] - T(t0[k]));
    T q0c[4] = {T(q0[0]), T(-q0[1]), T(-q0[2]), T(-q0[3])}, e[4];
    ceres::QuaternionProduct(q0c, q, e);
    for (int k = 0; k < 3; ++k) r[3 + k] = T(sw[3 + k]) * (T(2.0) * e[1 + k]);
    for (int k = 0; k < 9; ++k) r[6 + k] = T(sw[6 + k]) * (sb[k] - T(sb0[k]));
    return true;
  }
};
struct BetweenF {
  double dp[3], dq[4], dv[3], dt, sw[15];
  template <typename T> bool operator()(const T* ti, const T* qi, const T* si, const T* tj, const T* qj, const T* sj, T* r) const {
    T qic[4] = {qi[0], -qi[1], -qi[2], -qi[3]};
    T d[3] = {tj[0] - ti[0] - si[0] * T(dt), tj[1] - ti[1] - si[1] * T(dt), tj[2] - ti[2] - si[2] * T(dt)}, rp[3];
    Rotate(qic, d, rp);
    for (int k = 0; k < 3; ++k) r[k] = T(sw[k]) * (rp[k] - T(dp[k]));
    T dqc[4] = {T(dq[0]), T(-dq[1]), T(-dq[2]), T(-dq[3])}, qij[4], e[4];
    ceres::QuaternionProduct(qic, qj, qij); ceres::QuaternionProduct(dqc, qij, e);
    for (int k = 0; k < 3; ++k) r[3 + k] = T(sw[3 + k]) * (T(2.0) * e[1 + k]);
    T dvv[3] = {sj[0] - si[0], sj[1] - si[1], sj[2] - si[2]}, rv[3];
    Rotate(qic, dvv, rv);
    for (int k = 0; k < 3; ++k) r[6 + k] = T(sw[6 + k]) * (rv[k] - T(dv[k]));
    for (int k = 0; k < 6; ++k) r[9 + k] = T(sw[9 + k]) * (sj[3 + k] - si[3 + k]);
    return true;
  }
};
struct RangeF {
  double lever[3], sat[3], rho, w;
  template <typename T> bool operator()(const T* t, const T* q, T* r) const {
    T lv[3] = {T(lever[0]), T(lever[1]), T(lever[2])}, pw[3];
    Rotate(q, lv, pw);
    T d[3] = {pw[0] + t[0] - T(sat[0]), pw[1] + t[1] - T(sat[1]), pw[2] + t[2] - T(sat[2])};
    r[0] = T(w) * (ceres::sqrt(d[0] * d[0] + d[1] * d[1] + d[2] * d[2]) - T(rho));
    return true;
  }
};

// one problem file (written by tests/test_shim_routes.py: write_problem)
struct Spec {
  int32_t W = 0, use_sb = 0;
  std::vector<double> poses, sb;
  double q_lb[4], t_lb[3], lidar_const, huber;
  int32_t unit_score = 0;
  std::vector<int32_t> t_param, q_const;            // per keyframe: t with an IdentityParameterization, q constant
  // kind (glio::FactorKind), keyframe, other keyframe (binary), then cp[3] a[3] b[3] d s q_lb[4] t_lb[3] loss (< 0: none, else
  // Huber delta).  plane / incre: a = n; edge: a, b = the line's points; binary: a = local normal, b = centroid
  struct Lidar { int32_t kind, kf, kf2; double v[19]; };
  std::vector<Lidar> lidar;
  std::vector<std::pair<int32_t, PriorF>> priors;
  struct Between { int32_t i, j; BetweenF f; };
  std::vector<Between> betweens;
  std::vector<std::pair<int32_t, RangeF>> ranges;
  int32_t strategy = 0, max_iter = 15;              // strategy 1: LEVENBERG_MARQUARDT (then DENSE_QR), 0: DOGLEG
  double time_limit = 1e9;
};

static Spec read_spec(const char* path) {
  FILE* f = fopen(path, "rb");
  if (!f) { fprintf(stderr, "cannot open %s\n", path); exit(2); }
  Spec s;
  rd(f, &s.W, 1); rd(f, &s.use_sb, 1);
  s.poses.resize(7 * (size_t)s.W); s.sb.resize(9 * (size_t)s.W);
  rd(f, s.poses.data(), s.poses.size()); rd(f, s.sb.data(), s.sb.size());
  rd(f, s.q_lb, 4); rd(f, s.t_lb, 3); rd(f, &s.lidar_const, 1); rd(f, &s.huber, 1); rd(f, &s.unit_score, 1);
  s.t_param.resize(s.W); s.q_const.resize(s.W);
  rd(f, s.t_param.data(), s.W); rd(f, s.q_const.data(), s.W);
  int32_t n; rd(f, &n, 1);
  s.lidar.resize(n);
  for (auto& l : s.lidar) { rd(f, &l.kind, 1); rd(f, &l.kf, 1); rd(f, &l.kf2, 1); rd(f, l.v, 19); }
  rd(f, &n, 1);
  for (int i = 0; i < n; ++i) { int32_t k; PriorF p; rd(f, &k, 1); rd(f, p.t0, 3); rd(f, p.q0, 4); rd(f, p.sb0, 9); rd(f, p.sw, 15); s.priors.push_back({k, p}); }
  rd(f, &n, 1);
  for (int i = 0; i < n; ++i) { Spec::Between b; rd(f, &b.i, 1); rd(f, &b.j, 1); rd(f, b.f.dp, 3); rd(f, b.f.dq, 4); rd(f, b.f.dv, 3); rd(f, &b.f.dt, 1); rd(f, b.f.sw, 15); s.betweens.push_back(b); }
  rd(f, &n, 1);
  for (int i = 0; i < n; ++i) { int32_t k; RangeF r; rd(f, &k, 1); rd(f, r.lever, 3); rd(f, r.sat, 3); rd(f, &r.rho, 1); rd(f, &r.w, 1); s.ranges.push_back({k, r}); }
  rd(f, &s.strategy, 1); rd(f, &s.max_iter, 1); rd(f, &s.time_limit, 1);
  fclose(f);
  return s;
}

struct Result { ceres::Solver::Summary summary; std::vector<double> t, q, sb, gradient; double wall_ms = 0, cost = 0; };

// builds the problem at the file's state; evaluate_only: Problem::Evaluate instead of ceres::Solve
static Result solve(const Spec& s, glio_ctx* ctx, bool evaluate_only = false) {
  Result R;
  const int W = s.W;
  R.t.resize(3 * (size_t)W); R.q.resize(4 * (size_t)W); R.sb = s.sb;
  for (int k = 0; k < W; ++k) {
    for (int i = 0; i < 3; ++i) R.t[3 * k + i] = s.poses[7 * k + i];
    for (int i = 0; i < 4; ++i) R.q[4 * k + i] = s.poses[7 * k + 3 + i];
  }
  double* t = R.t.data(); double* q = R.q.data(); double* sb = R.sb.data();
  ceres::Problem::Options po;
  po.loss_function_ownership = ceres::DO_NOT_TAKE_OWNERSHIP;
  std::vector<std::unique_ptr<ceres::LossFunction>> losses;
  auto loss_for = [&](double delta) -> ceres::LossFunction* {
    if (delta < 0) return nullptr;
    losses.emplace_back(new ceres::HuberLoss(delta));
    return losses.back().get();
  };
  ceres::Problem problem(po);
  problem.SetGlioContext(ctx);
  for (int k = 0; k < W; ++k) {                     // Estimator.cpp:2130-2137; the front end adds q first (LidarOdometry.cpp:503-504)
    if (s.strategy == 1) {
      problem.AddParameterBlock(q + 4 * k, 4, new ceres::QuaternionParameterization());
      problem.AddParameterBlock(t + 3 * k, 3, s.t_param[k] ? new ceres::IdentityParameterization(3) : nullptr);
    } else {
      problem.AddParameterBlock(t + 3 * k, 3, s.t_param[k] ? new ceres::IdentityParameterization(3) : nullptr);
      problem.AddParameterBlock(q + 4 * k, 4, new ceres::QuaternionParameterization());
    }
    if (s.use_sb) problem.AddParameterBlock(sb + 9 * k, 9);
    if (s.q_const[k]) problem.SetParameterBlockConstant(q + 4 * k);
  }
  // one HuberLoss object per distinct delta, shared by the blocks as in the reference
  std::map<double, ceres::LossFunction*> loss_of;
  for (const Spec::Lidar& l : s.lidar) {
    const double* v = l.v;
    ceres::LossFunction* loss = nullptr;
    if (v[18] >= 0) { auto it = loss_of.find(v[18]); loss = it != loss_of.end() ? it->second : (loss_of[v[18]] = loss_for(v[18])); }
    double* tk = t + 3 * l.kf; double* qk = q + 4 * l.kf;
    if (l.kind == glio::FACTOR_EDGE_UNARY) {
      LidarEdgeFactor* e = new LidarEdgeFactor();
      for (int k = 0; k < 3; ++k) { e->curr_point[k] = v[k]; e->last_point_a[k] = v[3 + k]; e->last_point_b[k] = v[6 + k]; e->tlb[k] = v[15 + k]; }
      for (int k = 0; k < 4; ++k) e->qlb[k] = v[11 + k];
      e->s = v[10];
      problem.AddResidualBlock(new ceres::AutoDiffCostFunction<LidarEdgeFactor, 1, 3, 4>(e), loss, tk, qk);
    } else if (l.kind == glio::FACTOR_PLANE_INCRE) {
      LidarPlaneNormIncreFactor* f = new LidarPlaneNormIncreFactor();
      for (int k = 0; k < 3; ++k) { f->curr_point[k] = v[k]; f->plane_unit_norm[k] = v[3 + k]; }
      f->negative_OA_dot_norm = v[9];
      problem.AddResidualBlock(new ceres::AutoDiffCostFunction<LidarPlaneNormIncreFactor, 1, 4, 3>(f), loss, qk, tk);   // LidarOdometry.cpp:518
    } else if (l.kind == glio::FACTOR_PLANE_BINARY) {
      BinaryLidarPlaneNormFactor* f = new BinaryLidarPlaneNormFactor();
      for (int k = 0; k < 3; ++k) { f->curr_point[k] = v[k]; f->planet_norm_cent[k] = v[3 + k]; f->planet_norm_cent[3 + k] = v[6 + k]; }
      f->score = v[10];
      problem.AddResidualBlock(new ceres::AutoDiffCostFunction<BinaryLidarPlaneNormFactor, 1, 3, 4, 3, 4>(f), loss, tk, qk, t + 3 * l.kf2, q + 4 * l.kf2);
    } else {
      LidarPlaneNormFactor* f = new LidarPlaneNormFactor();
      for (int k = 0; k < 3; ++k) { f->curr_point[k] = v[k]; f->plane_unit_norm[k] = v[3 + k]; f->tlb[k] = v[15 + k]; }
      for (int k = 0; k < 4; ++k) f->qlb[k] = v[11 + k];
      f->negative_OA_dot_norm = v[9]; f->score = v[10];
      problem.AddResidualBlock(new ceres::AutoDiffCostFunction<LidarPlaneNormFactor, 1, 3, 4>(f), loss, tk, qk);
    }
  }
  for (auto& p : s.priors)
    problem.AddResidualBlock(new ceres::AutoDiffCostFunction<PriorF, 15, 3, 4, 9>(new PriorF(p.second)), nullptr, t + 3 * p.first, q + 4 * p.first, sb + 9 * p.first);
  for (auto& b : s.betweens)
    problem.AddResidualBlock(new ceres::AutoDiffCostFunction<BetweenF, 15, 3, 4, 9, 3, 4, 9>(new BetweenF(b.f)), nullptr,
                             std::vector<double*>{t + 3 * b.i, q + 4 * b.i, sb + 9 * b.i, t + 3 * b.j, q + 4 * b.j, sb + 9 * b.j});
  for (auto& r : s.ranges)
    problem.AddResidualBlock(new ceres::AutoDiffCostFunction<RangeF, 1, 3, 4>(new RangeF(r.second)), nullptr, t + 3 * r.first, q + 4 * r.first);
  if (evaluate_only) {
    problem.Evaluate(ceres::Problem::EvaluateOptions(), &R.cost, nullptr, &R.gradient, nullptr);
    return R;
  }
  ceres::Solver::Options options;
  if (s.strategy == 1) {                            // LidarOdometry.cpp:521-530
    options.linear_solver_type = ceres::DENSE_QR;
    options.trust_region_strategy_type = ceres::LEVENBERG_MARQUARDT;
  } else {                                          // Estimator.cpp:2424-2430
    options.linear_solver_type = ceres::SPARSE_NORMAL_CHOLESKY;
    options.trust_region_strategy_type = ceres::DOGLEG;
  }
  options.max_num_iterations = s.max_iter;
  options.max_solver_time_in_seconds = s.time_limit;
  options.minimizer_progress_to_stdout = false;
  const auto t0 = std::chrono::steady_clock::now();
  ceres::Solve(options, &problem, &R.summary);
  R.wall_ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
  return R;
}

static int64_t edge_launches(glio_ctx* ctx) { return launches(ctx, {"k_eval_edge", "k_eval_edge_cost"}); }

int main(int argc, char** argv) {
  if (argc < 3) { fprintf(stderr, "usage: shim_routes_test host|device|evaluate [--repeat R] [--use-edges] [--preload-edges N] problem.bin...\n"); return 2; }
  const bool device = std::string(argv[1]) == "device", evaluate = std::string(argv[1]) == "evaluate";
  int repeat = 0, preload = 0; bool use_edges = false;
  std::vector<const char*> files;
  for (int i = 2; i < argc; ++i) {
    const std::string a = argv[i];
    if (a == "--repeat" && i + 1 < argc) repeat = atoi(argv[++i]);
    else if (a == "--use-edges") use_edges = true;
    else if (a == "--preload-edges" && i + 1 < argc) preload = atoi(argv[++i]);
    else files.push_back(argv[i]);
  }
  if (files.empty()) return 2;
  glio_ctx* ctx = nullptr;
  if (device) {
    const Spec s0 = read_spec(files[0]);
    glio_params prm; glio_default_params(&prm);
    for (int k = 0; k < 4; ++k) prm.q_lb[k] = s0.q_lb[k];
    for (int k = 0; k < 3; ++k) prm.t_lb[k] = s0.t_lb[k];
    prm.lidar_const = s0.lidar_const; prm.huber_delta = s0.huber; prm.unit_score = s0.unit_score;
    ctx = create_context(prm, !repeat);
    if (use_edges && glio_window_use_edges(ctx, 1) != GLIO_OK) return 3;
    if (preload > 0) {
      // points 1 m off the x axis, against the x axis as the line: every edge has a residual at any pose near the identity
      std::vector<float> cp(3 * (size_t)preload), pa(3 * (size_t)preload, 0.f), pb(3 * (size_t)preload, 0.f);
      std::vector<double> sc(preload, 1.0);
      for (int i = 0; i < preload; ++i) { cp[3 * i] = 0.01f * (float)i; cp[3 * i + 1] = 1.f; cp[3 * i + 2] = 2.f; pb[3 * i] = 1.f; }
      std::vector<int64_t> streams(s0.W);
      for (int k = 0; k < s0.W; ++k) {
        streams[k] = k;
        if (glio_set_edges(ctx, k, cp.data(), pa.data(), pb.data(), sc.data(), preload) != GLIO_OK) return 3;
      }
      glio_select_options so; glio_select_default_options(&so);
      if (glio_select_random_edges(ctx, s0.W, streams.data(), &so, nullptr) != GLIO_OK) return 3;
      std::vector<double> cost(s0.W);
      if (glio_eval_edge(ctx, s0.W, s0.poses.data(), nullptr, nullptr, cost.data()) != GLIO_OK) return 3;
      double tot = 0; for (double c : cost) tot += c;
      printf("preload_cost %.17g\n", tot);
    }
  }
  for (size_t fi = 0; fi < files.size(); ++fi) {
    const Spec s = read_spec(files[fi]);
    printf("solve %d\n", (int)fi);
    if (evaluate) {
      const Result R = solve(s, nullptr, true);
      printf("eval_cost %.17g\n", R.cost);
      printf("gradient"); for (double v : R.gradient) printf(" %.17g", v); printf("\n");
      continue;
    }
    if (repeat) {
      for (int r = 0; r < repeat; ++r) {
        const Result R = solve(s, ctx);
        printf("time %.6f %d\n", R.wall_ms, (int)R.summary.iterations.size());
      }
      continue;
    }
    const int64_t e0 = edge_launches(ctx);
    const Result R = solve(s, ctx);
    const int64_t e1 = edge_launches(ctx);
    const ceres::Solver::Summary& S = R.summary;
    const int dev_edges = S.num_device_edge_residual_blocks;
    print_solve_head(S);
    printf("device_blocks %d\n", S.num_device_residual_blocks);
    printf("device_kinds %d %d\n", S.num_device_residual_blocks - dev_edges, dev_edges);
    printf("edge_launches %lld\n", (long long)(e1 - e0));
    print_solve_tail(S, s.W, R.t, R.q, &R.sb);
  }
  if (ctx) glio_destroy(ctx);
  return 0;
}
