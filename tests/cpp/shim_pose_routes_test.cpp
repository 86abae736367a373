// shim_pose_routes_test.cpp — the Ceres-API shim's route for the batch refinement's pose factors (K2p):
// LidarPoseFactorBatchRelativeAutoDiff and delta_q_factor_auto blocks added the way optimizeBatchWithLandMark adds them
// (Estimator.cpp:2783-2954: receiver-clock blocks, then per keyframe t, q (QuaternionParameterization) and speed-bias, a
// constant yaw and anchor, the attitude factors, the clock-drift block, the relative factors).  Used by
// tests/test_shim_pose_routes.py and scripts/bench_shim_pose_routes.py:
//   shim_pose_routes_test host   [--repeat R] [--max-iter M] problem.bin...   every block evaluated on the host (no GPU needed)
//   shim_pose_routes_test evaluate problem.bin...                              Problem::Evaluate (host): cost and tangent gradient
//   shim_pose_routes_test describe problem.bin...                              each pose block's trait description, in hex
//   shim_pose_routes_test device [--repeat R] [--max-iter M] [--use-pose] [--preload-pose N] problem.bin...
//       the described blocks are routed to the GPU; all problems are solved in turn on ONE context, after
//       glio_batch_use_pose_factors(ctx, 1) if asked.  One problem per call is a fresh context.  --preload-pose N first leaves
//       what a direct (Level-2) caller would: a list of N other pose factors (glio_batch_set_pose_factors) and the switch on.
// For each problem it prints the iterations, poses and costs (%.17g), the device block counts and the K2p launches of that solve.
// With --repeat R each problem is rebuilt from its file and solved R times, and each solve's wall time is printed.
//
// The functors are Eigen-free restatements of the reference's from their formulas, with Eigen's semantics at any quaternion
// (inverse() = conj / |q|^2, q * v = v + 2w (u x v) + 2 u x (u x v), products left to right):
//   relative: r[0..2] = 10 (2 vec(dq^-1 q_i^-1 q_j)),  r[3..5] = 20 (q_i^-1 (t_j - t_i) - dp)
//   delta_q : r = 10000 vec(dq^-1 q_i^-1 q_j)
// LidarPoseFactorBatchRelativeAutoDiff keeps delta_q and delta_p private, as the reference does (LidarPoseFactor.h:92-94), so
// its trait reads them the way INTEGRATION.md shows: through pointers to members named in an explicit instantiation.
#include <algorithm>
#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <string>
#include <vector>

#include "ceres/ceres.h"
#include "ceres/rotation.h"
#include "shim_driver.h"

// the parts of Eigen::Quaterniond / Eigen::Vector3d the factors and their traits use
struct Quaterniond {
  double c[4];   // w, x, y, z
  double w() const { return c[0]; } double x() const { return c[1]; } double y() const { return c[2]; } double z() const { return c[3]; }
};
struct Vector3d {
  double c[3];
  double operator[](int k) const { return c[k]; }
  double x() const { return c[0]; } double y() const { return c[1]; } double z() const { return c[2]; }
};

template <typename T> static void QMul(const T a[4], const T b[4], T o[4]) {   // Eigen's product, (w, x, y, z)
  o[0] = a[0] * b[0] - a[1] * b[1] - a[2] * b[2] - a[3] * b[3];
  o[1] = a[0] * b[1] + a[1] * b[0] + a[2] * b[3] - a[3] * b[2];
  o[2] = a[0] * b[2] + a[2] * b[0] + a[3] * b[1] - a[1] * b[3];
  o[3] = a[0] * b[3] + a[3] * b[0] + a[1] * b[2] - a[2] * b[1];
}
template <typename T> static void QInv(const T q[4], T o[4]) {
  const T n2 = q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3];
  o[0] = q[0] / n2; o[1] = -q[1] / n2; o[2] = -q[2] / n2; o[3] = -q[3] / n2;
}
template <typename T> static void Rotate(const T q[4], const T v[3], T o[3]) {
  T uv[3] = {q[2] * v[2] - q[3] * v[1], q[3] * v[0] - q[1] * v[2], q[1] * v[1] - q[2] * v[0]};
  for (int k = 0; k < 3; ++k) uv[k] = uv[k] + uv[k];
  T uuv[3] = {q[2] * uv[2] - q[3] * uv[1], q[3] * uv[0] - q[1] * uv[2], q[1] * uv[1] - q[2] * uv[0]};
  for (int k = 0; k < 3; ++k) o[k] = v[k] + q[0] * uv[k] + uuv[k];
}
// w_rot (2 vec(dq^-1 q_i^-1 q_j)) and w_pos (q_i^-1 (t_j - t_i) - dp) of the reference's pose functors
template <typename T> static void PoseResidual(const Quaterniond& dq, const Vector3d& dp, double w_rot, double w_pos, const T* p1,
                                               const T* q1, const T* p2, const T* q2, T* r) {
  const T dqv[4] = {T(dq.w()), T(dq.x()), T(dq.y()), T(dq.z())};
  T dqi[4], q1i[4], a[4], e[4];
  QInv(dqv, dqi); QInv(q1, q1i); QMul(dqi, q1i, a); QMul(a, q2, e);
  const T d[3] = {p2[0] - p1[0], p2[1] - p1[1], p2[2] - p1[2]};
  T b[3];
  Rotate(q1i, d, b);
  for (int k = 0; k < 3; ++k) r[k] = T(w_rot) * (T(2.0) * e[1 + k]);
  for (int k = 0; k < 3; ++k) r[3 + k] = T(w_pos) * (b[k] - T(dp[k]));
}

struct LidarPoseFactorBatchRelativeAutoDiff {
 public:
  LidarPoseFactorBatchRelativeAutoDiff(Quaterniond delta_q_, Vector3d delta_p_) : delta_q(delta_q_), delta_p(delta_p_) {}
  template <typename T> bool operator()(const T* p1, const T* p2, const T* p3, const T* p4, T* residuals) const {
    PoseResidual(delta_q, delta_p, 10.0, 20.0, p1, p2, p3, p4, residuals);
    return true;
  }
  static ceres::CostFunction* Create(Quaterniond delta_q_, Vector3d delta_p_) {
    return new ceres::AutoDiffCostFunction<LidarPoseFactorBatchRelativeAutoDiff, 6, 3, 4, 3, 4>(new LidarPoseFactorBatchRelativeAutoDiff(delta_q_, delta_p_));
  }

 private:
  Quaterniond delta_q;
  Vector3d delta_p;
};

// the optimizeLocalGraph factor (LidarPoseFactor.h:11-52): the same blocks and formula with the weights 0.2; it has no trait,
// so its blocks stay on the host
struct LidarPoseFactorAutoDiff {
 public:
  LidarPoseFactorAutoDiff(Quaterniond delta_q_, Vector3d delta_p_) : delta_q(delta_q_), delta_p(delta_p_) {}
  template <typename T> bool operator()(const T* p1, const T* p2, const T* p3, const T* p4, T* residuals) const {
    PoseResidual(delta_q, delta_p, 0.2, 0.2, p1, p2, p3, p4, residuals);
    return true;
  }

 private:
  Quaterniond delta_q;
  Vector3d delta_p;
};

struct delta_q_factor_auto {
  delta_q_factor_auto(const Quaterniond& delta_q) : delta_q(delta_q) {}
  template <typename T> bool operator()(const T* quat_i, const T* quat_j, T* residuals) const {
    const T dqv[4] = {T(delta_q.w()), T(delta_q.x()), T(delta_q.y()), T(delta_q.z())};
    T dqi[4], qii[4], a[4], e[4];
    QInv(dqv, dqi); QInv(quat_i, qii); QMul(dqi, qii, a); QMul(a, quat_j, e);
    for (int k = 0; k < 3; ++k) residuals[k] = T(10000) * e[1 + k];
    return true;
  }
  Quaterniond delta_q;
};

// ---- what a maintainer adds next to the reference's functors (INTEGRATION.md, Level 1) ----
// Access checks do not apply to the names in an explicit instantiation, so instantiating PoseFactorMember with
// &LidarPoseFactorBatchRelativeAutoDiff::delta_q defines the friend member_ptr(RelDeltaQ), which returns that pointer.
template <class Tag, typename Tag::type Member> struct PoseFactorMember { friend typename Tag::type member_ptr(Tag) { return Member; } };
struct RelDeltaQ { typedef Quaterniond LidarPoseFactorBatchRelativeAutoDiff::*type; friend type member_ptr(RelDeltaQ); };
struct RelDeltaP { typedef Vector3d LidarPoseFactorBatchRelativeAutoDiff::*type; friend type member_ptr(RelDeltaP); };
template struct PoseFactorMember<RelDeltaQ, &LidarPoseFactorBatchRelativeAutoDiff::delta_q>;
template struct PoseFactorMember<RelDeltaP, &LidarPoseFactorBatchRelativeAutoDiff::delta_p>;

namespace glio {
template <> struct DeviceFactorTraits<LidarPoseFactorBatchRelativeAutoDiff> {
  static bool describe(const LidarPoseFactorBatchRelativeAutoDiff& f, FactorDesc* d) {
    const Quaterniond& q = f.*member_ptr(RelDeltaQ());
    const Vector3d& p = f.*member_ptr(RelDeltaP());
    d->kind = FACTOR_POSE_RELATIVE;
    d->dq[0] = q.w(); d->dq[1] = q.x(); d->dq[2] = q.y(); d->dq[3] = q.z();
    for (int k = 0; k < 3; ++k) d->dp[k] = p[k];
    return true;
  }
};
template <> struct DeviceFactorTraits<delta_q_factor_auto> {
  static bool describe(const delta_q_factor_auto& f, FactorDesc* d) {
    d->kind = FACTOR_POSE_DELTA_Q;
    d->dq[0] = f.delta_q.w(); d->dq[1] = f.delta_q.x(); d->dq[2] = f.delta_q.y(); d->dq[3] = f.delta_q.z();
    return true;
  }
};
}  // namespace glio

// the binary plane factor of tests/cpp/shim_routes_test.cpp, with its trait
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
namespace glio {
template <> struct DeviceFactorTraits<BinaryLidarPlaneNormFactor> {
  static bool describe(const BinaryLidarPlaneNormFactor& f, FactorDesc* d) {
    d->kind = FACTOR_PLANE_BINARY;
    for (int k = 0; k < 3; ++k) d->cp[k] = f.curr_point[k];
    for (int k = 0; k < 6; ++k) d->nc[k] = f.planet_norm_cent[k];
    d->score = f.score;
    return true;
  }
};
}  // namespace glio

// host stand-ins: the prior and IMU-like between factor of tests/cpp/shim_routes_test.cpp (glio_hf_add_prior / _add_between),
// and a pseudorange-like factor with dd_psr_factor_20's block shape [t_i, t_j, yaw, anchor]: per keyframe the range difference
// to two satellites placed at anchor + Rz(yaw) s
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
struct DDF {
  double s1[3], s2[3], rho_i, rho_j, w;
  template <typename T> bool operator()(const T* ti, const T* tj, const T* yaw, const T* anc, T* r) const {
    const T c = ceres::cos(yaw[0]), s = ceres::sin(yaw[0]);
    T a[3], b[3];
    a[0] = anc[0] + c * T(s1[0]) - s * T(s1[1]); a[1] = anc[1] + s * T(s1[0]) + c * T(s1[1]); a[2] = anc[2] + T(s1[2]);
    b[0] = anc[0] + c * T(s2[0]) - s * T(s2[1]); b[1] = anc[1] + s * T(s2[0]) + c * T(s2[1]); b[2] = anc[2] + T(s2[2]);
    auto dist = [](const T* p, const T* q) { return ceres::sqrt((p[0] - q[0]) * (p[0] - q[0]) + (p[1] - q[1]) * (p[1] - q[1]) + (p[2] - q[2]) * (p[2] - q[2])); };
    r[0] = T(w) * (dist(ti, a) - dist(ti, b) - T(rho_i));
    r[1] = T(w) * (dist(tj, a) - dist(tj, b) - T(rho_j));
    return true;
  }
};

// one problem file (written by tests/test_shim_pose_routes.py: write_problem)
struct Spec {
  int32_t K = 0, n_rcv = 0, epoch = 0;
  std::vector<double> poses, sb, alt_t;
  double yaw = 0, anchor[3] = {0, 0, 0};
  std::vector<int32_t> t_param, q_const, q_ident;   // per keyframe: t with an IdentityParameterization, q constant, q with
                                                    // IdentityParameterization(4) instead of QuaternionParameterization
  // kind 0 relative, 1 delta_q, 2 LidarPoseFactorAutoDiff; alt >= 0: t_i is extra t block alt; loss < 0: none, else Huber delta
  struct Pose { int32_t kind, i, j, alt; double dq[4], dp[3], loss; };
  std::vector<Pose> pose;
  struct Bin { int32_t kc, ko; double cp[3], nc[6], score; };
  std::vector<Bin> bin;
  std::vector<std::pair<int32_t, PriorF>> priors;
  struct Between { int32_t i, j; BetweenF f; };
  std::vector<Between> betweens;
  struct DD { int32_t i, j; DDF f; };
  std::vector<DD> dds;
  int32_t max_iter = 10;
  double time_limit = 1e9;
};

static Spec read_spec(const char* path) {
  FILE* f = fopen(path, "rb");
  if (!f) { fprintf(stderr, "cannot open %s\n", path); exit(2); }
  Spec s;
  rd(f, &s.K, 1); rd(f, &s.n_rcv, 1); rd(f, &s.epoch, 1);
  s.poses.resize(7 * (size_t)s.K); s.sb.resize(9 * (size_t)s.K);
  rd(f, s.poses.data(), s.poses.size()); rd(f, s.sb.data(), s.sb.size());
  rd(f, &s.yaw, 1); rd(f, s.anchor, 3);
  s.t_param.resize(s.K); s.q_const.resize(s.K); s.q_ident.resize(s.K);
  rd(f, s.t_param.data(), s.K); rd(f, s.q_const.data(), s.K); rd(f, s.q_ident.data(), s.K);
  int32_t n;
  rd(f, &n, 1); s.pose.resize(n);
  for (auto& p : s.pose) { rd(f, &p.kind, 1); rd(f, &p.i, 1); rd(f, &p.j, 1); rd(f, &p.alt, 1); rd(f, p.dq, 4); rd(f, p.dp, 3); rd(f, &p.loss, 1); }
  rd(f, &n, 1); s.alt_t.resize(3 * (size_t)n); rd(f, s.alt_t.data(), s.alt_t.size());
  rd(f, &n, 1); s.bin.resize(n);
  for (auto& b : s.bin) { rd(f, &b.kc, 1); rd(f, &b.ko, 1); rd(f, b.cp, 3); rd(f, b.nc, 6); rd(f, &b.score, 1); }
  rd(f, &n, 1);
  for (int i = 0; i < n; ++i) { int32_t k; PriorF p; rd(f, &k, 1); rd(f, p.t0, 3); rd(f, p.q0, 4); rd(f, p.sb0, 9); rd(f, p.sw, 15); s.priors.push_back({k, p}); }
  rd(f, &n, 1);
  for (int i = 0; i < n; ++i) { Spec::Between b; rd(f, &b.i, 1); rd(f, &b.j, 1); rd(f, b.f.dp, 3); rd(f, b.f.dq, 4); rd(f, b.f.dv, 3); rd(f, &b.f.dt, 1); rd(f, b.f.sw, 15); s.betweens.push_back(b); }
  rd(f, &n, 1);
  for (int i = 0; i < n; ++i) { Spec::DD d; rd(f, &d.i, 1); rd(f, &d.j, 1); rd(f, d.f.s1, 3); rd(f, d.f.s2, 3); rd(f, &d.f.rho_i, 1); rd(f, &d.f.rho_j, 1); rd(f, &d.f.w, 1); s.dds.push_back(d); }
  rd(f, &s.max_iter, 1); rd(f, &s.time_limit, 1);
  fclose(f);
  return s;
}

struct Result { ceres::Solver::Summary summary; std::vector<double> t, q, sb, gradient; double wall_ms = 0, cost = 0; };

enum Mode { SOLVE, EVALUATE, DESCRIBE };

// builds the problem at the file's state in the Estimator's order; then solves, evaluates or prints the descriptions
static Result solve(const Spec& s, glio_ctx* ctx, Mode mode = SOLVE, int max_iter = -1) {
  Result R;
  const int K = s.K;
  R.t.resize(3 * (size_t)K); R.q.resize(4 * (size_t)K); R.sb = s.sb;
  for (int k = 0; k < K; ++k) {
    for (int i = 0; i < 3; ++i) R.t[3 * k + i] = s.poses[7 * k + i];
    for (int i = 0; i < 4; ++i) R.q[4 * k + i] = s.poses[7 * k + 3 + i];
  }
  double* t = R.t.data(); double* q = R.q.data(); double* sb = R.sb.data();
  std::vector<double> rcv((size_t)3 * s.n_rcv, 0.0), rcv_ddt(std::max(s.epoch, 1), 0.0), alt = s.alt_t;
  double yaw = s.yaw, anchor[3] = {s.anchor[0], s.anchor[1], s.anchor[2]};
  ceres::Problem::Options po;
  po.loss_function_ownership = ceres::DO_NOT_TAKE_OWNERSHIP;
  std::vector<std::unique_ptr<ceres::LossFunction>> losses;
  ceres::Problem problem(po);
  problem.SetGlioContext(ctx);
  for (int i = 0; i < s.n_rcv; ++i) problem.AddParameterBlock(&rcv[3 * i], 3);                 // Estimator.cpp:2783-2790
  ceres::LocalParameterization* quat = new ceres::QuaternionParameterization();                  // one object, as the reference
  for (int k = 0; k < K; ++k) {                                                                   // :2794-2821
    problem.AddParameterBlock(t + 3 * k, 3, s.t_param[k] ? new ceres::IdentityParameterization(3) : nullptr);
    problem.AddParameterBlock(q + 4 * k, 4, s.q_ident[k] ? new ceres::IdentityParameterization(4) : quat);
    problem.AddParameterBlock(sb + 9 * k, 9);
    if (s.q_const[k]) problem.SetParameterBlockConstant(q + 4 * k);
  }
  for (size_t a = 0; a < alt.size() / 3; ++a) problem.AddParameterBlock(&alt[3 * a], 3);
  problem.AddParameterBlock(&yaw, 1); problem.SetParameterBlockConstant(&yaw);                     // :2822-2828
  problem.AddParameterBlock(anchor, 3); problem.SetParameterBlockConstant(anchor);
  bool ddt_added = false;
  for (const Spec::Pose& p : s.pose) {
    if (p.kind != 1 && !ddt_added && s.epoch > 0) { problem.AddParameterBlock(rcv_ddt.data(), s.epoch); ddt_added = true; }   // :2894
    ceres::LossFunction* loss = nullptr;
    if (p.loss >= 0) { losses.emplace_back(new ceres::HuberLoss(p.loss)); loss = losses.back().get(); }
    const Quaterniond dq{{p.dq[0], p.dq[1], p.dq[2], p.dq[3]}};
    const Vector3d dp{{p.dp[0], p.dp[1], p.dp[2]}};
    double* ti = p.alt >= 0 ? &alt[3 * p.alt] : t + 3 * p.i;
    if (p.kind == 1) {                                                                            // :2861-2863
      problem.AddResidualBlock(new ceres::AutoDiffCostFunction<delta_q_factor_auto, 3, 4, 4>(new delta_q_factor_auto(dq)), loss, q + 4 * p.i, q + 4 * p.j);
    } else if (p.kind == 0) {                                                                     // :2922-2925
      problem.AddResidualBlock(LidarPoseFactorBatchRelativeAutoDiff::Create(dq, dp), loss, ti, q + 4 * p.i, t + 3 * p.j, q + 4 * p.j);
    } else {
      problem.AddResidualBlock(new ceres::AutoDiffCostFunction<LidarPoseFactorAutoDiff, 6, 3, 4, 3, 4>(new LidarPoseFactorAutoDiff(dq, dp)), loss,
                               ti, q + 4 * p.i, t + 3 * p.j, q + 4 * p.j);
    }
  }
  if (!ddt_added && s.epoch > 0) problem.AddParameterBlock(rcv_ddt.data(), s.epoch);
  for (const Spec::Bin& b : s.bin) {
    BinaryLidarPlaneNormFactor* f = new BinaryLidarPlaneNormFactor();
    for (int k = 0; k < 3; ++k) f->curr_point[k] = b.cp[k];
    for (int k = 0; k < 6; ++k) f->planet_norm_cent[k] = b.nc[k];
    f->score = b.score;
    problem.AddResidualBlock(new ceres::AutoDiffCostFunction<BinaryLidarPlaneNormFactor, 1, 3, 4, 3, 4>(f), nullptr, t + 3 * b.kc, q + 4 * b.kc, t + 3 * b.ko, q + 4 * b.ko);
  }
  for (auto& p : s.priors)
    problem.AddResidualBlock(new ceres::AutoDiffCostFunction<PriorF, 15, 3, 4, 9>(new PriorF(p.second)), nullptr, t + 3 * p.first, q + 4 * p.first, sb + 9 * p.first);
  for (auto& b : s.betweens)
    problem.AddResidualBlock(new ceres::AutoDiffCostFunction<BetweenF, 15, 3, 4, 9, 3, 4, 9>(new BetweenF(b.f)), nullptr,
                             std::vector<double*>{t + 3 * b.i, q + 4 * b.i, sb + 9 * b.i, t + 3 * b.j, q + 4 * b.j, sb + 9 * b.j});
  for (auto& d : s.dds)
    problem.AddResidualBlock(new ceres::AutoDiffCostFunction<DDF, 2, 3, 3, 1, 3>(new DDF(d.f)), nullptr, t + 3 * d.i, t + 3 * d.j, &yaw, anchor);
  if (mode == DESCRIBE) {
    // the trait descriptions, printed exactly (C99 hex floats), next to the values the functors were constructed from
    for (const Spec::Pose& p : s.pose) {
      glio::FactorDesc d;
      bool ok;
      if (p.kind == 1) ok = glio::DeviceFactorTraits<delta_q_factor_auto>::describe(delta_q_factor_auto(Quaterniond{{p.dq[0], p.dq[1], p.dq[2], p.dq[3]}}), &d);
      else if (p.kind == 0) ok = glio::DeviceFactorTraits<LidarPoseFactorBatchRelativeAutoDiff>::describe(
                                LidarPoseFactorBatchRelativeAutoDiff(Quaterniond{{p.dq[0], p.dq[1], p.dq[2], p.dq[3]}}, Vector3d{{p.dp[0], p.dp[1], p.dp[2]}}), &d);
      else ok = glio::DeviceFactorTraits<LidarPoseFactorAutoDiff>::describe(LidarPoseFactorAutoDiff(Quaterniond{{1, 0, 0, 0}}, Vector3d{{0, 0, 0}}), &d);
      printf("desc %d %d", (int)ok, d.kind);
      for (int k = 0; k < 4; ++k) printf(" %a", d.dq[k]);
      for (int k = 0; k < 3; ++k) printf(" %a", d.dp[k]);
      printf("\n");
    }
    return R;
  }
  if (mode == EVALUATE) {
    problem.Evaluate(ceres::Problem::EvaluateOptions(), &R.cost, nullptr, &R.gradient, nullptr);
    return R;
  }
  ceres::Solver::Options options;                                                                 // Estimator.cpp:3275-3281
  options.linear_solver_type = ceres::SPARSE_NORMAL_CHOLESKY;
  options.num_threads = 1;
  options.max_num_iterations = max_iter >= 0 ? max_iter : s.max_iter;
  options.trust_region_strategy_type = ceres::DOGLEG;
  options.dogleg_type = ceres::SUBSPACE_DOGLEG;
  options.use_nonmonotonic_steps = true;
  options.max_solver_time_in_seconds = s.time_limit;
  const auto t0 = std::chrono::steady_clock::now();
  ceres::Solve(options, &problem, &R.summary);
  R.wall_ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
  return R;
}

static int64_t pose_launches(glio_ctx* ctx) { return launches(ctx, {"k_pose_pair_sums", "k_pose_pair_sums_cost", "k_pose_assemble"}); }

int main(int argc, char** argv) {
  if (argc < 3) { fprintf(stderr, "usage: shim_pose_routes_test host|device|evaluate|describe [--repeat R] [--max-iter M] [--use-pose] [--preload-pose N] problem.bin...\n"); return 2; }
  const std::string m = argv[1];
  const bool device = m == "device";
  int repeat = 0, preload = 0, max_iter = -1; bool use_pose = false;
  std::vector<const char*> files;
  for (int i = 2; i < argc; ++i) {
    const std::string a = argv[i];
    if (a == "--repeat" && i + 1 < argc) repeat = atoi(argv[++i]);
    else if (a == "--max-iter" && i + 1 < argc) max_iter = atoi(argv[++i]);
    else if (a == "--use-pose") use_pose = true;
    else if (a == "--preload-pose" && i + 1 < argc) preload = atoi(argv[++i]);
    else files.push_back(argv[i]);
  }
  if (files.empty()) return 2;
  glio_ctx* ctx = nullptr;
  if (device) {
    glio_params prm; glio_default_params(&prm);
    ctx = create_context(prm, !repeat);
    if (preload > 0) {
      // relative factors between keyframes 1 .. 9 with a large measured offset: any of them evaluated would add cost
      std::vector<glio_pose_factor> f(preload);
      for (int i = 0; i < preload; ++i) {
        f[i].i = 1 + i % 8; f[i].j = 2 + i % 8; f[i].kind = i % 2 ? GLIO_POSE_DELTA_Q : GLIO_POSE_RELATIVE; f[i].active = 1;
        f[i].dq[0] = 0.8; f[i].dq[1] = 0.6; f[i].dq[2] = 0; f[i].dq[3] = 0; f[i].dp[0] = 5; f[i].dp[1] = -3; f[i].dp[2] = 1;
      }
      if (glio_batch_set_pose_factors(ctx, f.data(), preload) != GLIO_OK || glio_batch_use_pose_factors(ctx, 1) != GLIO_OK) return 3;
      printf("preload %d\n", preload);
    }
    if (use_pose && glio_batch_use_pose_factors(ctx, 1) != GLIO_OK) return 3;
  }
  for (size_t fi = 0; fi < files.size(); ++fi) {
    const Spec s = read_spec(files[fi]);
    printf("solve %d\n", (int)fi);
    if (m == "evaluate") {
      const Result R = solve(s, nullptr, EVALUATE);
      printf("eval_cost %.17g\n", R.cost);
      printf("gradient"); for (double v : R.gradient) printf(" %.17g", v); printf("\n");
      continue;
    }
    if (m == "describe") { solve(s, nullptr, DESCRIBE); continue; }
    if (repeat) {
      for (int r = 0; r < repeat; ++r) {
        const Result R = solve(s, ctx, SOLVE, max_iter);
        printf("time %.6f %d %d\n", R.wall_ms, (int)R.summary.iterations.size(), R.summary.num_device_pose_residual_blocks);
      }
      continue;
    }
    const int64_t l0 = pose_launches(ctx);
    const Result R = solve(s, ctx, SOLVE, max_iter);
    const int64_t l1 = pose_launches(ctx);
    const ceres::Solver::Summary& S = R.summary;
    print_solve_head(S);
    printf("device_blocks %d\n", S.num_device_residual_blocks);
    printf("device_pose %d\n", S.num_device_pose_residual_blocks);
    printf("pose_launches %lld\n", (long long)(l1 - l0));
    print_solve_tail(S, s.K, R.t, R.q, &R.sb);
  }
  if (ctx) glio_destroy(ctx);
  return 0;
}
