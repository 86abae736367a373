// shim_test.cpp — builds a sliding-window problem through the Ceres-API shim exactly the way Estimator.cpp does
// (AddParameterBlock / QuaternionParameterization / AddResidualBlock(AutoDiffCostFunction, HuberLoss, t, q) /
// ceres::Solve with the options of Estimator.cpp:2424-2433) and prints the result.  Used by tests/test_shim.py:
//   host mode   : every residual block is evaluated on the host through CostFunction::Evaluate (no GPU needed)
//   device mode : the LidarPlaneNormFactor blocks describe themselves (glio::DeviceFactorTraits) and run on the GPU
// The functor below is an Eigen-free transcription of the reference's LidarPlaneNormFactor::operator()
// (GLIO/include/factors/LidarKeyframeFactor.h:88-103); the reference header itself needs Eigen, absent in this image.
#include <cstdio>
#include <cstdlib>
#include <vector>

#include "ceres/ceres.h"
#include "ceres/rotation.h"

template <typename T> static void QuatRotate(const T q[4], const T v[3], T o[3]) {   // Eigen Quaternion * Vector3
  T uv[3] = {q[2] * v[2] - q[3] * v[1], q[3] * v[0] - q[1] * v[2], q[1] * v[1] - q[2] * v[0]};
  uv[0] = uv[0] + uv[0]; uv[1] = uv[1] + uv[1]; uv[2] = uv[2] + uv[2];
  T c[3] = {q[2] * uv[2] - q[3] * uv[1], q[3] * uv[0] - q[1] * uv[2], q[1] * uv[1] - q[2] * uv[0]};
  for (int k = 0; k < 3; ++k) o[k] = v[k] + q[0] * uv[k] + c[k];
}

struct LidarPlaneNormFactor {
  LidarPlaneNormFactor(const double* cp_, const double* n_, const double* qlb_, const double* tlb_, double d_, double s_) : negative_OA_dot_norm(d_), score(s_) {
    for (int k = 0; k < 3; ++k) { curr_point[k] = cp_[k]; plane_unit_norm[k] = n_[k]; tlb[k] = tlb_[k]; }
    for (int k = 0; k < 4; ++k) qlb[k] = qlb_[k];
  }
  template <typename T> bool operator()(const T* t, const T* q, T* residual) const {
    T cp[3] = {T(curr_point[0]), T(curr_point[1]), T(curr_point[2])};
    T ql[4] = {T(qlb[0]), T(qlb[1]), T(qlb[2]), T(qlb[3])}, tl[3] = {T(tlb[0]), T(tlb[1]), T(tlb[2])};
    T n2 = ql[0] * ql[0] + ql[1] * ql[1] + ql[2] * ql[2] + ql[3] * ql[3];
    T qi[4] = {ql[0] / n2, -ql[1] / n2, -ql[2] / n2, -ql[3] / n2};
    T d[3] = {cp[0] - tl[0], cp[1] - tl[1], cp[2] - tl[2]}, pb[3], pw[3];
    QuatRotate(qi, d, pb); QuatRotate(q, pb, pw);
    for (int k = 0; k < 3; ++k) pw[k] = pw[k] + t[k];
    residual[0] = T(score) * (T(plane_unit_norm[0]) * pw[0] + T(plane_unit_norm[1]) * pw[1] + T(plane_unit_norm[2]) * pw[2] + T(negative_OA_dot_norm));
    return true;
  }
  static ceres::CostFunction* Create(const double* cp, const double* n, const double* qlb, const double* tlb, double d, double s) {
    return new ceres::AutoDiffCostFunction<LidarPlaneNormFactor, 1, 3, 4>(new LidarPlaneNormFactor(cp, n, qlb, tlb, d, s));
  }
  double curr_point[3], plane_unit_norm[3], qlb[4], tlb[3], negative_OA_dot_norm, score;
};

// the 10 lines a maintainer adds next to the reference's factor (INTEGRATION.md)
namespace glio {
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

// Eigen-free transcription of the reference's BinaryLidarPlaneNormFactor::operator() (LidarKeyframeFactor.h:132-150)
struct BinaryLidarPlaneNormFactor {
  BinaryLidarPlaneNormFactor(const double* cp_, const double* nc_, double s_) : score(s_) {
    for (int k = 0; k < 3; ++k) curr_point[k] = cp_[k];
    for (int k = 0; k < 6; ++k) planet_norm_cent[k] = nc_[k];
  }
  template <typename T> bool operator()(const T* t1, const T* q1, const T* t2, const T* q2, T* residual) const {
    T cp[3] = {T(curr_point[0]), T(curr_point[1]), T(curr_point[2])};
    T nl[3] = {T(planet_norm_cent[0]), T(planet_norm_cent[1]), T(planet_norm_cent[2])}, cl[3] = {T(planet_norm_cent[3]), T(planet_norm_cent[4]), T(planet_norm_cent[5])};
    T pw[3], no[3], co[3];
    QuatRotate(q1, cp, pw); QuatRotate(q2, nl, no); QuatRotate(q2, cl, co);
    for (int k = 0; k < 3; ++k) { pw[k] = pw[k] + t1[k]; co[k] = co[k] + t2[k]; }
    residual[0] = T(score) * (no[0] * (pw[0] - co[0]) + no[1] * (pw[1] - co[1]) + no[2] * (pw[2] - co[2]));
    return true;
  }
  static ceres::CostFunction* Create(const double* cp, const double* nc, double s) {
    return new ceres::AutoDiffCostFunction<BinaryLidarPlaneNormFactor, 1, 3, 4, 3, 4>(new BinaryLidarPlaneNormFactor(cp, nc, s));
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

// stand-ins for the host factors (IMU-chain-like / prior-like / pseudorange-like), autodiff on the host
struct PriorF {
  double t0[3], q0[4], sb0[9], sw[15];
  template <typename T> bool operator()(const T* t, const T* q, const T* sb, T* r) const {
    for (int k = 0; k < 3; ++k) r[k] = T(sw[k]) * (t[k] - T(t0[k]));
    T q0c[4] = {T(q0[0]), T(-q0[1]), T(-q0[2]), T(-q0[3])}, e[4];
    ceres::QuaternionProduct(q0c, q, e);      // same algebra as Eigen's product
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
    QuatRotate(qic, d, rp);
    for (int k = 0; k < 3; ++k) r[k] = T(sw[k]) * (rp[k] - T(dp[k]));
    T dqc[4] = {T(dq[0]), T(-dq[1]), T(-dq[2]), T(-dq[3])}, qij[4], e[4];
    ceres::QuaternionProduct(qic, qj, qij); ceres::QuaternionProduct(dqc, qij, e);
    for (int k = 0; k < 3; ++k) r[3 + k] = T(sw[3 + k]) * (T(2.0) * e[1 + k]);
    T dvv[3] = {sj[0] - si[0], sj[1] - si[1], sj[2] - si[2]}, rv[3];
    QuatRotate(qic, dvv, rv);
    for (int k = 0; k < 3; ++k) r[6 + k] = T(sw[6 + k]) * (rv[k] - T(dv[k]));
    for (int k = 0; k < 6; ++k) r[9 + k] = T(sw[9 + k]) * (sj[3 + k] - si[3 + k]);
    return true;
  }
};
struct RangeF {
  double lever[3], sat[3], rho, w;
  template <typename T> bool operator()(const T* t, const T* q, T* r) const {
    T lv[3] = {T(lever[0]), T(lever[1]), T(lever[2])}, pw[3];
    QuatRotate(q, lv, pw);
    T d[3] = {pw[0] + t[0] - T(sat[0]), pw[1] + t[1] - T(sat[1]), pw[2] + t[2] - T(sat[2])};
    r[0] = T(w) * (ceres::sqrt(d[0] * d[0] + d[1] * d[1] + d[2] * d[2]) - T(rho));
    return true;
  }
};

template <class T> static bool rd(FILE* f, T* p, size_t n) { return fread(p, sizeof(T), n, f) == n; }

int main(int argc, char** argv) {
  if (argc < 3) { fprintf(stderr, "usage: shim_test host|device problem.bin\n"); return 2; }
  FILE* f = fopen(argv[2], "rb");
  if (!f) return 2;
  const bool device = std::string(argv[1]) == "device";
  int32_t W, use_sb;
  rd(f, &W, 1); rd(f, &use_sb, 1);
  std::vector<double> poses(7 * W), sb(9 * W);
  rd(f, poses.data(), poses.size()); rd(f, sb.data(), sb.size());
  double q_lb[4], t_lb[3], lidar_const, huber;
  rd(f, q_lb, 4); rd(f, t_lb, 3); rd(f, &lidar_const, 1); rd(f, &huber, 1);
  int32_t N; rd(f, &N, 1);
  std::vector<int32_t> kf(N); std::vector<float> cp(3 * N), nsd(4 * N), w(N);
  rd(f, kf.data(), N); rd(f, cp.data(), 3 * N); rd(f, nsd.data(), 4 * N); rd(f, w.data(), N);

  // parameter blocks as the Estimator keeps them: raw double* arrays identified by address
  std::vector<double*> tmpTrans(W), tmpQuat(W), tmpSpeedBias(W);
  for (int k = 0; k < W; ++k) {
    tmpTrans[k] = new double[3]; tmpQuat[k] = new double[4]; tmpSpeedBias[k] = new double[9];
    for (int i = 0; i < 3; ++i) tmpTrans[k][i] = poses[7 * k + i];
    for (int i = 0; i < 4; ++i) tmpQuat[k][i] = poses[7 * k + 3 + i];
    for (int i = 0; i < 9; ++i) tmpSpeedBias[k][i] = sb[9 * k + i];
  }
  double para_yaw[1] = {0.3}, para_anchor[3] = {1, 2, 3}, unused_rcv[3] = {0, 0, 0};

  glio_ctx* ctx = nullptr;
  if (device) {
    glio_params prm; glio_default_params(&prm);
    for (int k = 0; k < 4; ++k) prm.q_lb[k] = q_lb[k];
    for (int k = 0; k < 3; ++k) prm.t_lb[k] = t_lb[k];
    prm.lidar_const = lidar_const; prm.huber_delta = huber;
    if (glio_create(0, &prm, &ctx) != GLIO_OK) { fprintf(stderr, "glio_create: %s\n", glio_last_error(nullptr)); return 3; }
  }
  ceres::Solver::Summary summary;
  {
    ceres::LossFunction* lossFunction = new ceres::HuberLoss(huber);                       // Estimator.cpp:2092
    ceres::LocalParameterization* quatParameterization = new ceres::QuaternionParameterization();
    ceres::Problem problem;
    problem.SetGlioContext(ctx);
    for (int k = 0; k < W; ++k) {                                                          // Estimator.cpp:2130-2137
      problem.AddParameterBlock(tmpTrans[k], 3);
      problem.AddParameterBlock(tmpQuat[k], 4, quatParameterization);
      if (use_sb) problem.AddParameterBlock(tmpSpeedBias[k], 9);
    }
    problem.AddParameterBlock(unused_rcv, 3);                                              // never used by a residual: dropped
    problem.AddParameterBlock(para_yaw, 1); problem.SetParameterBlockConstant(para_yaw);   // Estimator.cpp:2140-2145
    problem.AddParameterBlock(para_anchor, 3); problem.SetParameterBlockConstant(para_anchor);
    for (int i = 0; i < N; ++i) {                                                          // Estimator.cpp:2226-2242
      const double c[3] = {cp[3 * i], cp[3 * i + 1], cp[3 * i + 2]}, n[3] = {nsd[4 * i], nsd[4 * i + 1], nsd[4 * i + 2]};
      ceres::CostFunction* cost = LidarPlaneNormFactor::Create(c, n, q_lb, t_lb, nsd[4 * i + 3], lidar_const * (double)w[i]);
      problem.AddResidualBlock(cost, lossFunction, tmpTrans[kf[i]], tmpQuat[kf[i]]);
    }
    int32_t np; rd(f, &np, 1);
    for (int i = 0; i < np; ++i) {
      int32_t k; PriorF* p = new PriorF(); rd(f, &k, 1); rd(f, p->t0, 3); rd(f, p->q0, 4); rd(f, p->sb0, 9); rd(f, p->sw, 15);
      if (use_sb) problem.AddResidualBlock(new ceres::AutoDiffCostFunction<PriorF, 15, 3, 4, 9>(p), NULL, tmpTrans[k], tmpQuat[k], tmpSpeedBias[k]);
      else delete p;
    }
    int32_t nbt; rd(f, &nbt, 1);
    for (int i = 0; i < nbt; ++i) {
      int32_t a, b; BetweenF* p = new BetweenF(); rd(f, &a, 1); rd(f, &b, 1); rd(f, p->dp, 3); rd(f, p->dq, 4); rd(f, p->dv, 3); rd(f, &p->dt, 1); rd(f, p->sw, 15);
      if (use_sb) problem.AddResidualBlock(new ceres::AutoDiffCostFunction<BetweenF, 15, 3, 4, 9, 3, 4, 9>(p), NULL,
                                           std::vector<double*>{tmpTrans[a], tmpQuat[a], tmpSpeedBias[a], tmpTrans[b], tmpQuat[b], tmpSpeedBias[b]});
      else delete p;
    }
    int32_t nrg; rd(f, &nrg, 1);
    for (int i = 0; i < nrg; ++i) {
      int32_t k; RangeF* p = new RangeF(); rd(f, &k, 1); rd(f, p->lever, 3); rd(f, p->sat, 3); rd(f, &p->rho, 1); rd(f, &p->w, 1);
      problem.AddResidualBlock(new ceres::AutoDiffCostFunction<RangeF, 1, 3, 4>(p), NULL, tmpTrans[k], tmpQuat[k]);
    }
    // optional trailing section: scan-to-multiscan (binary) plane factors between keyframes of the same problem,
    // added the way optimizeBatchWithLandMark does (Estimator.cpp:3049-3051, :3073-3074: loss == NULL, four blocks)
    int32_t nbin = 0;
    if (rd(f, &nbin, 1) && nbin > 0) {
      std::vector<int32_t> kc(nbin), ko(nbin); std::vector<float> bcp(3 * (size_t)nbin); std::vector<double> bnc(6 * (size_t)nbin), bsc(nbin);
      rd(f, kc.data(), nbin); rd(f, ko.data(), nbin); rd(f, bcp.data(), bcp.size()); rd(f, bnc.data(), bnc.size()); rd(f, bsc.data(), nbin);
      for (int i = 0; i < nbin; ++i) {
        const double c[3] = {bcp[3 * i], bcp[3 * i + 1], bcp[3 * i + 2]};
        problem.AddResidualBlock(BinaryLidarPlaneNormFactor::Create(c, &bnc[6 * (size_t)i], bsc[i]), NULL, tmpTrans[kc[i]], tmpQuat[kc[i]], tmpTrans[ko[i]], tmpQuat[ko[i]]);
      }
    }
    fclose(f);
    ceres::Solver::Options options;                                                        // Estimator.cpp:2424-2430
    options.linear_solver_type = ceres::SPARSE_NORMAL_CHOLESKY;
    options.num_threads = 1;
    options.max_num_iterations = 15;
    options.trust_region_strategy_type = ceres::DOGLEG;
    options.minimizer_progress_to_stdout = false;
    options.use_nonmonotonic_steps = false;
    ceres::Solve(options, &problem, &summary);
  }
  printf("solve\n");
  printf("termination %d\n", (int)summary.termination_type);
  printf("iters %d\n", (int)summary.iterations.size());
  printf("device_blocks %d\n", summary.num_device_residual_blocks);
  printf("blocks %d %d\n", summary.num_parameter_blocks, summary.num_effective_parameters);
  for (auto& it : summary.iterations) printf("it %d %d %.17g %.17g\n", it.iteration, (int)it.step_is_successful, it.cost, it.trust_region_radius);
  for (int k = 0; k < W; ++k) {
    printf("pose %d %.17g %.17g %.17g %.17g %.17g %.17g %.17g\n", k, tmpTrans[k][0], tmpTrans[k][1], tmpTrans[k][2], tmpQuat[k][0], tmpQuat[k][1], tmpQuat[k][2], tmpQuat[k][3]);
    printf("sb %d", k); for (int i = 0; i < 9; ++i) printf(" %.17g", tmpSpeedBias[k][i]); printf("\n");
  }
  printf("const %.17g %.17g\n", para_yaw[0], para_anchor[2]);
  if (ctx) glio_destroy(ctx);
  return 0;
}
