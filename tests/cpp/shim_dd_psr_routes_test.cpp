// shim_dd_psr_routes_test.cpp — the Ceres-API shim's route for the batch refinement's DD pseudorange factors (K2g):
// dd_psr_factor_20 blocks added the way optimizeBatchWithLandMark adds them (Estimator.cpp:2794-2954 and :3086-3272: per keyframe
// t and q (QuaternionParameterization), the constant yaw and anchor, the attitude factors, the relative factors, then the DD
// factors per epoch and constellation through addDDPsrResFactor_gl, :1902-1913).  Used by tests/test_shim_dd_psr_routes.py and
// scripts/bench_shim_dd_psr_routes.py:
//   shim_dd_psr_routes_test host   [--repeat R] [--max-iter M] problem.bin...   every block evaluated on the host (no GPU needed)
//   shim_dd_psr_routes_test evaluate problem.bin...                              Problem::Evaluate (host): cost and tangent gradient
//   shim_dd_psr_routes_test describe problem.bin...                              each DD block's trait description and each frame's
//                                                                                R_ecef_local, in hex
//   shim_dd_psr_routes_test device [--repeat R] [--max-iter M] [--use-pose] [--use-dd] [--preload-dd N] problem.bin...
//       the described blocks are routed to the GPU; all problems are solved in turn on ONE context, after
//       glio_batch_use_pose_factors / glio_batch_use_dd_psr_factors(ctx, 1) if asked.  One problem per call is a fresh context.
//       --preload-dd N first leaves what a direct (Level-2) caller would: a list of N other DD factors and the switch on.
//   --dd-as-cost-function (any mode): every DD factor is added through a ceres::CostFunction*, so its blocks stay on the host
// For each problem it prints the iterations, poses and costs (%.17g), the residual and device block counts, the K2g and K2p
// launches of that solve, and the smallest | |e_k| - threshold | over every DD row the host evaluated (the gate margin).  With
// --repeat R each problem is rebuilt from its file and solved R times, and each solve's wall time is printed.
//
// dd_psr_factor_20 is restated without Eigen from its formula (glio_b200.h, K2g), with Eigen's semantics: normalized() of a zero
// vector is the vector itself, the 19 x 19 weight is the (n_sat-1) x (n_sat-1) W padded with zeros, r = W r and J = W J.  It keeps
// its data members private, as the reference does (dd_psr_factor.hpp:173-188), so its trait reads them the way INTEGRATION.md
// shows: through pointers to members named in an explicit instantiation.
#include <algorithm>
#include <chrono>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <limits>
#include <string>
#include <vector>

#include "ceres/ceres.h"
#include "shim_driver.h"

// ---- the parts of Eigen, nlosExclusion and gnss_comm the factor and its trait use ----------------------------------------------
struct Quaterniond {
  double c[4];   // w, x, y, z
  double w() const { return c[0]; } double x() const { return c[1]; } double y() const { return c[2]; } double z() const { return c[3]; }
};
struct Vector3d {
  double c[3];
  double operator[](int k) const { return c[k]; }
  double x() const { return c[0]; } double y() const { return c[1]; } double z() const { return c[2]; }
};
struct Matrix3d {   // row-major; products sum over k in index order, as Eigen's lazy 3 x 3 product
  double m[9];
  double operator()(int r, int c) const { return m[3 * r + c]; }
  Matrix3d operator*(const Matrix3d& b) const {
    Matrix3d o;
    for (int r = 0; r < 3; ++r)
      for (int c = 0; c < 3; ++c) o.m[3 * r + c] = m[3 * r] * b.m[c] + m[3 * r + 1] * b.m[3 + c] + m[3 * r + 2] * b.m[6 + c];
    return o;
  }
};
struct MatrixXd {   // dynamic, row-major storage
  int r = 0, c = 0;
  std::vector<double> v;
  int rows() const { return r; } int cols() const { return c; }
  double operator()(int i, int j) const { return v[(size_t)i * c + j]; }
};
namespace nlosExclusion {
struct GNSS_Raw { double sat_pos_x = 0, sat_pos_y = 0, sat_pos_z = 0, raw_pseudorange = 0; double prn_satellites_index = 0; };
struct GNSS_Raw_Array { std::vector<GNSS_Raw> GNSS_Raws; };
}  // namespace nlosExclusion

// gnss_comm's ecef2rotation (gnss_utility.cpp: ecef2geo, geo2rotation), with gnss_constant.hpp's WGS 84 constants
namespace gnss_comm {
static Vector3d ecef2geo(const Vector3d& xyz) {
  const double R2D = 180.0 / M_PI;
  if (xyz.x() == 0 && xyz.y() == 0) return Vector3d{{0, 0, 0}};
  const double e2 = 6.69437999014e-3, a = 6378137;
  const double a2 = a * a, b2 = a2 * (1 - e2), b = std::sqrt(b2), ep2 = (a2 - b2) / b2;
  const double p = std::sqrt(xyz.x() * xyz.x() + xyz.y() * xyz.y());
  double s1 = xyz.z() * a, s2 = p * b;
  double h = std::sqrt(s1 * s1 + s2 * s2);
  const double sin_theta = s1 / h, cos_theta = s2 / h;
  s1 = xyz.z() + ep2 * b * std::pow(sin_theta, 3);
  s2 = p - a * e2 * std::pow(cos_theta, 3);
  h = std::sqrt(s1 * s1 + s2 * s2);
  const double tan_lat = s1 / s2, sin_lat = s1 / h, cos_lat = s2 / h;
  const double lat_deg = std::atan(tan_lat) * R2D;
  const double N = a2 * std::pow((a2 * cos_lat * cos_lat + b2 * sin_lat * sin_lat), -0.5);
  const double alt = p / cos_lat - N;
  const double lon_deg = std::atan2(xyz.y(), xyz.x()) * R2D;
  return Vector3d{{lat_deg, lon_deg, alt}};
}
static Matrix3d geo2rotation(const Vector3d& geo) {
  const double D2R = M_PI / 180.0;
  const double lat = geo.x() * D2R, lon = geo.y() * D2R;
  const double sin_lat = std::sin(lat), cos_lat = std::cos(lat), sin_lon = std::sin(lon), cos_lon = std::cos(lon);
  return Matrix3d{{-sin_lon, -sin_lat * cos_lon, cos_lat * cos_lon, cos_lon, -sin_lat * sin_lon, cos_lat * sin_lon, 0, cos_lat, sin_lat}};
}
static Matrix3d ecef2rotation(const Vector3d& ref_ecef) { return geo2rotation(ecef2geo(ref_ecef)); }
}  // namespace gnss_comm

// R_ecef_local = ecef2rotation(anchor) * R_enu_local(yaw), as dd_psr_factor_20::Evaluate forms it
static Matrix3d ecef_local(double yaw, const double* anchor) {
  const double s = std::sin(yaw), c = std::cos(yaw);
  const Matrix3d R_enu_local{{c, -s, 0, s, c, 0, 0, 0, 1}};
  return gnss_comm::ecef2rotation(Vector3d{{anchor[0], anchor[1], anchor[2]}}) * R_enu_local;
}

static double g_gate_margin = std::numeric_limits<double>::infinity();   // min | |e_k| - threshold | over the host evaluations
static bool g_dd_as_cost_function = false;                                   // --dd-as-cost-function

// ---- dd_psr_factor_20 (dd_psr_factor.hpp:15-189), restated ---------------------------------------------------------------------
class dd_psr_factor_20 : public ceres::SizedCostFunction<19, 3, 3, 1, 3> {
 public:
  dd_psr_factor_20(const nlosExclusion::GNSS_Raw_Array& _gnss_data, const nlosExclusion::GNSS_Raw_Array& _ref_gnss_data, const MatrixXd& _DD_W_matrix,
                   const int& _mPrn, const double& _ratio, const Vector3d& _Station_pos, const double& _DDpsrThreshold)
      : ratio(_ratio), DDpsrThreshold(_DDpsrThreshold), Station_pos(_Station_pos), gnss_data(_gnss_data), ref_gnss_data(_ref_gnss_data),
        DD_W_matrix(_DD_W_matrix), mPrn(_mPrn) {}
  bool Evaluate(double const* const* parameters, double* residuals, double** jacobians) const override {
    const double* Pi = parameters[0]; const double* Pj = parameters[1];
    const Matrix3d R = ecef_local(parameters[2][0], parameters[3]);
    double local[3], P[3];
    for (int k = 0; k < 3; ++k) local[k] = ratio * Pi[k] + (1.0 - ratio) * Pj[k];
    for (int r = 0; r < 3; ++r) P[r] = (R(r, 0) * local[0] + R(r, 1) * local[1] + R(r, 2) * local[2]) + parameters[3][r];
    const auto& U = gnss_data.GNSS_Raws; const auto& F = ref_gnss_data.GNSS_Raws;
    const int n = (int)U.size(), m = mPrn;
    auto sat = [](const nlosExclusion::GNSS_Raw& g, double* o) { o[0] = g.sat_pos_x; o[1] = g.sat_pos_y; o[2] = g.sat_pos_z; };
    auto norm = [](const double* v) { return std::sqrt(v[0] * v[0] + v[1] * v[1] + v[2] * v[2]); };
    auto unit = [&](const double* v, double* u) { const double sq = v[0] * v[0] + v[1] * v[1] + v[2] * v[2], l = std::sqrt(sq); for (int k = 0; k < 3; ++k) u[k] = sq > 0 ? v[k] / l : v[k]; };
    double Ji[19][3] = {}, Jj[19][3] = {}, r[19] = {};
    int row = 0;
    for (int i = 0; i < n; ++i) {
      if (i == m) continue;
      double su[3], sm[3], rm[3], ri[3], du[3], dm[3], dri[3], drm[3], uu[3], um[3];
      sat(U[i], su); sat(U[m], sm); sat(F[m], rm); sat(F[i], ri);
      for (int k = 0; k < 3; ++k) { du[k] = su[k] - P[k]; dm[k] = sm[k] - P[k]; dri[k] = ri[k] - Station_pos[k]; drm[k] = rm[k] - Station_pos[k]; }
      unit(du, uu); unit(dm, um);
      const double est = (norm(du) - norm(dri)) - (norm(dm) - norm(drm));
      const double meas = (U[i].raw_pseudorange - F[i].raw_pseudorange) - (U[m].raw_pseudorange - F[m].raw_pseudorange);
      double w = 1.0;
      r[row] = w * (est - meas);
      g_gate_margin = std::min(g_gate_margin, std::fabs(std::fabs(r[row]) - DDpsrThreshold));
      if (std::fabs(r[row]) > DDpsrThreshold) w = 0.05 * w;
      r[row] = w * (est - meas);
      for (int c = 0; c < 3; ++c) {
        const double a = -uu[0] * R(0, c) + -uu[1] * R(1, c) + -uu[2] * R(2, c), b = -um[0] * R(0, c) + -um[1] * R(1, c) + -um[2] * R(2, c);
        Ji[row][c] = (a * w * ratio) - (b * w * ratio);
        Jj[row][c] = (a * w * (1.0 - ratio)) - (b * w * (1.0 - ratio));
      }
      ++row;
    }
    double Wp[19][19] = {};                                        // DD_W_matrix_ep: W in the top-left block, zeros elsewhere
    for (int a = 0; a < DD_W_matrix.rows(); ++a) for (int b = 0; b < DD_W_matrix.cols(); ++b) Wp[a][b] = DD_W_matrix(a, b);
    for (int a = 0; a < 19; ++a) {
      double s = 0, si[3] = {0, 0, 0}, sj[3] = {0, 0, 0};
      for (int b = 0; b < 19; ++b) {
        s += Wp[a][b] * r[b];
        for (int c = 0; c < 3; ++c) { si[c] += Wp[a][b] * Ji[b][c]; sj[c] += Wp[a][b] * Jj[b][c]; }
      }
      residuals[a] = s;
      if (jacobians && jacobians[0]) for (int c = 0; c < 3; ++c) jacobians[0][3 * a + c] = si[c];
      if (jacobians && jacobians[1]) for (int c = 0; c < 3; ++c) jacobians[1][3 * a + c] = sj[c];
    }
    return true;
  }

 private:
  double ratio;
  double DDpsrThreshold;
  Vector3d Station_pos;
  const nlosExclusion::GNSS_Raw_Array gnss_data;
  const nlosExclusion::GNSS_Raw_Array ref_gnss_data;
  MatrixXd DD_W_matrix;
  int mPrn;
};

// ---- what a maintainer adds next to dd_psr_factor.hpp (INTEGRATION.md, Level 1) ---------------------------------------------
// Access checks do not apply to the names in an explicit instantiation, so instantiating DdMember with &dd_psr_factor_20::mPrn
// defines the friend member_ptr(DdMaster), which returns that pointer.
template <class Tag, typename Tag::type Member> struct DdMember { friend typename Tag::type member_ptr(Tag) { return Member; } };
struct DdUser { typedef const nlosExclusion::GNSS_Raw_Array dd_psr_factor_20::*type; friend type member_ptr(DdUser); };
struct DdRef { typedef const nlosExclusion::GNSS_Raw_Array dd_psr_factor_20::*type; friend type member_ptr(DdRef); };
struct DdW { typedef MatrixXd dd_psr_factor_20::*type; friend type member_ptr(DdW); };
struct DdMaster { typedef int dd_psr_factor_20::*type; friend type member_ptr(DdMaster); };
struct DdRatio { typedef double dd_psr_factor_20::*type; friend type member_ptr(DdRatio); };
struct DdThreshold { typedef double dd_psr_factor_20::*type; friend type member_ptr(DdThreshold); };
struct DdStation { typedef Vector3d dd_psr_factor_20::*type; friend type member_ptr(DdStation); };
template struct DdMember<DdUser, &dd_psr_factor_20::gnss_data>;
template struct DdMember<DdRef, &dd_psr_factor_20::ref_gnss_data>;
template struct DdMember<DdW, &dd_psr_factor_20::DD_W_matrix>;
template struct DdMember<DdMaster, &dd_psr_factor_20::mPrn>;
template struct DdMember<DdRatio, &dd_psr_factor_20::ratio>;
template struct DdMember<DdThreshold, &dd_psr_factor_20::DDpsrThreshold>;
template struct DdMember<DdStation, &dd_psr_factor_20::Station_pos>;

namespace glio {
template <> struct DeviceCostTraits<dd_psr_factor_20> {
  static bool describe(const dd_psr_factor_20& f, DdPsrDesc* d) {
    const auto& user = (f.*member_ptr(DdUser())).GNSS_Raws;
    const auto& ref = (f.*member_ptr(DdRef())).GNSS_Raws;
    const MatrixXd& W = f.*member_ptr(DdW());
    const int n = (int)user.size(), m = f.*member_ptr(DdMaster());
    if (n < 2 || n > GLIO_DD_PSR_MAX_SAT || (int)ref.size() != n || m < 0 || m >= n || W.rows() != n - 1 || W.cols() != n - 1) return false;
    d->n_sat = n; d->master = m;
    d->ratio = f.*member_ptr(DdRatio()); d->threshold = f.*member_ptr(DdThreshold());
    const Vector3d& st = f.*member_ptr(DdStation());
    for (int k = 0; k < 3; ++k) d->station[k] = st[k];
    for (int s = 0; s < n; ++s) {
      d->sat_user[s][0] = user[s].sat_pos_x; d->sat_user[s][1] = user[s].sat_pos_y; d->sat_user[s][2] = user[s].sat_pos_z;
      d->sat_ref[s][0] = ref[s].sat_pos_x; d->sat_ref[s][1] = ref[s].sat_pos_y; d->sat_ref[s][2] = ref[s].sat_pos_z;
      d->psr_user[s] = user[s].raw_pseudorange; d->psr_ref[s] = ref[s].raw_pseudorange;
    }
    d->w_identity = 1;
    for (int a = 0; a < n - 1; ++a)
      for (int b = 0; b < n - 1; ++b) {
        d->W[a * (n - 1) + b] = W(a, b);
        if (W(a, b) != (a == b ? 1.0 : 0.0)) d->w_identity = 0;
      }
    return true;
  }
  static void frame(const double* yaw, const double* anchor, double R_ecef_local[9]) {
    const Matrix3d R = ecef_local(yaw[0], anchor);
    for (int k = 0; k < 9; ++k) R_ecef_local[k] = R.m[k];
  }
};
}  // namespace glio

// ---- the pose functors and the binary plane factor of tests/cpp/shim_pose_routes_test.cpp, with their traits --------------------
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
struct LidarPoseFactorBatchRelativeAutoDiff {
  LidarPoseFactorBatchRelativeAutoDiff(Quaterniond delta_q_, Vector3d delta_p_) : delta_q(delta_q_), delta_p(delta_p_) {}
  template <typename T> bool operator()(const T* p1, const T* q1, const T* p2, const T* q2, T* r) const {
    const T dqv[4] = {T(delta_q.w()), T(delta_q.x()), T(delta_q.y()), T(delta_q.z())};
    T dqi[4], q1i[4], a[4], e[4];
    QInv(dqv, dqi); QInv(q1, q1i); QMul(dqi, q1i, a); QMul(a, q2, e);
    const T d[3] = {p2[0] - p1[0], p2[1] - p1[1], p2[2] - p1[2]};
    T b[3];
    Rotate(q1i, d, b);
    for (int k = 0; k < 3; ++k) r[k] = T(10.0) * (T(2.0) * e[1 + k]);
    for (int k = 0; k < 3; ++k) r[3 + k] = T(20.0) * (b[k] - T(delta_p[k]));
    return true;
  }
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
template <> struct DeviceFactorTraits<LidarPoseFactorBatchRelativeAutoDiff> {
  static bool describe(const LidarPoseFactorBatchRelativeAutoDiff& f, FactorDesc* d) {
    d->kind = FACTOR_POSE_RELATIVE;
    d->dq[0] = f.delta_q.w(); d->dq[1] = f.delta_q.x(); d->dq[2] = f.delta_q.y(); d->dq[3] = f.delta_q.z();
    for (int k = 0; k < 3; ++k) d->dp[k] = f.delta_p[k];
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

// a host prior that keeps a variable yaw or anchor block near its value (the DD factor leaves their Jacobians zero)
template <int N> struct PriorN {
  double x0[N];
  template <typename T> bool operator()(const T* x, T* r) const { for (int k = 0; k < N; ++k) r[k] = T(10.0) * (x[k] - T(x0[k])); return true; }
};

// one problem file (written by tests/test_shim_dd_psr_routes.py: write_problem)
struct Spec {
  int32_t K = 0;
  std::vector<double> poses, q_alt;
  std::vector<int32_t> t_const;
  struct Frame { double yaw, anchor[3]; int32_t yaw_const, anchor_const; };
  std::vector<Frame> frames;
  struct Pose { int32_t kind, i, j, alt_q; double dq[4], dp[3]; };   // kind 0 relative, 1 delta_q; alt_q >= 0: q_i is extra q block alt_q
  std::vector<Pose> pose;
  struct Bin { int32_t kc, ko; double cp[3], nc[6], score; };
  std::vector<Bin> bin;
  // n_ref: the station's satellite count (n_sat unless a test gives it another length); w_rows 0: an identity W
  struct DD { int32_t i, j, n_sat, n_ref, master, frame, as_base, w_rows; double ratio, threshold, station[3], loss; std::vector<double> user, ref, W; };
  std::vector<DD> dds;
  int32_t max_iter = 10;
  double time_limit = 1e9;
};

static Spec read_spec(const char* path) {
  FILE* f = fopen(path, "rb");
  if (!f) { fprintf(stderr, "cannot open %s\n", path); exit(2); }
  Spec s;
  int32_t n_alt, n_frames, n;
  rd(f, &s.K, 1); rd(f, &n_alt, 1); rd(f, &n_frames, 1);
  s.poses.resize(7 * (size_t)s.K); rd(f, s.poses.data(), s.poses.size());
  s.t_const.resize(s.K); rd(f, s.t_const.data(), s.K);
  s.frames.resize(n_frames);
  for (auto& fr : s.frames) { rd(f, &fr.yaw, 1); rd(f, fr.anchor, 3); rd(f, &fr.yaw_const, 1); rd(f, &fr.anchor_const, 1); }
  s.q_alt.resize(4 * (size_t)n_alt); rd(f, s.q_alt.data(), s.q_alt.size());
  rd(f, &n, 1); s.pose.resize(n);
  for (auto& p : s.pose) { rd(f, &p.kind, 1); rd(f, &p.i, 1); rd(f, &p.j, 1); rd(f, &p.alt_q, 1); rd(f, p.dq, 4); rd(f, p.dp, 3); }
  rd(f, &n, 1); s.bin.resize(n);
  for (auto& b : s.bin) { rd(f, &b.kc, 1); rd(f, &b.ko, 1); rd(f, b.cp, 3); rd(f, b.nc, 6); rd(f, &b.score, 1); }
  rd(f, &n, 1); s.dds.resize(n);
  for (auto& d : s.dds) {
    rd(f, &d.i, 1); rd(f, &d.j, 1); rd(f, &d.n_sat, 1); rd(f, &d.n_ref, 1); rd(f, &d.master, 1); rd(f, &d.frame, 1); rd(f, &d.as_base, 1); rd(f, &d.w_rows, 1);
    rd(f, &d.ratio, 1); rd(f, &d.threshold, 1); rd(f, d.station, 3); rd(f, &d.loss, 1);
    d.user.resize(4 * (size_t)d.n_sat); rd(f, d.user.data(), d.user.size());
    d.ref.resize(4 * (size_t)d.n_ref); rd(f, d.ref.data(), d.ref.size());
    d.W.resize((size_t)d.w_rows * d.w_rows); rd(f, d.W.data(), d.W.size());
  }
  rd(f, &s.max_iter, 1); rd(f, &s.time_limit, 1);
  fclose(f);
  return s;
}

static nlosExclusion::GNSS_Raw_Array raws(const std::vector<double>& v) {   // rows of (sat x, y, z, pseudorange)
  nlosExclusion::GNSS_Raw_Array a;
  for (size_t s = 0; s < v.size() / 4; ++s) {
    nlosExclusion::GNSS_Raw g;
    g.sat_pos_x = v[4 * s]; g.sat_pos_y = v[4 * s + 1]; g.sat_pos_z = v[4 * s + 2]; g.raw_pseudorange = v[4 * s + 3]; g.prn_satellites_index = (double)(s + 1);
    a.GNSS_Raws.push_back(g);
  }
  return a;
}

static dd_psr_factor_20* make_dd(const Spec::DD& d) {   // addDDPsrResFactor_gl: identity weight of the rover's size unless given
  MatrixXd W;
  if (d.w_rows > 0) { W.r = W.c = d.w_rows; W.v = d.W; }
  else { W.r = W.c = d.n_sat - 1; W.v.assign((size_t)W.r * W.c, 0.0); for (int k = 0; k < W.r; ++k) W.v[(size_t)k * W.c + k] = 1.0; }
  return new dd_psr_factor_20(raws(d.user), raws(d.ref), W, d.master, d.ratio, Vector3d{{d.station[0], d.station[1], d.station[2]}}, d.threshold);
}

struct Result { ceres::Solver::Summary summary; std::vector<double> t, q, gradient; double wall_ms = 0, cost = 0; };

enum Mode { SOLVE, EVALUATE, DESCRIBE };

// builds the problem at the file's state in the Estimator's order; then solves, evaluates or prints the descriptions
static Result solve(const Spec& s, glio_ctx* ctx, Mode mode = SOLVE, int max_iter = -1) {
  Result R;
  const int K = s.K;
  R.t.resize(3 * (size_t)K); R.q.resize(4 * (size_t)K);
  for (int k = 0; k < K; ++k) {
    for (int i = 0; i < 3; ++i) R.t[3 * k + i] = s.poses[7 * k + i];
    for (int i = 0; i < 4; ++i) R.q[4 * k + i] = s.poses[7 * k + 3 + i];
  }
  double* t = R.t.data(); double* q = R.q.data();
  std::vector<double> q_alt = s.q_alt;
  std::vector<double> yaw(s.frames.size()), anchor(3 * s.frames.size());
  ceres::Problem::Options po;
  po.loss_function_ownership = ceres::DO_NOT_TAKE_OWNERSHIP;
  std::vector<std::unique_ptr<ceres::LossFunction>> losses;
  ceres::Problem problem(po);
  problem.SetGlioContext(ctx);
  ceres::LocalParameterization* quat = new ceres::QuaternionParameterization();                  // one object, as the reference
  for (int k = 0; k < K; ++k) {                                                                   // Estimator.cpp:2794-2821
    problem.AddParameterBlock(t + 3 * k, 3);
    problem.AddParameterBlock(q + 4 * k, 4, quat);
    if (s.t_const[k]) problem.SetParameterBlockConstant(t + 3 * k);
  }
  for (size_t a = 0; a < q_alt.size() / 4; ++a) problem.AddParameterBlock(&q_alt[4 * a], 4, quat);
  for (size_t fi = 0; fi < s.frames.size(); ++fi) {                                               // :2822-2828
    yaw[fi] = s.frames[fi].yaw;
    for (int k = 0; k < 3; ++k) anchor[3 * fi + k] = s.frames[fi].anchor[k];
    problem.AddParameterBlock(&yaw[fi], 1);
    if (s.frames[fi].yaw_const) problem.SetParameterBlockConstant(&yaw[fi]);
    problem.AddParameterBlock(&anchor[3 * fi], 3);
    if (s.frames[fi].anchor_const) problem.SetParameterBlockConstant(&anchor[3 * fi]);
  }
  for (const Spec::Pose& p : s.pose) {
    const Quaterniond dq{{p.dq[0], p.dq[1], p.dq[2], p.dq[3]}};
    double* qi = p.alt_q >= 0 ? &q_alt[4 * p.alt_q] : q + 4 * p.i;
    if (p.kind == 1)                                                                              // :2861-2863
      problem.AddResidualBlock(new ceres::AutoDiffCostFunction<delta_q_factor_auto, 3, 4, 4>(new delta_q_factor_auto(dq)), nullptr, qi, q + 4 * p.j);
    else                                                                                          // :2922-2925
      problem.AddResidualBlock(new ceres::AutoDiffCostFunction<LidarPoseFactorBatchRelativeAutoDiff, 6, 3, 4, 3, 4>(
                                   new LidarPoseFactorBatchRelativeAutoDiff(dq, Vector3d{{p.dp[0], p.dp[1], p.dp[2]}})),
                               nullptr, t + 3 * p.i, qi, t + 3 * p.j, q + 4 * p.j);
  }
  for (const Spec::Bin& b : s.bin) {
    BinaryLidarPlaneNormFactor* f = new BinaryLidarPlaneNormFactor();
    for (int k = 0; k < 3; ++k) f->curr_point[k] = b.cp[k];
    for (int k = 0; k < 6; ++k) f->planet_norm_cent[k] = b.nc[k];
    f->score = b.score;
    problem.AddResidualBlock(new ceres::AutoDiffCostFunction<BinaryLidarPlaneNormFactor, 1, 3, 4, 3, 4>(f), nullptr, t + 3 * b.kc, q + 4 * b.kc, t + 3 * b.ko, q + 4 * b.ko);
  }
  for (const Spec::DD& d : s.dds) {                                                               // :3086-3272, :1902-1913
    ceres::LossFunction* loss = nullptr;
    if (d.loss >= 0) { losses.emplace_back(new ceres::HuberLoss(d.loss)); loss = losses.back().get(); }
    double* y = &yaw[d.frame]; double* an = &anchor[3 * d.frame];
    if (d.as_base || g_dd_as_cost_function) {
      ceres::CostFunction* c = make_dd(d);
      problem.AddResidualBlock(c, loss, t + 3 * d.i, t + 3 * d.j, y, an);
    } else {
      dd_psr_factor_20* dd_psr_factor = make_dd(d);
      problem.AddResidualBlock(dd_psr_factor, loss, t + 3 * d.i, t + 3 * d.j, y, an);
    }
  }
  for (size_t fi = 0; fi < s.frames.size(); ++fi) {                                               // variable yaw / anchor: held by a prior
    if (!s.frames[fi].yaw_const) {
      PriorN<1>* p = new PriorN<1>(); p->x0[0] = yaw[fi];
      problem.AddResidualBlock(new ceres::AutoDiffCostFunction<PriorN<1>, 1, 1>(p), nullptr, &yaw[fi]);
    }
    if (!s.frames[fi].anchor_const) {
      PriorN<3>* p = new PriorN<3>(); for (int k = 0; k < 3; ++k) p->x0[k] = anchor[3 * fi + k];
      problem.AddResidualBlock(new ceres::AutoDiffCostFunction<PriorN<3>, 3, 3>(p), nullptr, &anchor[3 * fi]);
    }
  }
  if (mode == DESCRIBE) {
    // the trait descriptions and frames, printed exactly (C99 hex floats)
    for (const Spec::DD& d : s.dds) {
      std::unique_ptr<dd_psr_factor_20> f(make_dd(d));
      std::unique_ptr<glio::DdPsrDesc> g(new glio::DdPsrDesc());
      const bool ok = glio::DeviceCostTraits<dd_psr_factor_20>::describe(*f, g.get());
      printf("desc %d %d %d %d %a %a %a %a %a", (int)ok, g->n_sat, g->master, g->w_identity, g->ratio, g->threshold, g->station[0], g->station[1], g->station[2]);
      for (int k = 0; ok && k < g->n_sat; ++k)
        printf(" %a %a %a %a %a %a %a %a", g->sat_user[k][0], g->sat_user[k][1], g->sat_user[k][2], g->psr_user[k], g->sat_ref[k][0], g->sat_ref[k][1], g->sat_ref[k][2], g->psr_ref[k]);
      for (int k = 0; ok && k < (g->n_sat - 1) * (g->n_sat - 1); ++k) printf(" %a", g->W[k]);
      printf("\n");
    }
    for (size_t fi = 0; fi < s.frames.size(); ++fi) {
      double Rf[9];
      glio::DeviceCostTraits<dd_psr_factor_20>::frame(&yaw[fi], &anchor[3 * fi], Rf);
      printf("frame"); for (double v : Rf) printf(" %a", v); printf("\n");
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

static int64_t dd_launches(glio_ctx* ctx) { return launches(ctx, {"k_psr_pair_sums", "k_psr_pair_sums_cost", "k_psr_assemble"}); }
static int64_t pose_launches(glio_ctx* ctx) { return launches(ctx, {"k_pose_pair_sums", "k_pose_pair_sums_cost", "k_pose_assemble"}); }

int main(int argc, char** argv) {
  if (argc < 3) {
    fprintf(stderr, "usage: shim_dd_psr_routes_test host|device|evaluate|describe [--repeat R] [--max-iter M] [--use-pose] [--use-dd] [--preload-dd N] [--dd-as-cost-function] problem.bin...\n");
    return 2;
  }
  const std::string m = argv[1];
  const bool device = m == "device";
  int repeat = 0, preload = 0, max_iter = -1; bool use_pose = false, use_dd = false;
  std::vector<const char*> files;
  for (int i = 2; i < argc; ++i) {
    const std::string a = argv[i];
    if (a == "--repeat" && i + 1 < argc) repeat = atoi(argv[++i]);
    else if (a == "--max-iter" && i + 1 < argc) max_iter = atoi(argv[++i]);
    else if (a == "--use-pose") use_pose = true;
    else if (a == "--use-dd") use_dd = true;
    else if (a == "--preload-dd" && i + 1 < argc) preload = atoi(argv[++i]);
    else if (a == "--dd-as-cost-function") g_dd_as_cost_function = true;
    else files.push_back(argv[i]);
  }
  if (files.empty()) return 2;
  glio_ctx* ctx = nullptr;
  if (device) {
    glio_params prm; glio_default_params(&prm);
    ctx = create_context(prm, !repeat);
    if (preload > 0) {
      // factors between keyframes 1 .. 9 whose satellites sit 1 km from a far-off anchor: any of them evaluated would add cost
      std::vector<glio_dd_psr_factor> f(preload);
      std::vector<glio_dd_psr_sat> sats(3 * (size_t)preload);
      for (int i = 0; i < preload; ++i) {
        glio_dd_psr_factor& x = f[i];
        x.i = 1 + i % 8; x.j = 2 + i % 8; x.n_sat = 3; x.master = i % 3; x.active = 1; x.reserved = 0;
        x.sat_offset = 3 * i; x.w_offset = -1; x.ratio = 0.25; x.threshold = 1e9; x.station[0] = x.station[1] = x.station[2] = 0;
        for (int k = 0; k < 3; ++k) {
          glio_dd_psr_sat& s = sats[3 * i + k];
          for (int c = 0; c < 3; ++c) { s.sat_user[c] = s.sat_ref[c] = (c == k ? 1000.0 : 0.0); }
          s.psr_user = 500.0 * (k + 1); s.psr_ref = 0;
        }
      }
      const double Rp[9] = {0, 1, 0, -1, 0, 0, 0, 0, 1}, ap[3] = {5e5, -2e5, 1e5};
      if (glio_batch_set_dd_psr_factors(ctx, f.data(), preload, sats.data(), (int64_t)sats.size(), nullptr, 0, Rp, ap) != GLIO_OK ||
          glio_batch_use_dd_psr_factors(ctx, 1) != GLIO_OK)
        return 3;
      printf("preload %d\n", preload);
    }
    if (use_pose && glio_batch_use_pose_factors(ctx, 1) != GLIO_OK) return 3;
    if (use_dd && glio_batch_use_dd_psr_factors(ctx, 1) != GLIO_OK) return 3;
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
        printf("time %.6f %d %d %d\n", R.wall_ms, (int)R.summary.iterations.size(), (int)R.summary.termination_type, R.summary.num_device_dd_psr_residual_blocks);
      }
      continue;
    }
    g_gate_margin = std::numeric_limits<double>::infinity();
    const int64_t d0 = dd_launches(ctx), p0 = pose_launches(ctx);
    const Result R = solve(s, ctx, SOLVE, max_iter);
    const int64_t d1 = dd_launches(ctx), p1 = pose_launches(ctx);
    const ceres::Solver::Summary& S = R.summary;
    print_solve_head(S);
    printf("blocks %d\n", S.num_residual_blocks);
    printf("device_blocks %d\n", S.num_device_residual_blocks);
    printf("device_pose %d\n", S.num_device_pose_residual_blocks);
    printf("device_dd %d\n", S.num_device_dd_psr_residual_blocks);
    printf("dd_launches %lld\n", (long long)(d1 - d0));
    printf("pose_launches %lld\n", (long long)(p1 - p0));
    printf("gate_margin %.17g\n", g_gate_margin);
    print_solve_tail(S, s.K, R.t, R.q, nullptr);
  }
  if (ctx) glio_destroy(ctx);
  return 0;
}
