// shim_imu_routes_test.cpp — the Ceres-API shim's route for the batch refinement's IMU factors (K2i): ImuFactor blocks added the
// way optimizeBatchWithLandMark adds them at sms_fusion_level 1 (Estimator.cpp:2794-3001: per keyframe t, q
// (QuaternionParameterization) and speed-bias sb, the attitude factors, the BinaryLidarPlaneNormFactor blocks, then one ImuFactor
// per consecutive keyframe pair), and window-shaped problems (LidarPlaneNormFactor blocks with HuberLoss, the IMU chain and a host
// speed-bias prior).  Used by tests/test_shim_imu_routes.py and scripts/bench_shim_imu_routes.py:
//   shim_imu_routes_test host   [--repeat R] [--max-iter M] problem.bin...   every block evaluated on the host (no GPU needed)
//   shim_imu_routes_test evaluate problem.bin...                              Problem::Evaluate (host): cost, residuals and tangent
//                                                                             gradient
//   shim_imu_routes_test describe problem.bin...                              each IMU block's trait description (glio_imu_factor
//                                                                             from sum_dt on), in hex
//   shim_imu_routes_test device [--repeat R] [--max-iter M] [--use-imu] [--preload-imu N] problem.bin...
//       the described blocks are routed to the GPU; all problems are solved in turn on ONE context, after
//       glio_batch_use_imu_factors(ctx, 1) if asked.  One problem per call is a fresh context.
//       --preload-imu N first leaves what a direct (Level-2) caller would: a list of N other IMU factors and the switch on.
//   --imu-as-cost-function (any mode): every ImuFactor is added through a ceres::CostFunction*, so its blocks stay on the host
// For each problem it prints the iterations, poses, speed-biases and costs (%.17g), the residual and device block counts and the
// K2i, K2p and K2b launches of that solve.  With --repeat R each problem is rebuilt from its file and solved R times, and each
// solve's wall time is printed.
//
// ImuFactor (ImuFactor.h:12-175) and the Preintegration members it reads (Preintegration.h:196-256) are restated without Eigen,
// with Eigen's semantics: Qi.normalize() and Qj.normalize(), inverse() = conj / |q|^2, q * v Eigen's rotation, deltaQ(theta) =
// (1, theta / 2), Qleft / Qright / LeftQuatMatrix (math_tools.h), and at every Evaluate the covariance's inverse (partial-pivot
// LU, as Eigen's inverse() of a 15 x 15 matrix) and its LLT.
#include <algorithm>
#include <chrono>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>

#include "ceres/ceres.h"
#include "shim_driver.h"

// ---- the parts of Eigen the factor and its trait use ---------------------------------------------------------------------------
struct Quaterniond {   // Eigen::Quaterniond, constructed (w, x, y, z)
  double w_, x_, y_, z_;
  double w() const { return w_; } double x() const { return x_; } double y() const { return y_; } double z() const { return z_; }
  double squaredNorm() const { return x_ * x_ + y_ * y_ + z_ * z_ + w_ * w_; }
  void normalize() { const double n = std::sqrt(squaredNorm()); if (n > 0) { w_ /= n; x_ /= n; y_ /= n; z_ /= n; } }
  Quaterniond normalized() const { Quaterniond q = *this; q.normalize(); return q; }
  Quaterniond inverse() const {
    const double n2 = squaredNorm();
    if (n2 > 0) return Quaterniond{w_ / n2, -x_ / n2, -y_ / n2, -z_ / n2};
    return Quaterniond{0, 0, 0, 0};
  }
  Quaterniond operator*(const Quaterniond& b) const {
    return Quaterniond{w_ * b.w_ - x_ * b.x_ - y_ * b.y_ - z_ * b.z_, w_ * b.x_ + x_ * b.w_ + y_ * b.z_ - z_ * b.y_,
                       w_ * b.y_ + y_ * b.w_ + z_ * b.x_ - x_ * b.z_, w_ * b.z_ + z_ * b.w_ + x_ * b.y_ - y_ * b.x_};
  }
};
struct Vec3 { double v[3]; double operator[](int k) const { return v[k]; } };
static Vec3 rotate(const Quaterniond& q, const Vec3& a) {   // Eigen's _transformVector
  double uv[3] = {q.y() * a[2] - q.z() * a[1], q.z() * a[0] - q.x() * a[2], q.x() * a[1] - q.y() * a[0]};
  for (int k = 0; k < 3; ++k) uv[k] += uv[k];
  const double uuv[3] = {q.y() * uv[2] - q.z() * uv[1], q.z() * uv[0] - q.x() * uv[2], q.x() * uv[1] - q.y() * uv[0]};
  return Vec3{{a[0] + q.w() * uv[0] + uuv[0], a[1] + q.w() * uv[1] + uuv[1], a[2] + q.w() * uv[2] + uuv[2]}};
}
static void to_rotation_matrix(const Quaterniond& q, double R[9]) {   // Eigen's toRotationMatrix()
  const double tx = 2 * q.x(), ty = 2 * q.y(), tz = 2 * q.z();
  const double twx = tx * q.w(), twy = ty * q.w(), twz = tz * q.w(), txx = tx * q.x(), txy = ty * q.x(), txz = tz * q.x();
  const double tyy = ty * q.y(), tyz = tz * q.y(), tzz = tz * q.z();
  const double M[9] = {1 - (tyy + tzz), txy - twz, txz + twy, txy + twz, 1 - (txx + tzz), tyz - twx, txz - twy, tyz + twx, 1 - (txx + tyy)};
  std::memcpy(R, M, sizeof(M));
}
static void skew(const double* v, double S[9]) {   // skewSymmetric
  const double M[9] = {0, -v[2], v[1], v[2], 0, -v[0], -v[1], v[0], 0};
  std::memcpy(S, M, sizeof(M));
}
static void qleft(const Quaterniond& q, double M[16]) {   // Qleft: [w, -v^T; v, w I + [v]x], over (w, x, y, z)
  const double v[3] = {q.x(), q.y(), q.z()};
  double S[9]; skew(v, S);
  M[0] = q.w(); for (int k = 0; k < 3; ++k) { M[1 + k] = -v[k]; M[4 * (1 + k)] = v[k]; }
  for (int r = 0; r < 3; ++r) for (int c = 0; c < 3; ++c) M[4 * (1 + r) + 1 + c] = (r == c ? q.w() : 0.0) + S[3 * r + c];
}
static void qright(const Quaterniond& p, double M[16]) {   // Qright: [w, -v^T; v, w I - [v]x]
  const double v[3] = {p.x(), p.y(), p.z()};
  double S[9]; skew(v, S);
  M[0] = p.w(); for (int k = 0; k < 3; ++k) { M[1 + k] = -v[k]; M[4 * (1 + k)] = v[k]; }
  for (int r = 0; r < 3; ++r) for (int c = 0; c < 3; ++c) M[4 * (1 + r) + 1 + c] = (r == c ? p.w() : 0.0) - S[3 * r + c];
}
static void left_quat_top_left(const Quaterniond& q, double M[9]) {   // LeftQuatMatrix(q).topLeftCorner<3, 3>() = w I + [v]x
  const double v[3] = {q.x(), q.y(), q.z()};
  skew(v, M);
  for (int k = 0; k < 3; ++k) M[4 * k] += q.w();
}
typedef std::vector<double> Mat;   // row-major, dimensions at the use
static Mat matmul(const Mat& A, const Mat& B, int n, int m, int p) {   // (n x m) (m x p)
  Mat C((size_t)n * p, 0.0);
  for (int i = 0; i < n; ++i) for (int j = 0; j < p; ++j) { double s = 0; for (int k = 0; k < m; ++k) s += A[(size_t)i * m + k] * B[(size_t)k * p + j]; C[(size_t)i * p + j] = s; }
  return C;
}
// Eigen's inverse() of a 15 x 15 matrix: PartialPivLU (row pivoting on the largest magnitude), then the solve against I
static Mat inverse15(const Mat& A0) {
  const int n = 15;
  Mat A = A0; int perm[15];
  for (int k = 0; k < n; ++k) perm[k] = k;
  for (int k = 0; k < n; ++k) {
    int piv = k;
    for (int i = k + 1; i < n; ++i) if (std::fabs(A[i * n + k]) > std::fabs(A[piv * n + k])) piv = i;
    if (piv != k) { for (int c = 0; c < n; ++c) std::swap(A[k * n + c], A[piv * n + c]); std::swap(perm[k], perm[piv]); }
    if (A[k * n + k] != 0)
      for (int i = k + 1; i < n; ++i) {
        A[i * n + k] /= A[k * n + k];
        for (int c = k + 1; c < n; ++c) A[i * n + c] -= A[i * n + k] * A[k * n + c];
      }
  }
  Mat X((size_t)n * n, 0.0);
  for (int col = 0; col < n; ++col) {
    double y[15];
    for (int i = 0; i < n; ++i) { y[i] = perm[i] == col ? 1.0 : 0.0; for (int k = 0; k < i; ++k) y[i] -= A[i * n + k] * y[k]; }
    for (int i = n - 1; i >= 0; --i) { for (int k = i + 1; k < n; ++k) y[i] -= A[i * n + k] * y[k]; y[i] /= A[i * n + i]; }
    for (int i = 0; i < n; ++i) X[i * n + col] = y[i];
  }
  return X;
}
// LLT<Matrix<double, 15, 15>>(A).matrixL().transpose(): the lower Cholesky factor of A's lower triangle, transposed.  As Eigen's
// unblocked LLT, a pivot that is not positive stops the factorisation and leaves the rest of the lower triangle as it was.
static Mat llt_upper15(const Mat& A) {
  const int n = 15;
  Mat L((size_t)n * n, 0.0);
  for (int i = 0; i < n; ++i) for (int j = 0; j <= i; ++j) L[i * n + j] = A[i * n + j];
  for (int k = 0; k < n; ++k) {
    double x = L[k * n + k];
    for (int j = 0; j < k; ++j) x -= L[k * n + j] * L[k * n + j];
    if (!(x > 0)) break;
    L[k * n + k] = std::sqrt(x);
    for (int i = k + 1; i < n; ++i) {
      double s = L[i * n + k];
      for (int j = 0; j < k; ++j) s -= L[i * n + j] * L[k * n + j];
      L[i * n + k] = s / L[k * n + k];
    }
  }
  Mat U((size_t)n * n);
  for (int i = 0; i < n; ++i) for (int j = 0; j < n; ++j) U[i * n + j] = L[j * n + i];
  return U;
}

// ---- Preintegration (the members ImuFactor reads) and ImuFactor, restated ----------------------------------------------------------
enum { O_P = 0, O_R = 3, O_V = 6, O_BA = 9, O_BG = 12 };
struct Preintegration {
  Vec3 linearized_ba_, linearized_bg_;
  Mat jacobian_ = Mat(225, 0.0), covariance_ = Mat(225, 0.0);   // 15 x 15, row-major
  double sum_dt_ = 0;
  Vec3 delta_p_;
  Quaterniond delta_q_{1, 0, 0, 0};
  Vec3 delta_v_;
  Vec3 g_vec_;
  void block(int r0, int c0, double* out) const { for (int r = 0; r < 3; ++r) for (int c = 0; c < 3; ++c) out[3 * r + c] = jacobian_[15 * (r0 + r) + c0 + c]; }
  // Preintegration::evaluate (Preintegration.h:196-235)
  void evaluate(const Vec3& Pi, const Quaterniond& Qi, const Vec3& Vi, const Vec3& Bai, const Vec3& Bgi, const Vec3& Pj, const Quaterniond& Qj,
                const Vec3& Vj, const Vec3& Baj, const Vec3& Bgj, double* r) const {
    double dp_dba[9], dp_dbg[9], dq_dbg[9], dv_dba[9], dv_dbg[9];
    block(O_P, O_BA, dp_dba); block(O_P, O_BG, dp_dbg); block(O_R, O_BG, dq_dbg); block(O_V, O_BA, dv_dba); block(O_V, O_BG, dv_dbg);
    double dba[3], dbg[3];
    for (int k = 0; k < 3; ++k) { dba[k] = Bai[k] - linearized_ba_[k]; dbg[k] = Bgi[k] - linearized_bg_[k]; }
    const Quaterniond cdq = delta_q_ * delta_Q(dq_dbg, dbg);
    double cdv[3], cdp[3];
    for (int m = 0; m < 3; ++m) {
      double a = 0, b = 0, c = 0, d = 0;
      for (int k = 0; k < 3; ++k) { a += dv_dba[3 * m + k] * dba[k]; b += dv_dbg[3 * m + k] * dbg[k]; c += dp_dba[3 * m + k] * dba[k]; d += dp_dbg[3 * m + k] * dbg[k]; }
      cdv[m] = delta_v_[m] + a + b; cdp[m] = delta_p_[m] + c + d;
    }
    const Quaterniond qii = Qi.inverse();
    Vec3 tp, tv;
    for (int k = 0; k < 3; ++k) {
      tp.v[k] = -0.5 * g_vec_[k] * sum_dt_ * sum_dt_ + Pj[k] - Pi[k] - Vi[k] * sum_dt_;
      tv.v[k] = -g_vec_[k] * sum_dt_ + Vj[k] - Vi[k];
    }
    const Vec3 rp = rotate(qii, tp), rv = rotate(qii, tv);
    const Quaterniond e = (cdq.inverse() * (qii * Qj)).normalized();
    const double ev[3] = {e.x(), e.y(), e.z()};
    for (int k = 0; k < 3; ++k) {
      r[O_P + k] = rp[k] - cdp[k]; r[O_R + k] = 2.0 * ev[k]; r[O_V + k] = rv[k] - cdv[k];
      r[O_BA + k] = Baj[k] - Bai[k]; r[O_BG + k] = Bgj[k] - Bgi[k];
    }
  }
  // deltaQ(dq_dbg dbg) (math_tools.h:126-138)
  static Quaterniond delta_Q(const double* M, const double* v) {
    double th[3];
    for (int m = 0; m < 3; ++m) th[m] = M[3 * m] * v[0] + M[3 * m + 1] * v[1] + M[3 * m + 2] * v[2];
    return Quaterniond{1.0, th[0] / 2.0, th[1] / 2.0, th[2] / 2.0};
  }
  Mat sqrt_info() const { return llt_upper15(inverse15(covariance_)); }
};

static bool g_imu_as_cost_function = false;   // --imu-as-cost-function

class ImuFactor : public ceres::SizedCostFunction<15, 3, 4, 9, 3, 4, 9> {
 public:
  explicit ImuFactor(Preintegration* pre_integration) : pre_integration_{pre_integration} { g_vec_ = pre_integration_->g_vec_; }
  bool Evaluate(double const* const* parameters, double* residuals, double** jacobians) const override {
    const double* p = parameters[0]; const double* s = parameters[2]; const double* pj = parameters[3]; const double* sj = parameters[5];
    const Vec3 Pi{{p[0], p[1], p[2]}}, Vi{{s[0], s[1], s[2]}}, Bai{{s[3], s[4], s[5]}}, Bgi{{s[6], s[7], s[8]}};
    const Vec3 Pj{{pj[0], pj[1], pj[2]}}, Vj{{sj[0], sj[1], sj[2]}}, Baj{{sj[3], sj[4], sj[5]}}, Bgj{{sj[6], sj[7], sj[8]}};
    Quaterniond Qi{parameters[1][0], parameters[1][1], parameters[1][2], parameters[1][3]}; Qi.normalize();
    Quaterniond Qj{parameters[4][0], parameters[4][1], parameters[4][2], parameters[4][3]}; Qj.normalize();
    const Preintegration& P = *pre_integration_;
    Mat raw(15);
    P.evaluate(Pi, Qi, Vi, Bai, Bgi, Pj, Qj, Vj, Baj, Bgj, raw.data());
    const Mat S = P.sqrt_info();
    const Mat r = matmul(S, raw, 15, 15, 1);
    std::copy(r.begin(), r.end(), residuals);
    if (!jacobians) return true;
    const double T = P.sum_dt_;
    double dp_dba[9], dp_dbg[9], dq_dbg[9], dv_dba[9], dv_dbg[9];
    P.block(O_P, O_BA, dp_dba); P.block(O_P, O_BG, dp_dbg); P.block(O_R, O_BG, dq_dbg); P.block(O_V, O_BA, dv_dba); P.block(O_V, O_BG, dv_dbg);
    double R[9];
    to_rotation_matrix(Qi.inverse(), R);
    double dbg[3];
    for (int k = 0; k < 3; ++k) dbg[k] = Bgi[k] - P.linearized_bg_[k];
    const Quaterniond cdq = P.delta_q_ * Preintegration::delta_Q(dq_dbg, dbg);
    auto put = [](Mat& J, int nc, int r0, int c0, const double* B, double sc) {
      for (int r = 0; r < 3; ++r) for (int c = 0; c < 3; ++c) J[(size_t)(r0 + r) * nc + c0 + c] = sc * B[3 * r + c];
    };
    const double I3[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1};
    auto out = [&](int b, const Mat& J, int nc) { const Mat SJ = matmul(S, J, 15, 15, nc); std::copy(SJ.begin(), SJ.end(), jacobians[b]); };
    if (jacobians[0]) { Mat J(45, 0.0); put(J, 3, O_P, O_P, R, -1.0); out(0, J, 3); }
    if (jacobians[1]) {
      Mat J(60, 0.0);
      const double qv[3] = {Qi.x(), Qi.y(), Qi.z()};
      auto qi_rows = [&](int r0, const double* t) {   // 2 (w t + [v]x t) and 2 (v.t I + v t^T - t v^T - w [t]x)
        double Sv[9], St[9]; skew(qv, Sv); skew(t, St);
        const double vt = qv[0] * t[0] + qv[1] * t[1] + qv[2] * t[2];
        for (int m = 0; m < 3; ++m) {
          J[(size_t)(r0 + m) * 4] = 2 * (Qi.w() * t[m] + (Sv[3 * m] * t[0] + Sv[3 * m + 1] * t[1] + Sv[3 * m + 2] * t[2]));
          for (int c = 0; c < 3; ++c) J[(size_t)(r0 + m) * 4 + 1 + c] = 2 * ((m == c ? vt : 0.0) + qv[m] * t[c] - t[m] * qv[c] - Qi.w() * St[3 * m + c]);
        }
      };
      double tp[3], tv[3];
      for (int k = 0; k < 3; ++k) { tp[k] = -0.5 * g_vec_[k] * T * T + Pj[k] - Pi[k] - Vi[k] * T; tv[k] = -g_vec_[k] * T + Vj[k] - Vi[k]; }
      qi_rows(O_P, tp);
      double A[16], B[16];
      qleft(Qj.inverse(), A); qright(cdq, B);
      const Mat AB = matmul(Mat(A, A + 16), Mat(B, B + 16), 4, 4, 4);
      for (int m = 0; m < 3; ++m) for (int c = 0; c < 4; ++c) J[(size_t)(O_R + m) * 4 + c] = -2 * AB[4 * (1 + m) + c];
      qi_rows(O_V, tv);
      out(1, J, 4);
    }
    if (jacobians[2]) {
      Mat J(135, 0.0);
      double RT[9]; for (int k = 0; k < 9; ++k) RT[k] = R[k] * T;
      put(J, 9, O_P, O_V - O_V, RT, -1.0); put(J, 9, O_P, O_BA - O_V, dp_dba, -1.0); put(J, 9, O_P, O_BG - O_V, dp_dbg, -1.0);
      double L[9]; left_quat_top_left(Qj.inverse() * Qi * cdq, L);
      const Mat Ld = matmul(Mat(L, L + 9), Mat(dq_dbg, dq_dbg + 9), 3, 3, 3);
      put(J, 9, O_R, O_BG - O_V, Ld.data(), -1.0);
      put(J, 9, O_V, O_V - O_V, R, -1.0); put(J, 9, O_V, O_BA - O_V, dv_dba, -1.0); put(J, 9, O_V, O_BG - O_V, dv_dbg, -1.0);
      put(J, 9, O_BA, O_BA - O_V, I3, -1.0); put(J, 9, O_BG, O_BG - O_V, I3, -1.0);
      out(2, J, 9);
    }
    if (jacobians[3]) { Mat J(45, 0.0); put(J, 3, O_P, O_P, R, 1.0); out(3, J, 3); }
    if (jacobians[4]) {
      Mat J(60, 0.0);
      double A[16]; qleft(cdq.inverse() * Qi.inverse(), A);
      for (int m = 0; m < 3; ++m) for (int c = 0; c < 4; ++c) J[(size_t)(O_R + m) * 4 + c] = 2 * A[4 * (1 + m) + c];
      out(4, J, 4);
    }
    if (jacobians[5]) {
      Mat J(135, 0.0);
      put(J, 9, O_V, O_V - O_V, R, 1.0); put(J, 9, O_BA, O_BA - O_V, I3, 1.0); put(J, 9, O_BG, O_BG - O_V, I3, 1.0);
      out(5, J, 9);
    }
    return true;
  }
  Preintegration* pre_integration_;
  Vec3 g_vec_;
};

// ---- what a maintainer adds next to ImuFactor.h (INTEGRATION.md, Level 1) --------------------------------------------------------
namespace glio {
template <> struct DeviceCostTraits<ImuFactor> {
  static bool describe(const ImuFactor& f, glio_imu_factor* d) {
    const Preintegration& p = *f.pre_integration_;
    d->sum_dt = p.sum_dt_;
    for (int k = 0; k < 3; ++k) {
      d->g_vec[k] = p.g_vec_[k]; d->delta_p[k] = p.delta_p_[k]; d->delta_v[k] = p.delta_v_[k];
      d->linearized_ba[k] = p.linearized_ba_[k]; d->linearized_bg[k] = p.linearized_bg_[k];
    }
    d->delta_q[0] = p.delta_q_.w(); d->delta_q[1] = p.delta_q_.x(); d->delta_q[2] = p.delta_q_.y(); d->delta_q[3] = p.delta_q_.z();
    p.block(O_P, O_BA, d->dp_dba); p.block(O_P, O_BG, d->dp_dbg); p.block(O_R, O_BG, d->dq_dbg); p.block(O_V, O_BA, d->dv_dba); p.block(O_V, O_BG, d->dv_dbg);
    const Mat S = p.sqrt_info();   // LLT(covariance_.inverse()).matrixL().transpose(), as the factor forms it
    std::copy(S.begin(), S.end(), d->sqrt_info);
    return true;
  }
};
}  // namespace glio

// ---- the attitude, binary-plane and LidarPlaneNormFactor functors of the other route drivers, with their traits -----------------
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
namespace glio {
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

// a host prior on one keyframe's speed-bias (the window's marginalisation prior stand-in): r = w (sb - sb0)
struct SbPrior {
  double sb0[9], w;
  template <typename T> bool operator()(const T* sb, T* r) const { for (int k = 0; k < 9; ++k) r[k] = T(w) * (sb[k] - T(sb0[k])); return true; }
};

// one problem file (written by tests/test_shim_imu_routes.py: write_problem)
struct Spec {
  int32_t K = 0;
  std::vector<double> poses, sb, q_alt;
  std::vector<int32_t> t_const, q_const, sb_const;
  struct Att { int32_t i, j; double dq[4]; };
  std::vector<Att> att;
  struct Bin { int32_t kc, ko; double cp[3], nc[6], score; };
  std::vector<Bin> bin;
  struct Plane { int32_t k; double cp[3], n[3], d, score, qlb[4], tlb[3], loss; };
  std::vector<Plane> planes;
  struct Prior { int32_t k; double sb0[9], w; };
  std::vector<Prior> priors;
  // sb_i / sb_j: the keyframe whose sb block each side uses; alt_q >= 0: q_i is extra q block alt_q; loss >= 0: HuberLoss(loss)
  struct Imu { int32_t i, j, sb_i, sb_j, alt_q, as_base; double loss, sum_dt, g[3], dp[3], dq[4], dv[3], ba[3], bg[3], jac[5][9], cov[225]; };
  std::vector<Imu> imu;
  int32_t max_iter = 10;
  double time_limit = 1e9;
};

static Spec read_spec(const char* path) {
  FILE* f = fopen(path, "rb");
  if (!f) { fprintf(stderr, "cannot open %s\n", path); exit(2); }
  Spec s;
  int32_t n_alt, n;
  rd(f, &s.K, 1); rd(f, &n_alt, 1);
  s.poses.resize(7 * (size_t)s.K); rd(f, s.poses.data(), s.poses.size());
  s.sb.resize(9 * (size_t)s.K); rd(f, s.sb.data(), s.sb.size());
  for (auto* c : {&s.t_const, &s.q_const, &s.sb_const}) { c->resize(s.K); rd(f, c->data(), s.K); }
  s.q_alt.resize(4 * (size_t)n_alt); rd(f, s.q_alt.data(), s.q_alt.size());
  rd(f, &n, 1); s.att.resize(n);
  for (auto& a : s.att) { rd(f, &a.i, 1); rd(f, &a.j, 1); rd(f, a.dq, 4); }
  rd(f, &n, 1); s.bin.resize(n);
  for (auto& b : s.bin) { rd(f, &b.kc, 1); rd(f, &b.ko, 1); rd(f, b.cp, 3); rd(f, b.nc, 6); rd(f, &b.score, 1); }
  rd(f, &n, 1); s.planes.resize(n);
  for (auto& p : s.planes) { rd(f, &p.k, 1); rd(f, p.cp, 3); rd(f, p.n, 3); rd(f, &p.d, 1); rd(f, &p.score, 1); rd(f, p.qlb, 4); rd(f, p.tlb, 3); rd(f, &p.loss, 1); }
  rd(f, &n, 1); s.priors.resize(n);
  for (auto& p : s.priors) { rd(f, &p.k, 1); rd(f, p.sb0, 9); rd(f, &p.w, 1); }
  rd(f, &n, 1); s.imu.resize(n);
  for (auto& m : s.imu) {
    rd(f, &m.i, 1); rd(f, &m.j, 1); rd(f, &m.sb_i, 1); rd(f, &m.sb_j, 1); rd(f, &m.alt_q, 1); rd(f, &m.as_base, 1); rd(f, &m.loss, 1);
    rd(f, &m.sum_dt, 1); rd(f, m.g, 3); rd(f, m.dp, 3); rd(f, m.dq, 4); rd(f, m.dv, 3); rd(f, m.ba, 3); rd(f, m.bg, 3);
    rd(f, &m.jac[0][0], 45); rd(f, m.cov, 225);
  }
  rd(f, &s.max_iter, 1); rd(f, &s.time_limit, 1);
  fclose(f);
  return s;
}

// the Preintegration a record stands for: jacobian_ is the identity with the five blocks ImuFactor reads
static Preintegration make_pre(const Spec::Imu& m) {
  Preintegration p;
  p.sum_dt_ = m.sum_dt;
  for (int k = 0; k < 3; ++k) {
    p.g_vec_.v[k] = m.g[k]; p.delta_p_.v[k] = m.dp[k]; p.delta_v_.v[k] = m.dv[k]; p.linearized_ba_.v[k] = m.ba[k]; p.linearized_bg_.v[k] = m.bg[k];
  }
  p.delta_q_ = Quaterniond{m.dq[0], m.dq[1], m.dq[2], m.dq[3]};
  for (int k = 0; k < 15; ++k) p.jacobian_[16 * k] = 1.0;
  const int at[5][2] = {{O_P, O_BA}, {O_P, O_BG}, {O_R, O_BG}, {O_V, O_BA}, {O_V, O_BG}};   // dp_dba, dp_dbg, dq_dbg, dv_dba, dv_dbg
  for (int b = 0; b < 5; ++b)
    for (int r = 0; r < 3; ++r) for (int c = 0; c < 3; ++c) p.jacobian_[15 * (at[b][0] + r) + at[b][1] + c] = m.jac[b][3 * r + c];
  std::copy(m.cov, m.cov + 225, p.covariance_.begin());
  return p;
}

struct Result { ceres::Solver::Summary summary; std::vector<double> t, q, sb, residuals, gradient; double wall_ms = 0, cost = 0; };

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
  std::vector<double> q_alt = s.q_alt;
  std::vector<Preintegration> pre(s.imu.size());
  for (size_t n = 0; n < s.imu.size(); ++n) pre[n] = make_pre(s.imu[n]);
  if (mode == DESCRIBE) {
    // the trait descriptions, printed exactly (C99 hex floats): the glio_imu_factor doubles from sum_dt on, in record order
    for (size_t n = 0; n < s.imu.size(); ++n) {
      ImuFactor f(&pre[n]);
      glio_imu_factor d;
      std::memset(&d, 0, sizeof(d));
      const bool ok = glio::DeviceCostTraits<ImuFactor>::describe(f, &d);
      printf("desc %d %d %d %d", (int)ok, d.i, d.j, d.active);
      const double* v = &d.sum_dt;
      for (size_t k = 0; k < (sizeof(d) - offsetof(glio_imu_factor, sum_dt)) / sizeof(double); ++k) printf(" %a", v[k]);
      printf("\n");
    }
    return R;
  }
  ceres::Problem::Options po;
  po.loss_function_ownership = ceres::DO_NOT_TAKE_OWNERSHIP;
  std::vector<std::unique_ptr<ceres::LossFunction>> losses;
  auto loss_for = [&](double a) -> ceres::LossFunction* {
    if (a < 0) return nullptr;
    losses.emplace_back(new ceres::HuberLoss(a));
    return losses.back().get();
  };
  ceres::Problem problem(po);
  problem.SetGlioContext(ctx);
  ceres::LocalParameterization* quat = new ceres::QuaternionParameterization();                  // one object, as the reference
  for (int k = 0; k < K; ++k) {                                                                   // Estimator.cpp:2794-2821
    problem.AddParameterBlock(t + 3 * k, 3);
    problem.AddParameterBlock(q + 4 * k, 4, quat);
    problem.AddParameterBlock(sb + 9 * k, 9);
    if (s.t_const[k]) problem.SetParameterBlockConstant(t + 3 * k);
    if (s.q_const[k]) problem.SetParameterBlockConstant(q + 4 * k);
    if (s.sb_const[k]) problem.SetParameterBlockConstant(sb + 9 * k);
  }
  for (size_t a = 0; a < q_alt.size() / 4; ++a) problem.AddParameterBlock(&q_alt[4 * a], 4, quat);
  for (const Spec::Att& a : s.att)                                                                // :2861-2863
    problem.AddResidualBlock(new ceres::AutoDiffCostFunction<delta_q_factor_auto, 3, 4, 4>(
                                 new delta_q_factor_auto(Quaterniond{a.dq[0], a.dq[1], a.dq[2], a.dq[3]})),
                             nullptr, q + 4 * a.i, q + 4 * a.j);
  for (const Spec::Bin& b : s.bin) {                                                              // :2768
    BinaryLidarPlaneNormFactor* f = new BinaryLidarPlaneNormFactor();
    for (int k = 0; k < 3; ++k) f->curr_point[k] = b.cp[k];
    for (int k = 0; k < 6; ++k) f->planet_norm_cent[k] = b.nc[k];
    f->score = b.score;
    problem.AddResidualBlock(new ceres::AutoDiffCostFunction<BinaryLidarPlaneNormFactor, 1, 3, 4, 3, 4>(f), nullptr, t + 3 * b.kc, q + 4 * b.kc, t + 3 * b.ko, q + 4 * b.ko);
  }
  for (const Spec::Plane& p : s.planes) {                                                         // the window's plane blocks
    LidarPlaneNormFactor* f = new LidarPlaneNormFactor();
    for (int k = 0; k < 3; ++k) { f->curr_point[k] = p.cp[k]; f->plane_unit_norm[k] = p.n[k]; f->tlb[k] = p.tlb[k]; }
    for (int k = 0; k < 4; ++k) f->qlb[k] = p.qlb[k];
    f->negative_OA_dot_norm = p.d; f->score = p.score;
    problem.AddResidualBlock(new ceres::AutoDiffCostFunction<LidarPlaneNormFactor, 1, 3, 4>(f), loss_for(p.loss), t + 3 * p.k, q + 4 * p.k);
  }
  for (size_t n = 0; n < s.imu.size(); ++n) {                                                     // :2993-3001
    const Spec::Imu& m = s.imu[n];
    double* qi = m.alt_q >= 0 ? &q_alt[4 * m.alt_q] : q + 4 * m.i;
    if (m.as_base || g_imu_as_cost_function) {
      ceres::CostFunction* c = new ImuFactor(&pre[n]);
      problem.AddResidualBlock(c, loss_for(m.loss), t + 3 * m.i, qi, sb + 9 * m.sb_i, t + 3 * m.j, q + 4 * m.j, sb + 9 * m.sb_j);
    } else {
      ImuFactor* imu_factor = new ImuFactor(&pre[n]);
      problem.AddResidualBlock(imu_factor, loss_for(m.loss), t + 3 * m.i, qi, sb + 9 * m.sb_i, t + 3 * m.j, q + 4 * m.j, sb + 9 * m.sb_j);
    }
  }
  for (const Spec::Prior& p : s.priors) {
    SbPrior* f = new SbPrior(); std::copy(p.sb0, p.sb0 + 9, f->sb0); f->w = p.w;
    problem.AddResidualBlock(new ceres::AutoDiffCostFunction<SbPrior, 9, 9>(f), nullptr, sb + 9 * p.k);
  }
  if (mode == EVALUATE) {
    problem.Evaluate(ceres::Problem::EvaluateOptions(), &R.cost, &R.residuals, &R.gradient, nullptr);
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

static int64_t imu_launches(glio_ctx* ctx) { return launches(ctx, {"k_imu_pair_sums", "k_imu_pair_sums_cost", "k_imu_assemble"}); }
static int64_t pose_launches(glio_ctx* ctx) { return launches(ctx, {"k_pose_pair_sums", "k_pose_pair_sums_cost", "k_pose_assemble"}); }

int main(int argc, char** argv) {
  if (argc < 3) {
    fprintf(stderr, "usage: shim_imu_routes_test host|device|evaluate|describe [--repeat R] [--max-iter M] [--use-imu] [--preload-imu N] [--imu-as-cost-function] problem.bin...\n");
    return 2;
  }
  const std::string m = argv[1];
  const bool device = m == "device";
  int repeat = 0, preload = 0, max_iter = -1; bool use_imu = false;
  std::vector<const char*> files;
  for (int i = 2; i < argc; ++i) {
    const std::string a = argv[i];
    if (a == "--repeat" && i + 1 < argc) repeat = atoi(argv[++i]);
    else if (a == "--max-iter" && i + 1 < argc) max_iter = atoi(argv[++i]);
    else if (a == "--use-imu") use_imu = true;
    else if (a == "--preload-imu" && i + 1 < argc) preload = atoi(argv[++i]);
    else if (a == "--imu-as-cost-function") g_imu_as_cost_function = true;
    else files.push_back(argv[i]);
  }
  if (files.empty()) return 2;
  glio_ctx* ctx = nullptr;
  if (device) {
    glio_params prm; glio_default_params(&prm);
    ctx = create_context(prm, !repeat);
    if (preload > 0) {
      // factors between keyframes 1 .. 9 with a large gravity and unit information: any of them evaluated would add cost
      std::vector<glio_imu_factor> f(preload);
      for (int i = 0; i < preload; ++i) {
        glio_imu_factor& x = f[i];
        std::memset(&x, 0, sizeof(x));
        x.i = 1 + i % 8; x.j = 2 + i % 8; x.active = 1;
        x.sum_dt = 0.5; x.g_vec[2] = 100.0 + i; x.delta_q[0] = 1.0;
        for (int k = 0; k < 15; ++k) x.sqrt_info[16 * k] = 1.0;
      }
      if (glio_batch_set_imu_factors(ctx, f.data(), preload) != GLIO_OK || glio_batch_use_imu_factors(ctx, 1) != GLIO_OK) return 3;
      printf("preload %d\n", preload);
    }
    if (use_imu && glio_batch_use_imu_factors(ctx, 1) != GLIO_OK) return 3;
  }
  for (size_t fi = 0; fi < files.size(); ++fi) {
    const Spec s = read_spec(files[fi]);
    printf("solve %d\n", (int)fi);
    if (m == "evaluate") {
      const Result R = solve(s, nullptr, EVALUATE);
      printf("eval_cost %.17g\n", R.cost);
      printf("residuals"); for (double v : R.residuals) printf(" %.17g", v); printf("\n");
      printf("gradient"); for (double v : R.gradient) printf(" %.17g", v); printf("\n");
      continue;
    }
    if (m == "describe") { solve(s, nullptr, DESCRIBE); continue; }
    if (repeat) {
      for (int r = 0; r < repeat; ++r) {
        const Result R = solve(s, ctx, SOLVE, max_iter);
        printf("time %.6f %d %d %d %d\n", R.wall_ms, (int)R.summary.iterations.size(), (int)R.summary.termination_type,
               R.summary.num_device_imu_residual_blocks, R.summary.num_device_residual_blocks);
      }
      continue;
    }
    const int64_t i0 = imu_launches(ctx), p0 = pose_launches(ctx), b0 = launches(ctx, {"k_eval_binary"});
    const Result R = solve(s, ctx, SOLVE, max_iter);
    const int64_t i1 = imu_launches(ctx), p1 = pose_launches(ctx), b1 = launches(ctx, {"k_eval_binary"});
    const ceres::Solver::Summary& S = R.summary;
    print_solve_head(S);
    printf("blocks %d\n", S.num_residual_blocks);
    printf("device_blocks %d\n", S.num_device_residual_blocks);
    printf("device_pose %d\n", S.num_device_pose_residual_blocks);
    printf("device_imu %d\n", S.num_device_imu_residual_blocks);
    printf("imu_launches %lld\n", (long long)(i1 - i0));
    printf("pose_launches %lld\n", (long long)(p1 - p0));
    printf("binary_launches %lld\n", (long long)(b1 - b0));
    print_solve_tail(S, s.K, R.t, R.q, &R.sb);
  }
  if (ctx) glio_destroy(ctx);
  return 0;
}
