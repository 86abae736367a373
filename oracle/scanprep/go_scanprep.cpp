/*
 * go_scanprep.cpp — CPU restatement ("oracle") of the front end's sweep preparation: Preprocessing::cloudHandler,
 * GLIO/src/Preprocessing.cpp:387-526, with undistortion (:176-200) and processIMU / solveRotation (:202-259).
 *
 * TEST INFRASTRUCTURE ONLY.  Nothing under glio_b200/ may include, link or call this; tests/ and scripts/bench_frontend.py
 * use it through oracle/pyoracle_scanprep.py.  It is written from the reference source as a literal, sequential restatement:
 * one pass in input order, halfPassed as a flag, one std::vector per ring, the reference's float / double types at every step.
 * Eigen 3.3 (slerp, quaternion product, inverse, _transformVector) is restated in scalar code.
 *
 * PARITY UNPINNED (no library in the image can check these):
 *   - atanf / atan2f.  The reference calls libm's float overloads; whether glibc rounds them correctly depends on its version.
 *     This oracle returns the correctly rounded float: the double libm result rounded to float, and inside a guard band of
 *     2^-40 relative around a float rounding boundary the long double result rounded to float.  The device decides the same
 *     cases in double-double (about 104 bits).  The x87 long double has a 64-bit significand and is then rounded to float a
 *     second time, so for an argument whose angle lies within about 2^-63 relative of a float midpoint this oracle, not the
 *     device, may round the wrong way.  No test input comes near that; tests/test_scan_prep.py checks the oracle against
 *     np.longdouble, which shares the limitation.
 *   - sin((1-t) theta) and sin(t theta) of Eigen's slerp: libm double sin here, the device's double sin there (xyz <= 1 float ulp).
 *   - Eigen's SSE2 quaternion product (Geometry/arch/Geometry_SSE.h) groups the sums of a * b differently from the generic
 *     quat_product restated here (Quaternion.h); likewise the packet order of dot() and squaredNorm().  With the identity
 *     extrinsic of the shipped configuration every such product is exact.
 *
 * Floating point: compiled with -ffp-contract=off (no FMA contraction), like the reference's baseline x86-64 build.
 */
#include <stdint.h>

#include <cfloat>
#include <cmath>
#include <vector>

/* ---- correctly rounded atan2f / atanf ---- */
static long long g_guard_hits = 0;

// float nearest to the angle whose double libm value is d; `slow` gives it in long double inside the guard band
template <class F>
static float cr_round(double d, F slow) {
  const float f = (float)d;
  if ((double)f == d) return f;
  float lo, hi;
  if ((double)f < d) { lo = f; hi = std::nextafter(f, INFINITY); } else { hi = f; lo = std::nextafter(f, -INFINITY); }
  const double m = ((double)lo + (double)hi) * 0.5;
  if (std::fabs(d - m) > std::fabs(m) * 0x1p-40) return f;
  ++g_guard_hits;
  return (float)slow();
}

extern "C" {

float go_cr_atan2f(float y, float x) {
  return cr_round(std::atan2((double)y, (double)x), [&] { return atan2l((long double)y, (long double)x); });
}
float go_cr_atanf(float a) {
  return cr_round(std::atan((double)a), [&] { return atanl((long double)a); });
}
long long go_cr_guard_hits(int reset) { const long long h = g_guard_hits; if (reset) g_guard_hits = 0; return h; }
void go_cr_atan2f_n(const float* y, const float* x, int64_t n, float* out) { for (int64_t i = 0; i < n; ++i) out[i] = go_cr_atan2f(y[i], x[i]); }
void go_cr_atanf_n(const float* a, int64_t n, float* out) { for (int64_t i = 0; i < n; ++i) out[i] = go_cr_atanf(a[i]); }
/* the host libm's own float overloads, for reporting how often they differ from the correctly rounded value */
void go_libm_atan2f_n(const float* y, const float* x, int64_t n, float* out) { for (int64_t i = 0; i < n; ++i) out[i] = atan2f(y[i], x[i]); }
void go_libm_atanf_n(const float* a, int64_t n, float* out) { for (int64_t i = 0; i < n; ++i) out[i] = atanf(a[i]); }

}  // extern "C"

namespace {

struct Quat { double w, x, y, z; };   // Eigen::Quaterniond, coeffs() = x, y, z, w

Quat qmul(const Quat& a, const Quat& b) {   // Eigen Quaternion.h quat_product (generic)
  return {a.w * b.w - a.x * b.x - a.y * b.y - a.z * b.z,
          a.w * b.x + a.x * b.w + a.y * b.z - a.z * b.y,
          a.w * b.y + a.y * b.w + a.z * b.x - a.x * b.z,
          a.w * b.z + a.z * b.w + a.x * b.y - a.y * b.x};
}
double qdot(const Quat& a, const Quat& b) { return ((a.x * b.x + a.y * b.y) + a.z * b.z) + a.w * b.w; }
Quat qinverse(const Quat& q) {              // Eigen QuaternionBase::inverse: conjugate().coeffs() / squaredNorm()
  const double n2 = ((q.x * q.x + q.y * q.y) + q.z * q.z) + q.w * q.w;
  if (n2 > 0.0) return {q.w / n2, -q.x / n2, -q.y / n2, -q.z / n2};
  return {0.0, 0.0, 0.0, 0.0};
}
Quat qslerp(const Quat& a, double t, const Quat& o) {   // Eigen 3.3 QuaternionBase::slerp
  const double one = 1.0 - DBL_EPSILON;
  const double d = qdot(a, o);
  const double absD = std::fabs(d);
  double scale0, scale1;
  if (absD >= one) { scale0 = 1.0 - t; scale1 = t; }
  else {
    const double theta = std::acos(absD);
    const double sinTheta = std::sin(theta);
    scale0 = std::sin((1.0 - t) * theta) / sinTheta;
    scale1 = std::sin(t * theta) / sinTheta;
  }
  if (d < 0.0) scale1 = -scale1;
  return {scale0 * a.w + scale1 * o.w, scale0 * a.x + scale1 * o.x, scale0 * a.y + scale1 * o.y, scale0 * a.z + scale1 * o.z};
}
void qrotate(const Quat& q, const double v[3], double out[3]) {   // Eigen QuaternionBase::_transformVector
  double uv[3] = {q.y * v[2] - q.z * v[1], q.z * v[0] - q.x * v[2], q.x * v[1] - q.y * v[0]};
  uv[0] += uv[0]; uv[1] += uv[1]; uv[2] += uv[2];
  const double c[3] = {q.y * uv[2] - q.z * uv[1], q.z * uv[0] - q.x * uv[2], q.x * uv[1] - q.y * uv[0]};
  out[0] = v[0] + q.w * uv[0] + c[0];
  out[1] = v[1] + q.w * uv[1] + c[1];
  out[2] = v[2] + q.w * uv[2] + c[2];
}

struct PointXYZI { float x, y, z, intensity; };

// Preprocessing::undistortion (:176-200)
PointXYZI undistortion(const PointXYZI& pt, const Quat& qIMU, const Quat& q_lb) {
  const double dt = 0.1;
  const int line = int(pt.intensity);
  const double dt_i = pt.intensity - line;
  double ratio_i = dt_i / dt;
  if (ratio_i >= 1.0) ratio_i = 1.0;
  const Quat q0 = {1.0, 0.0, 0.0, 0.0};
  Quat q_si = qslerp(q0, ratio_i, qIMU);
  const double pt_i[3] = {pt.x, pt.y, pt.z};
  q_si = qmul(qmul(q_lb, q_si), qinverse(q_lb));
  double pt_s[3];
  qrotate(q_si, pt_i, pt_s);
  return {(float)pt_s[0], (float)pt_s[1], (float)pt_s[2], pt.intensity};
}

}  // namespace

extern "C" {

/* Preprocessing::cloudHandler, :387-526.  raw: n points at stride_floats (x, y, z at 0..2).  q_imu / q_lb: w,x,y,z, NULL = identity.
 * out_xyzi[4 * n] (room for every input point), scan_start / scan_end[n_scans].  *half_index = the index (into the raw sweep) of
 * the point after which halfPassed is true, -1 if it never is.  Returns 0, or -3 for n_scans not in {16, 32, 64} or a sweep
 * with no point left after the NaN / 3 m filters. */
int go_prepare_scan(const float* raw, int64_t n, int stride, int n_scans, const double* q_imu_wxyz, const double* q_lb_wxyz,
                    float* out_xyzi, int64_t* n_out, int32_t* scan_start, int32_t* scan_end, int64_t* half_index) {
  const int N_SCANS = n_scans;
  if (N_SCANS != 16 && N_SCANS != 32 && N_SCANS != 64) return -3;   // "wrong scan number" (:484-487)
  Quat qIMU = {1.0, 0.0, 0.0, 0.0}, q_lb = {1.0, 0.0, 0.0, 0.0};
  if (q_imu_wxyz) qIMU = {q_imu_wxyz[0], q_imu_wxyz[1], q_imu_wxyz[2], q_imu_wxyz[3]};
  if (q_lb_wxyz) q_lb = {q_lb_wxyz[0], q_lb_wxyz[1], q_lb_wxyz[2], q_lb_wxyz[3]};

  // pcl::removeNaNFromPointCloud + removeClosedPointCloud(.., 3.0) (:396-397, :144-168); the raw index rides along
  std::vector<PointXYZI> cloud; std::vector<int64_t> src;
  const float thres = 3.0f;
  for (int64_t i = 0; i < n; ++i) {
    const float* p = raw + i * stride;
    if (!std::isfinite(p[0]) || !std::isfinite(p[1]) || !std::isfinite(p[2])) continue;
    if (p[0] * p[0] + p[1] * p[1] + p[2] * p[2] < thres * thres) continue;
    cloud.push_back({p[0], p[1], p[2], 0.0f}); src.push_back(i);
  }
  const int cloudSize = (int)cloud.size();
  if (cloudSize == 0) return -3;

  // :401-410
  const float startOri = -go_cr_atan2f(cloud[0].y, cloud[0].x);
  float endOri = -go_cr_atan2f(cloud[cloudSize - 1].y, cloud[cloudSize - 1].x) + 2 * M_PI;
  if (endOri - startOri > 3 * M_PI) endOri -= 2 * M_PI;
  else if (endOri - startOri < M_PI) endOri += 2 * M_PI;

  // :415-417
  if (std::isnan(qIMU.w) || std::isnan(qIMU.x) || std::isnan(qIMU.y) || std::isnan(qIMU.z)) qIMU = {1.0, 0.0, 0.0, 0.0};

  bool halfPassed = false;
  *half_index = -1;
  std::vector<std::vector<PointXYZI>> laserCloudScans(N_SCANS);
  for (int i = 0; i < cloudSize; i++) {                                    // :424-515
    PointXYZI point = cloud[i];
    const float angle = go_cr_atanf(point.z / std::sqrt(point.x * point.x + point.y * point.y)) * 180 / M_PI;
    int scanID = 0;
    if (N_SCANS == 16) {
      scanID = int((angle + 15) / 2 + 0.5);
      if (scanID > (N_SCANS - 1) || scanID < 0) continue;
    } else if (N_SCANS == 32) {
      scanID = int((angle + 92.0 / 3.0) * 3.0 / 4.0);
      if (scanID > (N_SCANS - 1) || scanID < 0) continue;
    } else {
      if (angle >= -8.83) scanID = int((2 - angle) * 3.0 + 0.5);
      else scanID = N_SCANS / 2 + int((-8.83 - angle) * 2.0 + 0.5);
      if (angle > 2 || angle < -24.33 || scanID > 50 || scanID < 0) continue;
    }
    float ori = -go_cr_atan2f(point.y, point.x);
    if (!halfPassed) {
      if (ori < startOri - M_PI / 2) ori += 2 * M_PI;
      else if (ori > startOri + M_PI * 3 / 2) ori -= 2 * M_PI;
      if (ori - startOri > M_PI) { halfPassed = true; *half_index = src[i]; }
    } else {
      ori += 2 * M_PI;
      if (ori < endOri - M_PI * 3 / 2) ori += 2 * M_PI;
      else if (ori > endOri + M_PI / 2) ori -= 2 * M_PI;
    }
    const float relTime = (ori - startOri) / (endOri - startOri);
    point.intensity = scanID + 0.1 * relTime;
    laserCloudScans[scanID].push_back(undistortion(point, qIMU, q_lb));
  }

  // :521-526
  std::vector<PointXYZI> laserCloud;
  for (int i = 0; i < N_SCANS; i++) {
    scan_start[i] = (int)laserCloud.size() + 5;
    laserCloud.insert(laserCloud.end(), laserCloudScans[i].begin(), laserCloudScans[i].end());
    scan_end[i] = (int)laserCloud.size() - 6;
  }
  for (size_t k = 0; k < laserCloud.size(); ++k) {
    out_xyzi[4 * k] = laserCloud[k].x; out_xyzi[4 * k + 1] = laserCloud[k].y;
    out_xyzi[4 * k + 2] = laserCloud[k].z; out_xyzi[4 * k + 3] = laserCloud[k].intensity;
  }
  *n_out = (int64_t)laserCloud.size();
  return 0;
}

/* Preprocessing::processIMU (:222-259) with solveRotation (:202-207) and deltaQ (GLIO/include/utils/math_tools.h:126-138) for one
 * sweep: qIMU from identity (:37, :675), the buffer stamps[n] / gyro[3n] as imu_buf, state = {idx_imu, current_time_imu,
 * gyr_0[3], first_imu}.  first_imu == 0 and n > 0: imuHandler's first-sample initialisation (:281-293).  q = w,x,y,z. */
typedef struct { int64_t idx_imu; double current_time_imu; double gyr_0[3]; int32_t first_imu; int32_t reserved; } go_imu_state;

void go_imu_sweep_rotation(go_imu_state* s, const double* stamps, const double* gyro, int64_t n, double t_cur, double q_out[4]) {
  Quat qIMU = {1.0, 0.0, 0.0, 0.0};
  if (!s->first_imu && n > 0) {
    s->current_time_imu = stamps[0];
    s->gyr_0[0] = gyro[0]; s->gyr_0[1] = gyro[1]; s->gyr_0[2] = gyro[2];
    s->first_imu = 1;
  }
  auto solveRotation = [&](double dt, const double w[3]) {
    double un_gyr[3], half[3];
    for (int d = 0; d < 3; ++d) un_gyr[d] = 0.5 * (s->gyr_0[d] + w[d]);
    for (int d = 0; d < 3; ++d) { half[d] = un_gyr[d] * dt; half[d] /= 2.0; }
    qIMU = qmul(qIMU, Quat{1.0, half[0], half[1], half[2]});
    for (int d = 0; d < 3; ++d) s->gyr_0[d] = w[d];
  };
  if (s->first_imu) {                                                       // if (first_imu) processIMU(time_scan_next)  (:413-414)
    double rx = 0, ry = 0, rz = 0;
    int64_t i = s->idx_imu;
    if (i >= n) i--;
    while (stamps[i] < t_cur) {
      double t = stamps[i];
      if (s->current_time_imu < 0) s->current_time_imu = t;
      double dt = t - s->current_time_imu;
      s->current_time_imu = stamps[i];
      rx = gyro[3 * i]; ry = gyro[3 * i + 1]; rz = gyro[3 * i + 2];
      const double w[3] = {rx, ry, rz};
      solveRotation(dt, w);
      i++;
      if (i >= n) break;
    }
    if (i < n) {
      double dt1 = t_cur - s->current_time_imu;
      double dt2 = stamps[i] - t_cur;
      double w1 = dt2 / (dt1 + dt2);
      double w2 = dt1 / (dt1 + dt2);
      rx = w1 * rx + w2 * gyro[3 * i];
      ry = w1 * ry + w2 * gyro[3 * i + 1];
      rz = w1 * rz + w2 * gyro[3 * i + 2];
      const double w[3] = {rx, ry, rz};
      solveRotation(dt1, w);
    }
    s->current_time_imu = t_cur;
    s->idx_imu = i;
  }
  if (std::isnan(qIMU.w) || std::isnan(qIMU.x) || std::isnan(qIMU.y) || std::isnan(qIMU.z)) qIMU = {1.0, 0.0, 0.0, 0.0};
  q_out[0] = qIMU.w; q_out[1] = qIMU.x; q_out[2] = qIMU.y; q_out[3] = qIMU.z;
}

}  // extern "C"
