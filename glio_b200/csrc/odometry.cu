// odometry.cu — the arithmetic of the front end's LidarOdometry node (GLIO/src/LidarOdometry.cpp) that is not scan matching:
// the pose bookkeeping of run() on the host and the de-skew of the published clouds on the device.  Built with -fmad=false;
// the host functions are scalar double code in Eigen's operation order (baseline x86-64: no FMA contraction either), so a
// scalar restatement in another language reproduces them bit for bit.
#include "common.cuh"
#include "devmath.cuh"
#include "hostmath.h"

namespace glio {

// ---- host: poses in the reference's layout, q(w,x,y,z) then t(x,y,z)

// Eigen Quaternion::inverse(): conjugate / squaredNorm() (coeffs() order x, y, z, w), zero for a zero quaternion
void odom_quat_inverse(const double q[4], double o[4]) {
  const double n2 = ((q[1] * q[1] + q[2] * q[2]) + q[3] * q[3]) + q[0] * q[0];
  if (n2 > 0.0) { o[0] = q[0] / n2; o[1] = -q[1] / n2; o[2] = -q[2] / n2; o[3] = -q[3] / n2; }
  else { o[0] = 0.0; o[1] = 0.0; o[2] = 0.0; o[3] = 0.0; }
}

// poseInitialization (:406-433): t0 = q0*dt + t0, then q0 = q0*dq
void odom_predict(double a[7], const double r[7]) {
  double v[3]; h_qrot(a, r + 4, v);
  const double t0 = v[0] + a[4], t1 = v[1] + a[5], t2 = v[2] + a[6];
  double q[4]; h_qmul(a, r, q);
  a[0] = q[0]; a[1] = q[1]; a[2] = q[2]; a[3] = q[3];
  a[4] = t0; a[5] = t1; a[6] = t2;
}

// computeRelative (:435-471): q_r = q1^-1 * q2, t_r = q1^-1 * (t2 - t1)
void odom_relative(const double p1[7], const double p2[7], double r[7]) {
  double qi[4]; odom_quat_inverse(p1, qi);
  double q[4]; h_qmul(qi, p2, q);
  const double d[3] = {p2[4] - p1[4], p2[5] - p1[5], p2[6] - p1[6]};
  double t[3]; h_qrot(qi, d, t);
  r[0] = q[0]; r[1] = q[1]; r[2] = q[2]; r[3] = q[3];
  r[4] = t[0]; r[5] = t[1]; r[6] = t[2];
}

// :566-578, with C++'s precedence: ((dis > 0.2 || ang > 0.1) && size - kf_num > 1 || size - kf_num > 2) || size <= 1.
// ang = 2*acos(w) of quat_last_kF.inverse()*quatCur: a w above 1 from rounding gives NaN, and NaN > 0.1 is false.
bool odom_keyframe_rule(const double t_cur[3], const double q_cur[4], const double t_kf[3], const double q_kf[4], int64_t size, int64_t kf_num) {
  const double d0 = t_cur[0] - t_kf[0], d1 = t_cur[1] - t_kf[1], d2 = t_cur[2] - t_kf[2];
  const double dis = std::sqrt((d0 * d0 + d1 * d1) + d2 * d2);
  double qi[4]; odom_quat_inverse(q_kf, qi);
  double q[4]; h_qmul(qi, q_cur, q);
  const double ang = 2 * std::acos(q[0]);
  return (((dis > 0.2 || ang > 0.1) && size - kf_num > 1) || size - kf_num > 2) || size <= 1;
}

// ---- device: undistortion (:176-200) with the identity quaternion publishCloudLast passes (:621).  Identity.slerp(r, Identity) has
// a zero vector part, and Eigen's _transformVector then returns the point itself, so the de-skew is float(double(p) + r*trans) with
// r = min(double(float(i - int(i))) / 0.1, 1).  deskew = 0: plain copy.  Intensity is kept.
__global__ void __launch_bounds__(256) k_odom_publish(const float4* __restrict__ surf, int64_t n_surf, const float4* __restrict__ full,
                                                     int64_t n_full, float4* __restrict__ surf_out, float4* __restrict__ full_out,
                                                     double tx, double ty, double tz, int deskew) {
  const int64_t n = n_surf + n_full;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const bool is_surf = i < n_surf;
    const int64_t k = is_surf ? i : i - n_surf;
    float4* out = is_surf ? surf_out : full_out;
    if (!out) continue;
    float4 p = is_surf ? surf[k] : full[k];
    if (deskew) {
      const int line = (int)p.w;
      const float dt_f = __fsub_rn(p.w, (float)line);          // pt.intensity - line: float arithmetic
      double ratio = __ddiv_rn((double)dt_f, 0.1);
      if (ratio > 1) ratio = 1;
      p.x = (float)dadd((double)p.x, dmul(ratio, tx));
      p.y = (float)dadd((double)p.y, dmul(ratio, ty));
      p.z = (float)dadd((double)p.z, dmul(ratio, tz));
    }
    out[k] = p;
  }
}

void odom_publish_run(const float4* surf, int64_t n_surf, const float4* full, int64_t n_full, float4* surf_out, float4* full_out,
                      const double trans[3], int deskew, cudaStream_t st, LaunchCounter& lc) {
  if (!surf_out) n_surf = 0;
  if (!full_out) n_full = 0;
  const int64_t n = n_surf + n_full;
  if (n <= 0) return;
  // full is indexed from n_surf on: with no surf output the whole range is full's
  const int nb = (int)std::min<int64_t>((n + 255) / 256, kNumSMs * 8);
  lc.begin("k_odom_publish", st);
  k_odom_publish<<<nb, 256, 0, st>>>(surf, n_surf, full, n_full, surf_out, full_out, trans[0], trans[1], trans[2], deskew);
  lc.end(st);
  GLIO_CUDA_TRY(cudaGetLastError());
}

}  // namespace glio
