// scanprep.cu — the front end's sweep preparation on the device (SURVEY 8 f-5): Preprocessing::cloudHandler,
// GLIO/src/Preprocessing.cpp:387-526.  Input = a raw sweep as received (pcl::PointXYZI: x, y, z at floats 0..2 of a caller
// stride); output = `laserCloud`: the kept points ring after ring as packed float4 (x, y, z, intensity = ring + 0.1 relTime),
// de-skewed by the sweep's IMU rotation, with scanStartInd / scanEndInd per ring.
//   k_sp_bounds    first and last point that survives removeNaNFromPointCloud + removeClosedPointCloud(3 m) (:144-168, :396-397)
//   k_sp_consts    one thread: startOri / endOri from those two points and the endOri correction (:401-410)
//   k_sp_classify  one thread per raw point: ring id (:438-483), raw azimuth, the first-half wrap and its "passed half" test
//                  (:489-498); the first kept index that passes is reduced with atomicMin: the sequential halfPassed flag
//                  flips right after that point.  Per-block ring histogram for the stable partition.
//   k_scan_*       exclusive scan of the histogram in ring-major order (grid.cu)
//   k_sp_ranges    scanStartInd = size_before + 5, scanEndInd = size_after - 6 per ring (:521-526), and the kept count
//   k_sp_emit      one thread per raw point: the azimuth branch chosen by the point's index relative to the halfPassed index,
//                  relTime, intensity, undistortion (:176-200), and the stable scatter (in-block rank by warp match per ring)
// Every rounding follows the reference's types and order with _rn intrinsics; compiled with -fmad=false.  atanf / atan2f are
// correctly rounded: the double result is rounded to float, and inside a guard band around a float rounding boundary the
// side of the boundary is decided in double-double (DESIGN 2).
#include "common.cuh"
#include "devmath.cuh"

namespace glio {

constexpr int SP_T = 256;
constexpr double kPi = 3.14159265358979323846;      // M_PI
constexpr double kTwoPi = 2 * kPi;                  // 2 * M_PI
constexpr double kHalfPi = kPi / 2;                 // M_PI / 2
constexpr double kThreeHalfPi = kPi * 3 / 2;        // M_PI * 3 / 2
constexpr int SP_NONE = 0x7f7f7f7f;                 // "no index" (memset pattern 0x7f; n < 2^30)

// ---------------------------------------------------------------------------------------------------------------------
// double-double arithmetic (Dekker / Knuth error-free transformations) for the guard-band decision
// ---------------------------------------------------------------------------------------------------------------------
struct DD { double hi, lo; };
__device__ __forceinline__ DD two_sum(double a, double b) {
  const double s = __dadd_rn(a, b), bb = __dsub_rn(s, a);
  return {s, __dadd_rn(__dsub_rn(a, __dsub_rn(s, bb)), __dsub_rn(b, bb))};
}
__device__ __forceinline__ DD quick_two_sum(double a, double b) { const double s = __dadd_rn(a, b); return {s, __dsub_rn(b, __dsub_rn(s, a))}; }
__device__ __forceinline__ DD two_prod(double a, double b) { const double p = __dmul_rn(a, b); return {p, __fma_rn(a, b, -p)}; }
__device__ __forceinline__ DD dd_add(DD a, DD b) {
  DD s = two_sum(a.hi, b.hi); const DD t = two_sum(a.lo, b.lo);
  s.lo = __dadd_rn(s.lo, t.hi); s = quick_two_sum(s.hi, s.lo);
  s.lo = __dadd_rn(s.lo, t.lo); return quick_two_sum(s.hi, s.lo);
}
__device__ __forceinline__ DD dd_mul(DD a, DD b) {
  DD p = two_prod(a.hi, b.hi);
  p.lo = __dadd_rn(p.lo, __dadd_rn(__dmul_rn(a.hi, b.lo), __dmul_rn(a.lo, b.hi)));
  return quick_two_sum(p.hi, p.lo);
}
__device__ __forceinline__ DD dd_mul_d(DD a, double b) { DD p = two_prod(a.hi, b); p.lo = __dadd_rn(p.lo, __dmul_rn(a.lo, b)); return quick_two_sum(p.hi, p.lo); }
__device__ __forceinline__ DD dd_div_d(DD a, double b) {
  const double q1 = __ddiv_rn(a.hi, b);
  const DD p = two_prod(q1, b);
  const double r = __dadd_rn(__dsub_rn(__dsub_rn(a.hi, p.hi), p.lo), a.lo);
  return quick_two_sum(q1, __ddiv_rn(r, b));
}

// sin m, cos m in double-double for |m| <= pi.  m - k pi/2 with a three-part pi/2: k in [-2, 2], so k*P1 is exact and so is
// m - k*P1 (Sterbenz); then Taylor series on |r| <= pi/4 to 2^-105.
__device__ void dd_sincos(double m, DD& s, DD& c) {
  const double P1 = 1.5707963267948966, P2 = 6.123233995736766e-17, P3 = -1.4973849048591698e-33;
  const double k = rint(__dmul_rn(m, 0.63661977236758138));
  DD r = two_sum(__dsub_rn(m, __dmul_rn(k, P1)), -__dmul_rn(k, P2));
  r.lo = __dsub_rn(r.lo, __dmul_rn(k, P3)); r = quick_two_sum(r.hi, r.lo);
  const DD r2 = dd_mul(r, r);
  DD ts = r, tc = {1.0, 0.0}, ss = r, cc = {1.0, 0.0};
  for (int j = 1; j <= 15; ++j) {
    ts = dd_div_d(dd_mul(ts, r2), -(double)((2 * j) * (2 * j + 1)));
    tc = dd_div_d(dd_mul(tc, r2), -(double)((2 * j - 1) * (2 * j)));
    ss = dd_add(ss, ts); cc = dd_add(cc, tc);
  }
  const DD nss = {-ss.hi, -ss.lo}, ncc = {-cc.hi, -cc.lo};
  switch (((int)k) & 3) {
    case 0: s = ss; c = cc; break;
    case 1: s = cc; c = nss; break;
    case 2: s = nss; c = ncc; break;
    default: s = ncc; c = ss; break;
  }
}

// true when atan2(y, x) > m (|atan2(y, x) - m| < pi):  r sin(theta - m) = y cos m - x sin m
__device__ __noinline__ bool angle_above(double y, double x, double m) {
  DD s, c;
  dd_sincos(m, s, c);
  const DD t = dd_add(dd_mul_d(c, y), dd_mul_d(s, -x));
  return t.hi > 0.0 || (t.hi == 0.0 && t.lo > 0.0);
}

// float nearest to the angle atan2(y, x) whose double evaluation is d (error <= 2 double ulp, CUDA math documentation)
__device__ __forceinline__ float cr_angle(double d, double y, double x, unsigned long long* hits) {
  const float lo = __double2float_rd(d), hi = __double2float_ru(d);
  if (lo == hi) return lo;
  const double m = __dmul_rn(__dadd_rn((double)lo, (double)hi), 0.5);     // the rounding boundary between lo and hi
  if (fabs(__dsub_rn(d, m)) > __dmul_rn(fabs(m), 0x1p-40)) return __double2float_rn(d);
  atomicAdd(hits, 1ull);
  return angle_above(y, x, m) ? hi : lo;
}
__device__ __forceinline__ float cr_atan2f(float y, float x, unsigned long long* hits) {
  return cr_angle(atan2((double)y, (double)x), (double)y, (double)x, hits);
}
__device__ __forceinline__ float cr_atanf(float a, unsigned long long* hits) {
  if (isinf(a)) return __double2float_rn(atan((double)a));                 // +-pi/2: far from any rounding boundary
  return cr_angle(atan((double)a), (double)a, 1.0, hits);
}

__device__ __forceinline__ bool sp_load(const ScanPrepArgs& a, int64_t i, float& x, float& y, float& z) {
  const float* p = a.raw + i * a.stride;
  x = p[0]; y = p[1]; z = p[2];
  if (!(isfinite(x) && isfinite(y) && isfinite(z))) return false;          // removeNaNFromPointCloud
  return !(fadd(fadd(fmul(x, x), fmul(y, y)), fmul(z, z)) < 9.0f);          // removeClosedPointCloud(.., 3.0): < thres * thres
}

// ring id of Preprocessing.cpp:438-483, -1 when the point is skipped
__device__ __forceinline__ int sp_ring(float x, float y, float z, int n_scans, unsigned long long* hits) {
  const float a0 = fmul(cr_atanf(__fdiv_rn(z, __fsqrt_rn(fadd(fmul(x, x), fmul(y, y)))), hits), 180.0f);
  const float angle = __double2float_rn(__ddiv_rn((double)a0, kPi));
  int id;
  if (n_scans == 16) {
    id = (int)__dadd_rn((double)__fdiv_rn(fadd(angle, 15.0f), 2.0f), 0.5);
    return (id > 15 || id < 0) ? -1 : id;
  }
  if (n_scans == 32) {
    id = (int)__ddiv_rn(__dmul_rn(__dadd_rn((double)angle, 92.0 / 3.0), 3.0), 4.0);
    return (id > 31 || id < 0) ? -1 : id;
  }
  if ((double)angle >= -8.83) id = (int)__dadd_rn(__dmul_rn((double)fsub(2.0f, angle), 3.0), 0.5);
  else id = 32 + (int)__dadd_rn(__dmul_rn(__dsub_rn(-8.83, (double)angle), 2.0), 0.5);
  return (angle > 2.0f || (double)angle < -24.33 || id > 50 || id < 0) ? -1 : id;
}

__device__ __forceinline__ float f_add_d(float f, double d) { return __double2float_rn(__dadd_rn((double)f, d)); }

// the first-half wrap of :490-495
__device__ __forceinline__ float sp_wrap_first(float ori, const SweepConsts& k) {
  if ((double)ori < k.c_first_lo) return f_add_d(ori, kTwoPi);
  if ((double)ori > k.c_first_hi) return f_add_d(ori, -kTwoPi);
  return ori;
}

__global__ void __launch_bounds__(SP_T) k_sp_bounds(ScanPrepArgs a) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  float x, y, z;
  const bool ok = i < a.n && sp_load(a, i, x, y, z);
  const int lo = __reduce_min_sync(0xffffffffu, ok ? (int)i : SP_NONE);
  const int hi = __reduce_max_sync(0xffffffffu, ok ? (int)i : -1);
  if ((threadIdx.x & 31) == 0) {
    if (lo != SP_NONE) atomicMin(a.small + 0, lo);
    if (hi >= 0) atomicMax(a.small + 1, hi);
  }
}

__global__ void k_sp_consts(ScanPrepArgs a) {
  SweepConsts k{};
  const int f = a.small[0], l = a.small[1];
  k.ok = f != SP_NONE;
  if (k.ok) {
    const float* p0 = a.raw + (int64_t)f * a.stride;
    const float* pn = a.raw + (int64_t)l * a.stride;
    k.start_ori = -cr_atan2f(p0[1], p0[0], a.guard_hits);
    float e = f_add_d(-cr_atan2f(pn[1], pn[0], a.guard_hits), kTwoPi);
    if ((double)fsub(e, k.start_ori) > 3 * kPi) e = f_add_d(e, -kTwoPi);
    else if ((double)fsub(e, k.start_ori) < kPi) e = f_add_d(e, kTwoPi);
    k.end_ori = e;
    k.c_first_lo = __dsub_rn((double)k.start_ori, kHalfPi); k.c_first_hi = __dadd_rn((double)k.start_ori, kThreeHalfPi);
    k.c_second_lo = __dsub_rn((double)k.end_ori, kThreeHalfPi); k.c_second_hi = __dadd_rn((double)k.end_ori, kHalfPi);
  }
  *a.consts = k;
}

__global__ void __launch_bounds__(SP_T) k_sp_classify(ScanPrepArgs a) {
  __shared__ int s_hist[64];
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const SweepConsts k = *a.consts;
  for (int r = threadIdx.x; r < 64; r += blockDim.x) s_hist[r] = 0;
  __syncthreads();
  int ring = -1;
  bool pre = false;
  if (k.ok && i < a.n) {
    float x, y, z;
    if (sp_load(a, i, x, y, z)) ring = sp_ring(x, y, z, a.n_scans, a.guard_hits);
    if (ring >= 0) {
      const float ori = -cr_atan2f(y, x, a.guard_hits);
      a.ori[i] = ori;
      pre = (double)fsub(sp_wrap_first(ori, k), k.start_ori) > kPi;
      atomicAdd(&s_hist[ring], 1);
    }
    a.ring[i] = (int8_t)ring;
  }
  const int h = __reduce_min_sync(0xffffffffu, pre ? (int)i : SP_NONE);
  if ((threadIdx.x & 31) == 0 && h != SP_NONE) atomicMin(a.small + 2, h);
  __syncthreads();
  for (int r = threadIdx.x; r < a.n_scans; r += blockDim.x) a.hist[(int64_t)r * a.nb + blockIdx.x] = s_hist[r];
}

// small[3] = ok, small[4] = kept count, small[5 + r] = scanStartInd[r], small[5 + S + r] = scanEndInd[r]
__global__ void k_sp_ranges(ScanPrepArgs a) {
  const int S = a.n_scans;
  const int64_t last = (int64_t)S * a.nb - 1;
  const int total = a.consts->ok ? a.hscan[last] + a.hist[last] : 0;
  for (int r = threadIdx.x; r < S; r += blockDim.x) {
    const int before = a.consts->ok ? a.hscan[(int64_t)r * a.nb] : 0;
    const int after = r + 1 < S ? (a.consts->ok ? a.hscan[(int64_t)(r + 1) * a.nb] : 0) : total;
    a.small[5 + r] = before + 5; a.small[5 + S + r] = after - 6;
  }
  if (threadIdx.x == 0) { a.small[3] = a.consts->ok; a.small[4] = total; }
}

// Eigen's generic quat_product (Quaternion.h): (w, x, y, z) of a * b, left to right
__device__ __forceinline__ void qmul_rn(const double a[4], const double b[4], double o[4]) {
  const double w = dsub(dsub(dsub(dmul(a[0], b[0]), dmul(a[1], b[1])), dmul(a[2], b[2])), dmul(a[3], b[3]));
  const double x = dsub(dadd(dadd(dmul(a[0], b[1]), dmul(a[1], b[0])), dmul(a[2], b[3])), dmul(a[3], b[2]));
  const double y = dsub(dadd(dadd(dmul(a[0], b[2]), dmul(a[2], b[0])), dmul(a[3], b[1])), dmul(a[1], b[3]));
  const double z = dsub(dadd(dadd(dmul(a[0], b[3]), dmul(a[3], b[0])), dmul(a[1], b[2])), dmul(a[2], b[1]));
  o[0] = w; o[1] = x; o[2] = y; o[3] = z;
}

__global__ void __launch_bounds__(SP_T) k_sp_emit(ScanPrepArgs a) {
  __shared__ int s_wcnt[SP_T / 32][64];
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const SweepConsts k = *a.consts;
  for (int t = threadIdx.x; t < (SP_T / 32) * 64; t += blockDim.x) (&s_wcnt[0][0])[t] = 0;
  const int ring = (k.ok && i < a.n) ? (int)a.ring[i] : -1;
  const unsigned peers = __match_any_sync(0xffffffffu, ring);
  __syncthreads();
  if (ring >= 0 && lane == __ffs(peers) - 1) s_wcnt[wid][ring] = __popc(peers);
  __syncthreads();
  if (ring < 0) return;
  int pos = a.hscan[(int64_t)ring * a.nb + blockIdx.x] + __popc(peers & ((1u << lane) - 1u));
  for (int w = 0; w < wid; ++w) pos += s_wcnt[w][ring];

  // azimuth: the branch of the sequential halfPassed state machine (:490-505)
  float ori = a.ori[i];
  if (i <= (int64_t)a.small[2]) {
    ori = sp_wrap_first(ori, k);
  } else {
    ori = f_add_d(ori, kTwoPi);
    if ((double)ori < k.c_second_lo) ori = f_add_d(ori, kTwoPi);
    else if ((double)ori > k.c_second_hi) ori = f_add_d(ori, -kTwoPi);
  }
  const float rel = __fdiv_rn(fsub(ori, k.start_ori), fsub(k.end_ori, k.start_ori));                 // :507
  const float inten = __double2float_rn(dadd((double)ring, dmul(0.1, (double)rel)));                // :509

  // undistortion (:176-200)
  const int line = (int)inten;
  const double dt_i = (double)fsub(inten, (float)line);
  double t = __ddiv_rn(dt_i, 0.1);
  if (t >= 1.0) t = 1.0;
  double s0, s1;
  if (a.slerp_linear) { s0 = dsub(1.0, t); s1 = t; }                                                  // Eigen slerp, |d| >= 1 - eps
  else { s0 = __ddiv_rn(sin(dmul(dsub(1.0, t), a.theta)), a.sin_theta); s1 = __ddiv_rn(sin(dmul(t, a.theta)), a.sin_theta); }
  if (a.dot < 0.0) s1 = -s1;
  // scale0 * Identity.coeffs() + scale1 * qIMU.coeffs(), coefficient by coefficient
  const double qsi[4] = {dadd(dmul(s0, 1.0), dmul(s1, a.q_imu[0])), dadd(dmul(s0, 0.0), dmul(s1, a.q_imu[1])),
                         dadd(dmul(s0, 0.0), dmul(s1, a.q_imu[2])), dadd(dmul(s0, 0.0), dmul(s1, a.q_imu[3]))};
  double q1[4], q2[4];
  qmul_rn(a.q_lb, qsi, q1);
  qmul_rn(q1, a.q_lb_inv, q2);
  const float* p = a.raw + i * a.stride;
  const double v[3] = {(double)p[0], (double)p[1], (double)p[2]};
  double o[3];
  qrot_rn(q2, v, o);
  if (pos < a.out_capacity) a.out[pos] = make_float4(__double2float_rn(o[0]), __double2float_rn(o[1]), __double2float_rn(o[2]), inten);
}

void scanprep_run(ScanPrepArgs& a, cudaStream_t st, LaunchCounter& lc) {
  const unsigned nb = (unsigned)a.nb;
  GLIO_CUDA_TRY(cudaMemsetAsync(a.small, 0x7f, 3 * sizeof(int), st));               // first, half = none
  GLIO_CUDA_TRY(cudaMemsetAsync(a.small + 1, 0xff, sizeof(int), st));               // last = -1
  lc.begin("k_sp_bounds", st); k_sp_bounds<<<nb, SP_T, 0, st>>>(a); lc.end(st);
  lc.begin("k_sp_consts", st); k_sp_consts<<<1, 1, 0, st>>>(a); lc.end(st);
  lc.begin("k_sp_classify", st); k_sp_classify<<<nb, SP_T, 0, st>>>(a); lc.end(st);
  exclusive_scan_i32(a.hist, a.hscan, (int64_t)a.n_scans * a.nb, *a.scan_tmp, st, lc);
  lc.begin("k_sp_ranges", st); k_sp_ranges<<<1, 64, 0, st>>>(a); lc.end(st);
  lc.begin("k_sp_emit", st); k_sp_emit<<<nb, SP_T, 0, st>>>(a); lc.end(st);
  GLIO_CUDA_TRY(cudaGetLastError());
}

// ---------------------------------------------------------------------------------------------------------------------
// host: per-sweep IMU rotation, Preprocessing::processIMU / solveRotation (:202-207, :222-259) with deltaQ
// (GLIO/include/utils/math_tools.h:126-138); qIMU starts from identity every sweep (:37, :675)
// ---------------------------------------------------------------------------------------------------------------------
static void host_qmul(const double a[4], const double b[4], double o[4]) {
  const double w = a[0] * b[0] - a[1] * b[1] - a[2] * b[2] - a[3] * b[3];
  const double x = a[0] * b[1] + a[1] * b[0] + a[2] * b[3] - a[3] * b[2];
  const double y = a[0] * b[2] + a[2] * b[0] + a[3] * b[1] - a[1] * b[3];
  const double z = a[0] * b[3] + a[3] * b[0] + a[1] * b[2] - a[2] * b[1];
  o[0] = w; o[1] = x; o[2] = y; o[3] = z;
}

static void solve_rotation(glio_imu_state* st, double q[4], double dt, const double w[3]) {
  double th[3];
  for (int d = 0; d < 3; ++d) th[d] = 0.5 * (st->gyr_0[d] + w[d]) * dt;
  const double dq[4] = {1.0, th[0] / 2.0, th[1] / 2.0, th[2] / 2.0};
  double o[4];
  host_qmul(q, dq, o);
  for (int d = 0; d < 4; ++d) q[d] = o[d];
  for (int d = 0; d < 3; ++d) st->gyr_0[d] = w[d];
}

void imu_sweep_rotation(glio_imu_state* st, const double* stamps, const double* gyro, int64_t n, double t_cur, double q[4]) {
  q[0] = 1.0; q[1] = q[2] = q[3] = 0.0;
  if (!st->first_imu) {
    if (n <= 0) return;                      // no IMU sample yet: processIMU is not called (:413)
    st->current_time_imu = stamps[0];        // imuHandler's first sample (:281-293)
    for (int d = 0; d < 3; ++d) st->gyr_0[d] = gyro[d];
    st->first_imu = 1;
  }
  double rx = 0, ry = 0, rz = 0;
  int64_t i = st->idx_imu;
  if (i >= n) i--;
  while (stamps[i] < t_cur) {
    const double t = stamps[i];
    if (st->current_time_imu < 0) st->current_time_imu = t;
    const double dt = t - st->current_time_imu;
    st->current_time_imu = stamps[i];
    rx = gyro[3 * i]; ry = gyro[3 * i + 1]; rz = gyro[3 * i + 2];
    const double w[3] = {rx, ry, rz};
    solve_rotation(st, q, dt, w);
    i++;
    if (i >= n) break;
  }
  if (i < n) {
    const double dt1 = t_cur - st->current_time_imu;
    const double dt2 = stamps[i] - t_cur;
    const double w1 = dt2 / (dt1 + dt2);
    const double w2 = dt1 / (dt1 + dt2);
    rx = w1 * rx + w2 * gyro[3 * i];
    ry = w1 * ry + w2 * gyro[3 * i + 1];
    rz = w1 * rz + w2 * gyro[3 * i + 2];
    const double w[3] = {rx, ry, rz};
    solve_rotation(st, q, dt1, w);
  }
  st->current_time_imu = t_cur;
  st->idx_imu = i;
  if (std::isnan(q[0]) || std::isnan(q[1]) || std::isnan(q[2]) || std::isnan(q[3])) { q[0] = 1.0; q[1] = q[2] = q[3] = 0.0; }   // :415-417
}

}  // namespace glio
