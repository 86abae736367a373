// eval.cu — K2 / K2b / K2e: residual + Jacobian + Huber + block J^T J / J^T r reduction.
//
// Replaces, for the LiDAR factors, ceres::ResidualBlock::Evaluate (ceres.tgz::internal/ceres/residual_block.cc:70-197:
// autodiff cost -> local parameterization -> Corrector) over LidarPlaneNormFactor / BinaryLidarPlaneNormFactor /
// LidarEdgeFactor (GLIO/include/factors/LidarKeyframeFactor.h:12-164) and the normal-equation accumulation that
// follows it (sparse J^T J in the solve, dense A/b in MarginalizationFactor.cpp:3-29).
//
// HBM traffic per unary residual: 2 x 16 B loads (cp+weight, weight*n + weight*d) = 32 B; outputs are W x 28 doubles.
// Arithmetic is fp64 (tolerance 1e-8 rad per iteration), inputs fp32 as the reference stores them (quirk Q5).
// Reduction: per-thread register accumulators over a run of one keyframe's (or pair's) residuals -> warp shuffle -> shared ->
// one partial per work item (block_partials); for the unary kernels the last block to finish sums the partials per keyframe in
// a fixed order (kf_sums; deterministic, no floating-point atomics).  The frame set-ups (kf_frame, pair_frame), the plane
// residual (plane_residual) and the binary 55-sum layout (pair_accumulate) are shared by the kernels below.
#include "common.cuh"

namespace glio {

// closed-form rotation matrix of Eigen's Quaternion * v for a (not necessarily unit) quaternion, as the
// polynomial the functor evaluates:  R v = v + 2w(u x v) + 2 u x (u x v)
__device__ __forceinline__ void quat_to_mat(const double q[4], double R[9]) {
  const double w = q[0], x = q[1], y = q[2], z = q[3];
  R[0] = 1.0 - 2.0 * (y * y + z * z); R[1] = 2.0 * (x * y - w * z);       R[2] = 2.0 * (x * z + w * y);
  R[3] = 2.0 * (x * y + w * z);       R[4] = 1.0 - 2.0 * (x * x + z * z); R[5] = 2.0 * (y * z - w * x);
  R[6] = 2.0 * (x * z - w * y);       R[7] = 2.0 * (y * z + w * x);       R[8] = 1.0 - 2.0 * (x * x + y * y);
}
__device__ __forceinline__ void mat_mul3(const double A[9], const double B[9], double C[9]) {
#pragma unroll
  for (int i = 0; i < 3; ++i)
#pragma unroll
    for (int j = 0; j < 3; ++j) C[3 * i + j] = A[3 * i] * B[j] + A[3 * i + 1] * B[3 + j] + A[3 * i + 2] * B[6 + j];
}
__device__ __forceinline__ void mat_vec3(const double A[9], double x, double y, double z, double o[3]) {
  o[0] = A[0] * x + A[1] * y + A[2] * z;
  o[1] = A[3] * x + A[4] * y + A[5] * z;
  o[2] = A[6] * x + A[7] * y + A[8] * z;
}

// Huber + Corrector for a scalar residual (loss_function.cc:48-62, corrector.cc:41-155; rho'' <= 0 always, so the
// simple branch: r <- sqrt(rho') r, J <- sqrt(rho') J).  Returns the block cost 0.5 * rho(s).
__device__ __forceinline__ double huber_scale(double r, double delta, double& scale) {
  const double s = r * r;
  if (delta > 0.0 && s > delta * delta) {
    const double a = sqrt(s);
    double rho1 = delta / a;
    rho1 = rho1 < 2.2250738585072014e-308 ? 2.2250738585072014e-308 : rho1;
    scale = sqrt(rho1);
    return 0.5 * (2.0 * delta * a - delta * delta);
  }
  scale = 1.0;
  return 0.5 * s;
}

constexpr int EV_T = 256;
constexpr int NACC = GLIO_NACC;   // 21 upper-triangular H + 6 g + 1 cost

struct KfFrame {           // per keyframe, prepared in shared memory
  double M[9];             // R(q) * R(q_lb)^-1   (maps cp - t_lb to the rotated body point a)
  double Rlbi[9];          // R(q_lb)^-1
  double t[3];
  double q[4];
};

// F from the pose P = (t, q) of one keyframe.  STORE_Q: also keep q (the ambient quaternion columns read it); the cost-only and
// tangent K2e kernels leave it out, which keeps k_eval_edge<false, 0> at 60 registers.
template <bool STORE_Q>
__device__ __forceinline__ void kf_frame(const double* P, const EvalParams& ep, KfFrame& F) {
  double qn[4] = {P[3], P[4], P[5], P[6]};
  double R[9]; quat_to_mat(qn, R);
  // q_lb^-1 = conj / |q|^2 (Eigen inverse()); rotation by it as the polynomial in its coefficients
  const double n2 = ep.q_lb[0] * ep.q_lb[0] + ep.q_lb[1] * ep.q_lb[1] + ep.q_lb[2] * ep.q_lb[2] + ep.q_lb[3] * ep.q_lb[3];
  double qi[4] = {ep.q_lb[0] / n2, -ep.q_lb[1] / n2, -ep.q_lb[2] / n2, -ep.q_lb[3] / n2};
  quat_to_mat(qi, F.Rlbi);
  mat_mul3(R, F.Rlbi, F.M);
  F.t[0] = P[0]; F.t[1] = P[1]; F.t[2] = P[2];
  if (STORE_Q) { F.q[0] = qn[0]; F.q[1] = qn[1]; F.q[2] = qn[2]; F.q[3] = qn[3]; }
}

// Reduces the NS per-thread sums of an NT-thread block (shuffle -> shared red -> one partial per block at
// partials[blockIdx.x * NS]).  The last sum is the cost; without WANT_JAC it is the only one reduced, the others are written as 0.
template <int NS, int NT, bool WANT_JAC>
__device__ __forceinline__ void block_partials(const double (&acc)[NS], double (&red)[NT / 32][NS], double* __restrict__ partials) {
  constexpr int COST = NS - 1;
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
#pragma unroll
  for (int k = WANT_JAC ? 0 : COST; k < NS; ++k) {
    double v = acc[k];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if (lane == 0) red[wid][k] = v;
  }
  __syncthreads();
  if (threadIdx.x < NS) {
    double v = 0.0;
    if (WANT_JAC || threadIdx.x == COST) {
#pragma unroll
      for (int w = 0; w < NT / 32; ++w) v += red[w][threadIdx.x];
    }
    partials[(size_t)blockIdx.x * NS + threadIdx.x] = v;
  }
}

// After block_partials: the block that takes the last ticket sums the partials per keyframe into out (W x NACC), in item order,
// then runs last_block() (every thread), which resets the ticket for the next launch.  is_last: the kernel's shared flag.
template <class LastBlock>
__device__ __forceinline__ void kf_sums(const double* __restrict__ partials, double* __restrict__ out, int W, const int* __restrict__ kf_item_start,
                                        unsigned int* __restrict__ ticket, int nitems, bool& is_last, LastBlock last_block) {
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) {
    const unsigned int tk = atomicAdd(ticket, 1u);
    is_last = (tk == (unsigned)nitems - 1);
  }
  __syncthreads();
  if (is_last) {
    __threadfence();
    for (int o = threadIdx.x; o < W * NACC; o += EV_T) {
      const int kf = o / NACC, k = o - kf * NACC;
      // same left-to-right order as a plain loop, but eight independent L2 loads in flight at a time: this tail is a serial
      // chain of ~15 dependent loads per output otherwise (the last block runs alone on the GPU)
      double v = 0.0;
      int b = kf_item_start[kf];
      const int b1 = kf_item_start[kf + 1];
      for (; b + 8 <= b1; b += 8) {
        double p[8];
#pragma unroll
        for (int u = 0; u < 8; ++u) p[u] = __ldcg(&partials[(size_t)(b + u) * NACC + k]);
#pragma unroll
        for (int u = 0; u < 8; ++u) v += p[u];
      }
      for (; b < b1; ++b) v += __ldcg(&partials[(size_t)b * NACC + k]);
      out[o] = v;
    }
    last_block();
  }
}

// One plane residual of the unary factor: adds its block cost to cost; r (before the Huber scale), the scale, and with WANT_JAC
// the scaled Jacobian row J.  M, t may live in registers or in F; R_lb^-1 and q (ambient columns) are read from F.
template <bool WANT_JAC, int JAC_KIND>
__device__ __forceinline__ void plane_residual(const float4 c4, const float4 n4, const double (&M)[9], const double (&t)[3], const KfFrame& F,
                                               const EvalParams& ep, double& cost, double& r, double& scale, double (&J)[6]) {
  const double s = ep.unit_score ? ep.lidar_const : ep.lidar_const * (double)c4.w;   // Estimator.cpp:3692 score = lidar_const*weight; front end: no score
  const double dx = (double)c4.x - ep.t_lb[0], dy = (double)c4.y - ep.t_lb[1], dz = (double)c4.z - ep.t_lb[2];
  double a[3]; mat_vec3(M, dx, dy, dz, a);                   // a = R(q) q_lb^-1 (cp - t_lb)
  const double nx = (double)n4.x, ny = (double)n4.y, nz = (double)n4.z;
  r = s * (nx * (a[0] + t[0]) + ny * (a[1] + t[1]) + nz * (a[2] + t[2]) + (double)n4.w);
  cost += huber_scale(r, ep.huber_delta, scale);
  if (WANT_JAC) {
    const double ss = s * scale;
    J[0] = ss * nx; J[1] = ss * ny; J[2] = ss * nz;
    if (JAC_KIND == 0) {
      // tangent (Ceres QuaternionParameterization):  2 s (a x n)
      const double s2 = 2.0 * ss;
      J[3] = s2 * (a[1] * nz - a[2] * ny);
      J[4] = s2 * (a[2] * nx - a[0] * nz);
      J[5] = s2 * (a[0] * ny - a[1] * nx);
    } else {
      // ambient x,y,z columns (MarginalizationFactor.cpp:9-12):
      //   s [ 2w (p_b x n) + 2( (u.p_b) n + (n.u) p_b - 2 (n.p_b) u ) ]
      double pb[3]; mat_vec3(F.Rlbi, dx, dy, dz, pb);
      const double w = F.q[0], ux = F.q[1], uy = F.q[2], uz = F.q[3];
      const double udp = ux * pb[0] + uy * pb[1] + uz * pb[2];
      const double ndu = nx * ux + ny * uy + nz * uz;
      const double ndp = nx * pb[0] + ny * pb[1] + nz * pb[2];
      J[3] = ss * (2.0 * w * (pb[1] * nz - pb[2] * ny) + 2.0 * (udp * nx + ndu * pb[0] - 2.0 * ndp * ux));
      J[4] = ss * (2.0 * w * (pb[2] * nx - pb[0] * nz) + 2.0 * (udp * ny + ndu * pb[1] - 2.0 * ndp * uy));
      J[5] = ss * (2.0 * w * (pb[0] * ny - pb[1] * nx) + 2.0 * (udp * nz + ndu * pb[2] - 2.0 * ndp * uz));
    }
  }
}

// the 21 upper-triangular J^T J and 6 J^T r sums of one scaled residual r with Jacobian row J
__device__ __forceinline__ void unary_sums(const double (&J)[6], double r, double (&acc)[NACC]) {
  int k = 0;
#pragma unroll
  for (int p = 0; p < 6; ++p)
#pragma unroll
    for (int c = p; c < 6; ++c) acc[k++] += J[p] * J[c];
#pragma unroll
  for (int p = 0; p < 6; ++p) acc[21 + p] += J[p] * r;
}

// per-residual math of the unary plane factor; M, t (and R_lb^-1, q for the marginalisation variant) live in registers
template <bool WANT_JAC, int JAC_KIND>
__device__ __forceinline__ void unary_accumulate(const float4 c4, const float4 n4, const double (&M)[9], const double (&t)[3],
                                                 const KfFrame& F, const EvalParams& ep, double (&acc)[NACC]) {
  double r, scale, J[6];
  plane_residual<WANT_JAC, JAC_KIND>(c4, n4, M, t, F, ep, acc[27], r, scale, J);
  if (WANT_JAC) unary_sums(J, r * scale, acc);
}

// One block per work item (a run of one keyframe's residuals, sized so the whole launch is about one wave of
// 2 blocks/SM).  Loads are issued two iterations ahead of their use (4 x 16 B in flight per thread).
// poses of up to EV_MAXW keyframes travel in the kernel parameters (no host-to-device copy on the per-iteration path)
struct PoseArgs { double p[EV_MAXW * 7]; };

#ifndef GLIO_EVAL_MINBLOCKS
#define GLIO_EVAL_MINBLOCKS 2
#endif
template <bool WANT_JAC, int JAC_KIND, bool POSE_ARGS>
__global__ void __launch_bounds__(EV_T, GLIO_EVAL_MINBLOCKS) k_eval_unary(const EvalItem* __restrict__ items, int nitems, int W,
                                                        const double* __restrict__ poses, const __grid_constant__ PoseArgs pa, EvalParams ep,
                                                        double* __restrict__ partials, double* __restrict__ out,
                                                        const int* __restrict__ kf_item_start, unsigned int* __restrict__ ticket,
                                                        unsigned int* done_flag, unsigned int epoch) {
  __shared__ KfFrame F;
  __shared__ double red[EV_T / 32][NACC];
  __shared__ bool is_last;
  const EvalItem it = items[blockIdx.x];
  if (threadIdx.x == 0) kf_frame<true>(POSE_ARGS ? pa.p + 7 * it.kf : poses + 7 * it.kf, ep, F);
  __syncthreads();
  double M[9], t[3];
#pragma unroll
  for (int k = 0; k < 9; ++k) M[k] = F.M[k];
#pragma unroll
  for (int k = 0; k < 3; ++k) t[k] = F.t[k];

  double acc[NACC];
#pragma unroll
  for (int k = 0; k < NACC; ++k) acc[k] = 0.0;

  const int n = it.count;
  int i = threadIdx.x;
  // software pipeline, depth 2
  float4 c0, n0, c1, n1;
  if (i < n) { c0 = __ldg(&it.cpw[i]); n0 = __ldg(&it.nsd[i]); }
  if (i + EV_T < n) { c1 = __ldg(&it.cpw[i + EV_T]); n1 = __ldg(&it.nsd[i + EV_T]); }
  for (; i < n; i += 2 * EV_T) {
    const float4 ca = c0, na = n0, cb = c1, nb = n1;
    const bool has_b = i + EV_T < n;
    if (i + 2 * EV_T < n) { c0 = __ldg(&it.cpw[i + 2 * EV_T]); n0 = __ldg(&it.nsd[i + 2 * EV_T]); }
    if (i + 3 * EV_T < n) { c1 = __ldg(&it.cpw[i + 3 * EV_T]); n1 = __ldg(&it.nsd[i + 3 * EV_T]); }
    unary_accumulate<WANT_JAC, JAC_KIND>(ca, na, M, t, F, ep, acc);
    if (has_b) unary_accumulate<WANT_JAC, JAC_KIND>(cb, nb, M, t, F, ep, acc);
  }

  block_partials<NACC, EV_T, WANT_JAC>(acc, red, partials);
  kf_sums(partials, out, W, kf_item_start, ticket, nitems, is_last, [&] {
    // `out` may be host-mapped pinned memory: publish the W x NACC doubles system-wide, then raise the epoch flag the
    // host spins on (no device-to-host copy, no stream synchronisation on the per-iteration path)
    if (done_flag) { __threadfence_system(); __syncthreads(); }
    if (threadIdx.x == 0) { *ticket = 0u; if (done_flag) *(volatile unsigned int*)done_flag = epoch; }
  });
}

// the instantiation for (want_jac, jac_kind, poses in the kernel parameters)
using UnaryKernel = decltype(&k_eval_unary<false, 0, false>);
UnaryKernel unary_kernel(bool want_jac, int jac_kind, bool pose_args) {
  if (pose_args) return !want_jac ? k_eval_unary<false, 0, true> : jac_kind == 0 ? k_eval_unary<true, 0, true> : k_eval_unary<true, 1, true>;
  return !want_jac ? k_eval_unary<false, 0, false> : jac_kind == 0 ? k_eval_unary<true, 0, false> : k_eval_unary<true, 1, false>;
}

void eval_unary_run(const EvalItem* d_items, int nitems, int W, const double* d_poses, const EvalParams& ep, int jac_kind,
                    bool want_jac, double* d_partials, double* d_out, const int* d_kf_item_start, unsigned int* d_ticket,
                    cudaStream_t st, LaunchCounter& lc, unsigned int* done_flag, unsigned int epoch, const double* h_poses) {
  if (nitems <= 0) {
    GLIO_CUDA_TRY(cudaMemsetAsync(d_out, 0, (size_t)W * NACC * sizeof(double), st));
    return;
  }
  static const PoseArgs none{};
  PoseArgs pa;
  const bool pose_args = h_poses && W <= EV_MAXW;
  if (pose_args) memcpy(pa.p, h_poses, (size_t)W * 7 * sizeof(double));
  lc.begin(want_jac ? "k_eval_unary" : "k_eval_unary_cost", st);
  unary_kernel(want_jac, jac_kind, pose_args)<<<nitems, EV_T, 0, st>>>(d_items, nitems, W, pose_args ? nullptr : d_poses, pose_args ? pa : none, ep,
                                                                       d_partials, d_out, d_kf_item_start, d_ticket, done_flag, epoch);
  lc.end(st);
  GLIO_CUDA_TRY(cudaGetLastError());
}

// per-residual r, J (the Ceres-API view of one keyframe's residual blocks)
__global__ void __launch_bounds__(256) k_unary_residuals(const float4* __restrict__ cpw, const float4* __restrict__ nsd, int64_t n,
                                                         const double* __restrict__ pose, EvalParams ep, int jac_kind,
                                                         double* __restrict__ r_out, double* __restrict__ J_out) {
  __shared__ KfFrame F;
  if (threadIdx.x == 0) kf_frame<true>(pose, ep, F);
  __syncthreads();
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float4 c4 = cpw[i], n4 = nsd[i];
  double cost = 0.0, r, scale, J[6];
  if (jac_kind == 0) plane_residual<true, 0>(c4, n4, F.M, F.t, F, ep, cost, r, scale, J);
  else plane_residual<true, 1>(c4, n4, F.M, F.t, F, ep, cost, r, scale, J);
  r_out[i] = r * scale;
#pragma unroll
  for (int k = 0; k < 6; ++k) J_out[6 * i + k] = J[k];
}

void eval_unary_residuals_run(const float4* cpw, const float4* nsd, int64_t n, const double* d_pose, const EvalParams& ep,
                              int jac_kind, double* d_r, double* d_J, cudaStream_t st, LaunchCounter& lc) {
  if (n <= 0) return;
  lc.begin("k_unary_residuals", st); k_unary_residuals<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(cpw, nsd, n, d_pose, ep, jac_kind, d_r, d_J); lc.end(st);
  GLIO_CUDA_TRY(cudaGetLastError());
}



// ---------------------------------------------------------------------------------------------------------------
// K2e: point-to-edge residuals, LidarEdgeFactor (LidarKeyframeFactor.h:12-70; defined by the reference but never
// instantiated, SURVEY fact 1):  lp = R(q) q_lb^-1 (cp - t_lb) + t ;  r = s |(lp-a) x (lp-b)| / |a-b|
// closed form (SURVEY 8 a-6):  e = (lp-a) x (lp-b), gv = s/|a-b| ((a-b) x e/|e|), dr/dt = gv, dr/ddelta = 2 (R p_b x gv).
// Inputs per residual: cp, a, b (float3 each) + s -> 3 x 16 B loads (s rides in cp.w).
// ---------------------------------------------------------------------------------------------------------------
// JAC_KIND 0: Ceres' tangent rotation columns (solve path); 1: the ambient x,y,z quaternion columns of MarginalizationFactor.cpp:9-17
// (marginalisation path), the K2 rule with gv in place of the plane's s n:  2w (p_b x gv) + 2((u.p_b) gv + (gv.u) p_b - 2 (gv.p_b) u)
template <bool WANT_JAC, int JAC_KIND>
__global__ void __launch_bounds__(EV_T) k_eval_edge(const EdgeItem* __restrict__ items, int nitems, int W, const double* __restrict__ poses,
                                                    EvalParams ep, double* __restrict__ partials, double* __restrict__ out,
                                                    const int* __restrict__ kf_item_start, unsigned int* __restrict__ ticket) {
  __shared__ KfFrame F;
  __shared__ double red[EV_T / 32][NACC];
  __shared__ bool is_last;
  const EdgeItem it = items[blockIdx.x];
  if (threadIdx.x == 0) kf_frame<JAC_KIND == 1>(poses + 7 * it.kf, ep, F);
  __syncthreads();
  double acc[NACC];
#pragma unroll
  for (int k = 0; k < NACC; ++k) acc[k] = 0.0;
  for (int i = threadIdx.x; i < it.count; i += EV_T) {
    const float4 c4 = __ldg(&it.cps[i]);
    const float4 a4 = __ldg(&it.pa[i]);
    const float4 b4 = __ldg(&it.pb[i]);
    const double s = (double)c4.w;
    const double dx = (double)c4.x - ep.t_lb[0], dy = (double)c4.y - ep.t_lb[1], dz = (double)c4.z - ep.t_lb[2];
    double a1[3]; mat_vec3(F.M, dx, dy, dz, a1);
    const double lp[3] = {a1[0] + F.t[0], a1[1] + F.t[1], a1[2] + F.t[2]};
    const double u[3] = {lp[0] - (double)a4.x, lp[1] - (double)a4.y, lp[2] - (double)a4.z};
    const double v[3] = {lp[0] - (double)b4.x, lp[1] - (double)b4.y, lp[2] - (double)b4.z};
    const double e[3] = {u[1] * v[2] - u[2] * v[1], u[2] * v[0] - u[0] * v[2], u[0] * v[1] - u[1] * v[0]};
    const double de[3] = {(double)a4.x - (double)b4.x, (double)a4.y - (double)b4.y, (double)a4.z - (double)b4.z};
    const double en = sqrt(e[0] * e[0] + e[1] * e[1] + e[2] * e[2]);
    const double dn = sqrt(de[0] * de[0] + de[1] * de[1] + de[2] * de[2]);
    double r = en / dn * s;
    double scale;
    acc[27] += huber_scale(r, ep.huber_delta, scale);
    if (WANT_JAC) {
      const double k = s / dn * scale / en;
      const double gv[3] = {k * (de[1] * e[2] - de[2] * e[1]), k * (de[2] * e[0] - de[0] * e[2]), k * (de[0] * e[1] - de[1] * e[0])};
      double J[6] = {gv[0], gv[1], gv[2], 2.0 * (a1[1] * gv[2] - a1[2] * gv[1]), 2.0 * (a1[2] * gv[0] - a1[0] * gv[2]), 2.0 * (a1[0] * gv[1] - a1[1] * gv[0])};
      if (JAC_KIND == 1) {
        double pb[3]; mat_vec3(F.Rlbi, dx, dy, dz, pb);
        const double w = F.q[0], ux = F.q[1], uy = F.q[2], uz = F.q[3];
        const double udp = ux * pb[0] + uy * pb[1] + uz * pb[2];
        const double gdu = gv[0] * ux + gv[1] * uy + gv[2] * uz;
        const double gdp = gv[0] * pb[0] + gv[1] * pb[1] + gv[2] * pb[2];
        J[3] = 2.0 * w * (pb[1] * gv[2] - pb[2] * gv[1]) + 2.0 * (udp * gv[0] + gdu * pb[0] - 2.0 * gdp * ux);
        J[4] = 2.0 * w * (pb[2] * gv[0] - pb[0] * gv[2]) + 2.0 * (udp * gv[1] + gdu * pb[1] - 2.0 * gdp * uy);
        J[5] = 2.0 * w * (pb[0] * gv[1] - pb[1] * gv[0]) + 2.0 * (udp * gv[2] + gdu * pb[2] - 2.0 * gdp * uz);
      }
      unary_sums(J, r * scale, acc);
    }
  }
  block_partials<NACC, EV_T, WANT_JAC>(acc, red, partials);
  kf_sums(partials, out, W, kf_item_start, ticket, nitems, is_last, [&] { if (threadIdx.x == 0) *ticket = 0u; });
}

// the instantiation for (want_jac, jac_kind)
using EdgeKernel = decltype(&k_eval_edge<false, 0>);
EdgeKernel edge_kernel(bool want_jac, int jac_kind) {
  return !want_jac ? k_eval_edge<false, 0> : jac_kind == 0 ? k_eval_edge<true, 0> : k_eval_edge<true, 1>;
}

void eval_edge_run(const EdgeItem* d_items, int nitems, int W, const double* d_poses, const EvalParams& ep, int jac_kind, bool want_jac,
                   double* d_partials, double* d_out, const int* d_kf_item_start, unsigned int* d_ticket, cudaStream_t st, LaunchCounter& lc) {
  if (nitems <= 0) { GLIO_CUDA_TRY(cudaMemsetAsync(d_out, 0, (size_t)W * NACC * sizeof(double), st)); return; }
  lc.begin(want_jac ? "k_eval_edge" : "k_eval_edge_cost", st);
  edge_kernel(want_jac, jac_kind)<<<nitems, EV_T, 0, st>>>(d_items, nitems, W, d_poses, ep, d_partials, d_out, d_kf_item_start, d_ticket);
  lc.end(st);
  GLIO_CUDA_TRY(cudaGetLastError());
}

// ---------------------------------------------------------------------------------------------------------------
// K2b: binary (scan-to-multiscan) plane factors, BinaryLidarPlaneNormFactor (LidarKeyframeFactor.h:124-164):
//   p_w = R(q_c) cp + t_c ;  N = R(q_o) n_l ;  c_w = R(q_o) c_l + t_o ;  r = s N.(p_w - c_w),  s = batch_score * weight
// tangent Jacobians (SURVEY 8 a-5):  J_c = [u | v],  J_o = [-u | z]  with  u = s N,  v = 2 s (R(q_c)cp x N),  z = 2 s (N x (p_w - t_o)).
// Because J_o's translation part is -u, the 12x12 outer product needs only 45 distinct sums (+9 for J^T r, +1 cost): the
// GLIO_NACC_BIN layout, accumulated by pair_accumulate.
// HBM traffic per residual: 16 B (cp, weight) + 48 B (n_l, c_l as the reference stores them: double) = 64 B.
// ---------------------------------------------------------------------------------------------------------------
constexpr int NB = GLIO_NACC_BIN;
constexpr int BIN_T = 128;

struct PairFrame { double R1[9], t1[3], R2[9], t2[3]; };

// F from the poses P1 of cur and P2 of oth
__device__ __forceinline__ void pair_frame(const double* P1, const double* P2, PairFrame& F) {
  double q1[4] = {P1[3], P1[4], P1[5], P1[6]}, q2[4] = {P2[3], P2[4], P2[5], P2[6]};
  quat_to_mat(q1, F.R1); quat_to_mat(q2, F.R2);
  F.t1[0] = P1[0]; F.t1[1] = P1[1]; F.t1[2] = P1[2]; F.t2[0] = P2[0]; F.t2[1] = P2[1]; F.t2[2] = P2[2];
}

// the 54 J^T J / J^T r sums of one residual r with J_c = [u | v], J_o = [-u | z] (GLIO_NACC_BIN, common.cuh; the cost is the caller's)
__device__ __forceinline__ void pair_accumulate(const double (&u)[3], const double (&v)[3], const double (&z)[3], double r, double (&acc)[NB]) {
  int k = 0;
#pragma unroll
  for (int a = 0; a < 3; ++a)
#pragma unroll
    for (int b = a; b < 3; ++b) acc[k++] += u[a] * u[b];          // uu  [0,6)
#pragma unroll
  for (int a = 0; a < 3; ++a)
#pragma unroll
    for (int b = 0; b < 3; ++b) acc[k++] += u[a] * v[b];          // uv  [6,15)
#pragma unroll
  for (int a = 0; a < 3; ++a)
#pragma unroll
    for (int b = a; b < 3; ++b) acc[k++] += v[a] * v[b];          // vv  [15,21)
#pragma unroll
  for (int a = 0; a < 3; ++a)
#pragma unroll
    for (int b = 0; b < 3; ++b) acc[k++] += u[a] * z[b];          // uz  [21,30)
#pragma unroll
  for (int a = 0; a < 3; ++a)
#pragma unroll
    for (int b = 0; b < 3; ++b) acc[k++] += v[a] * z[b];          // vz  [30,39)
#pragma unroll
  for (int a = 0; a < 3; ++a)
#pragma unroll
    for (int b = a; b < 3; ++b) acc[k++] += z[a] * z[b];          // zz  [39,45)
#pragma unroll
  for (int a = 0; a < 3; ++a) { acc[45 + a] += r * u[a]; acc[48 + a] += r * v[a]; acc[51 + a] += r * z[a]; }
}

template <bool WANT_JAC>
__global__ void __launch_bounds__(BIN_T) k_eval_binary(const BinItem* __restrict__ items, const double* __restrict__ poses, double score_scale,
                                                       double huber_delta, double* __restrict__ partials) {
  __shared__ PairFrame F;
  __shared__ double red[BIN_T / 32][NB];
  const BinItem it = items[blockIdx.x];
  if (threadIdx.x == 0) pair_frame(poses + 7 * it.kf_c, poses + 7 * it.kf_o, F);
  __syncthreads();
  double acc[NB];
#pragma unroll
  for (int k = 0; k < NB; ++k) acc[k] = 0.0;
  for (int i = threadIdx.x; i < it.count; i += BIN_T) {
    const float4 c4 = __ldg(&it.cpw[i]);
    const double2* ncp = reinterpret_cast<const double2*>(it.nc + 6 * (int64_t)i);
    const double2 n01 = __ldg(ncp), n2c0 = __ldg(ncp + 1), c12 = __ldg(ncp + 2);
    const double s = score_scale * (double)c4.w;
    double a1[3]; mat_vec3(F.R1, (double)c4.x, (double)c4.y, (double)c4.z, a1);
    const double pw[3] = {a1[0] + F.t1[0], a1[1] + F.t1[1], a1[2] + F.t1[2]};
    double N[3]; mat_vec3(F.R2, n01.x, n01.y, n2c0.x, N);
    double co[3]; mat_vec3(F.R2, n2c0.y, c12.x, c12.y, co);
    const double pm[3] = {pw[0] - F.t2[0], pw[1] - F.t2[1], pw[2] - F.t2[2]};     // p_w - t_o
    const double dd[3] = {pm[0] - co[0], pm[1] - co[1], pm[2] - co[2]};           // p_w - c_w
    double r = s * (N[0] * dd[0] + N[1] * dd[1] + N[2] * dd[2]);
    double scale;
    acc[54] += huber_scale(r, huber_delta, scale);
    if (WANT_JAC) {
      const double ss = s * scale;
      const double u[3] = {ss * N[0], ss * N[1], ss * N[2]};
      const double v[3] = {2.0 * ss * (a1[1] * N[2] - a1[2] * N[1]), 2.0 * ss * (a1[2] * N[0] - a1[0] * N[2]), 2.0 * ss * (a1[0] * N[1] - a1[1] * N[0])};
      const double z[3] = {2.0 * ss * (N[1] * pm[2] - N[2] * pm[1]), 2.0 * ss * (N[2] * pm[0] - N[0] * pm[2]), 2.0 * ss * (N[0] * pm[1] - N[1] * pm[0])};
      pair_accumulate(u, v, z, r * scale, acc);
    }
  }
  block_partials<NB, BIN_T, WANT_JAC>(acc, red, partials);
}

// ---------------------------------------------------------------------------------------------------------------
// K2be: binary point-to-edge factors (glio_batch_use_edges, glio_eval_binary_edge), the conventions of
// BinaryLidarPlaneNormFactor (no extrinsic, the line moves with oth, no loss):
//   p_w = R(q_c) cp + t_c ;  A = R(q_o) a_l + t_o ;  B = R(q_o) b_l + t_o ;  e = (p_w - A) x (p_w - B) ;  r = s |e| / |A - B|
// tangent Jacobians:  J_c = [g | 2 (R(q_c)cp x g)],  J_o = [-g | 2 (g x (p_w - t_o))]  with  g = s/|A-B| ((A-B) x e/|e|),
// i.e. K2b's u, v, z with g in place of s N: the same 55 sums, so k_bin_pair_sums and the block assembly take them unchanged.
// Differences are formed relative to t_o (p_w - t_o and R(q_o) a_l), so kilometre offsets cancel before the cross product.
// A point exactly on its line (|e| = 0) behaves as in K2e: r = 0 and a non-finite g.
// HBM traffic per residual: 3 x 16 B (cp with s in .w, a_l, b_l).
// ---------------------------------------------------------------------------------------------------------------
template <bool WANT_JAC>
__global__ void __launch_bounds__(BIN_T) k_eval_binary_edge(const BinEdgeItem* __restrict__ items, const double* __restrict__ poses,
                                                            double* __restrict__ partials) {
  __shared__ PairFrame F;
  __shared__ double red[BIN_T / 32][NB];
  const BinEdgeItem it = items[blockIdx.x];
  if (threadIdx.x == 0) pair_frame(poses + 7 * it.kf_c, poses + 7 * it.kf_o, F);
  __syncthreads();
  double acc[NB];
#pragma unroll
  for (int k = 0; k < NB; ++k) acc[k] = 0.0;
  for (int i = threadIdx.x; i < it.count; i += BIN_T) {
    const float4 c4 = __ldg(&it.cps[i]);
    const float4 a4 = __ldg(&it.pa[i]);
    const float4 b4 = __ldg(&it.pb[i]);
    const double s = (double)c4.w;
    double a1[3]; mat_vec3(F.R1, (double)c4.x, (double)c4.y, (double)c4.z, a1);
    const double pm[3] = {a1[0] + F.t1[0] - F.t2[0], a1[1] + F.t1[1] - F.t2[1], a1[2] + F.t1[2] - F.t2[2]};   // p_w - t_o
    double ra[3]; mat_vec3(F.R2, (double)a4.x, (double)a4.y, (double)a4.z, ra);                             // A - t_o
    double rb[3]; mat_vec3(F.R2, (double)b4.x, (double)b4.y, (double)b4.z, rb);                             // B - t_o
    const double u[3] = {pm[0] - ra[0], pm[1] - ra[1], pm[2] - ra[2]};
    const double w[3] = {pm[0] - rb[0], pm[1] - rb[1], pm[2] - rb[2]};
    const double e[3] = {u[1] * w[2] - u[2] * w[1], u[2] * w[0] - u[0] * w[2], u[0] * w[1] - u[1] * w[0]};
    const double de[3] = {ra[0] - rb[0], ra[1] - rb[1], ra[2] - rb[2]};
    const double en = sqrt(e[0] * e[0] + e[1] * e[1] + e[2] * e[2]);
    const double dn = sqrt(de[0] * de[0] + de[1] * de[1] + de[2] * de[2]);
    const double r = en / dn * s;
    acc[54] += 0.5 * (r * r);
    if (WANT_JAC) {
      const double k = s / dn / en;
      const double gv[3] = {k * (de[1] * e[2] - de[2] * e[1]), k * (de[2] * e[0] - de[0] * e[2]), k * (de[0] * e[1] - de[1] * e[0])};
      const double v[3] = {2.0 * (a1[1] * gv[2] - a1[2] * gv[1]), 2.0 * (a1[2] * gv[0] - a1[0] * gv[2]), 2.0 * (a1[0] * gv[1] - a1[1] * gv[0])};
      const double z[3] = {2.0 * (gv[1] * pm[2] - gv[2] * pm[1]), 2.0 * (gv[2] * pm[0] - gv[0] * pm[2]), 2.0 * (gv[0] * pm[1] - gv[1] * pm[0])};
      pair_accumulate(gv, v, z, r, acc);
    }
  }
  block_partials<NB, BIN_T, WANT_JAC>(acc, red, partials);
}

// S += S_edge over n_pairs x NB sums (the binary plane and edge factors of a pair share one block assembly)
__global__ void __launch_bounds__(256) k_bin_pair_add(double* __restrict__ S, const double* __restrict__ S_edge, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) S[i] += S_edge[i];
}

// per pair: sum of its items' partials, in item order (deterministic)
__global__ void __launch_bounds__(64) k_bin_pair_sums(const double* __restrict__ partials, const int* __restrict__ pair_item_start,
                                                      double* __restrict__ pair_sums) {
  const int p = blockIdx.x, k = threadIdx.x;
  if (k >= NB) return;
  double v = 0.0;
  for (int b = pair_item_start[p]; b < pair_item_start[p + 1]; ++b) v += partials[(size_t)b * NB + k];
  pair_sums[(size_t)p * NB + k] = v;
}

// ---------------------------------------------------------------------------------------------------------------
// Block assembly of the pair kinds (K2b / K2be, K2p, K2g, K2i): per-pair sums S (n_pairs x L::NS) -> per keyframe the L::ND
// entries of its diagonal block, g and cost, each summed over the keyframe's incidence list in order (deterministic, no atomics),
// and with WANT_JAC per pair its L::NO off-diagonal entries.  A layout L says where the entries come from: L::diag(s, role, e) is
// the term one incidence with pair sums s adds to entry e, +0.0 for none (the sum starts at +0.0, so it is never -0.0, and adding
// +0.0 leaves its bits as they are); L::off(s, e) is off-diagonal entry e.  Without WANT_JAC only the cost entry L::COST is summed,
// the others are written as 0.
// Thread t < K * ND: diag entry (kf, e), with no terms for kf >= n_inc_kf, added to diag's contents when add, else written; then,
// with WANT_JAC, one thread per entry of the n_pairs off-diagonal blocks.
// ---------------------------------------------------------------------------------------------------------------
template <class L, bool WANT_JAC>
__global__ void __launch_bounds__(256) k_pair_assemble(const double* __restrict__ S, int K, int n_pairs, int n_inc_kf,
                                                       const int* __restrict__ kf_inc_start, const BinIncidence* __restrict__ inc, bool add,
                                                       double* __restrict__ diag, double* __restrict__ off) {
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t nd = (int64_t)K * L::ND;
  if (t < nd) {
    const int kf = (int)(t / L::ND), e = (int)(t - (int64_t)kf * L::ND);
    double v = 0.0;
    if (kf < n_inc_kf && (WANT_JAC || e == L::COST)) {
      for (int i = kf_inc_start[kf]; i < kf_inc_start[kf + 1]; ++i) v += L::diag(S + (size_t)inc[i].pair * L::NS, inc[i].role, e);
    }
    diag[t] = add ? diag[t] + v : v;
  } else if (WANT_JAC) {
    const int64_t o = t - nd;
    if (o < (int64_t)n_pairs * L::NO) {
      const int64_t pr = o / L::NO;
      off[o] = L::off(S + pr * L::NS, (int)(o - pr * L::NO));
    }
  }
}

template <class L>
void pair_assemble_run(const double* d_sums, int K, int n_pairs, int n_inc_kf, const int* d_kf_inc_start, const BinIncidence* d_inc,
                       bool want_jac, bool add, double* d_diag, double* d_off, cudaStream_t st) {
  const int64_t n = (int64_t)K * L::ND + (want_jac ? (int64_t)n_pairs * L::NO : 0);
  (want_jac ? k_pair_assemble<L, true> : k_pair_assemble<L, false>)<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(
      d_sums, K, n_pairs, n_inc_kf, d_kf_inc_start, d_inc, add, d_diag, d_off);
  GLIO_CUDA_TRY(cudaGetLastError());
}

// K2b / K2be: diagonal 6x6 (21 upper-tri) + g (6) + per-KF cost share (cost is attributed to cur); off-diagonal 6x6 (row = cur
// tangent, col = oth tangent)
struct BinLayout {
  static constexpr int NS = NB, ND = GLIO_NACC, NO = 36, COST = 27;
  __device__ static __forceinline__ int sym3(int a, int b) { return a <= b ? (a * 3 - a * (a - 1) / 2 + (b - a)) : (b * 3 - b * (b - 1) / 2 + (a - b)); }
  __device__ static __forceinline__ double diag(const double* s, int role, int e) {
    if (e < 21) {
      // decode entry e: [0,21) upper-tri (p<=q) of the 6x6, [21,27) g, 27 cost
      int p = 0, q = 0, k = e;
      for (p = 0; p < 6; ++p) { if (k < 6 - p) { q = p + k; break; } k -= 6 - p; }
      if (p < 3 && q < 3) return s[sym3(p, q)];                                            // uu (both roles)
      if (p < 3) return role == 0 ? s[6 + 3 * p + (q - 3)] : -s[21 + 3 * p + (q - 3)];    // uv | -uz
      return role == 0 ? s[15 + sym3(p - 3, q - 3)] : s[39 + sym3(p - 3, q - 3)];          // vv | zz
    }
    if (e < 27) {
      const int c = e - 21;
      if (c < 3) return role == 0 ? s[45 + c] : -s[45 + c];                                // r u | -r u
      return role == 0 ? s[48 + (c - 3)] : s[51 + (c - 3)];                                // r v | r z
    }
    return role == 0 ? s[54] : 0.0;
  }
  __device__ static __forceinline__ double off(const double* s, int e) {
    const int p = e / 6, q = e % 6;
    if (p < 3 && q < 3) return -s[sym3(p, q)];                 // -u u^T
    if (p < 3) return s[21 + 3 * p + (q - 3)];                 //  u z^T
    if (q < 3) return -s[6 + 3 * q + (p - 3)];                 // -v u^T
    return s[30 + 3 * (p - 3) + (q - 3)];                      //  v z^T
  }
};
template void pair_assemble_run<BinLayout>(const double*, int, int, int, const int*, const BinIncidence*, bool, bool, double*, double*,
                                           cudaStream_t);

void eval_binary_run(const BinItem* d_items, int nitems, const int* d_pair_item_start, int n_pairs, int K, const double* d_poses,
                     double score_scale, double huber_delta, bool want_jac, double* d_partials, double* d_pair_sums,
                     const int* d_kf_inc_start, const BinIncidence* d_inc, double* d_diag, double* d_off,
                     cudaStream_t st, LaunchCounter& lc, const double* d_pair_sums_edge) {
  if (nitems > 0) {
    lc.begin(want_jac ? "k_eval_binary" : "k_eval_binary_cost", st);
    (want_jac ? k_eval_binary<true> : k_eval_binary<false>)<<<nitems, BIN_T, 0, st>>>(d_items, d_poses, score_scale, huber_delta, d_partials);
    lc.end(st);
  }
  if (n_pairs > 0) {
    lc.begin("k_bin_pair_sums", st); k_bin_pair_sums<<<n_pairs, 64, 0, st>>>(d_partials, d_pair_item_start, d_pair_sums); lc.end(st);
    if (d_pair_sums_edge) {
      const int n = n_pairs * NB;
      lc.begin("k_bin_pair_add", st); k_bin_pair_add<<<(n + 255) / 256, 256, 0, st>>>(d_pair_sums, d_pair_sums_edge, n); lc.end(st);
    }
  }
  lc.begin("k_bin_assemble", st);
  pair_assemble_run<BinLayout>(d_pair_sums, K, n_pairs, K, d_kf_inc_start, d_inc, want_jac, false, d_diag, d_off, st);
  lc.end(st);
}

void eval_binary_edge_run(const BinEdgeItem* d_items, int nitems, const int* d_pair_item_start, int n_pairs, const double* d_poses,
                          bool want_jac, double* d_partials, double* d_pair_sums, cudaStream_t st, LaunchCounter& lc) {
  if (nitems > 0) {
    lc.begin(want_jac ? "k_eval_binary_edge" : "k_eval_binary_edge_cost", st);
    (want_jac ? k_eval_binary_edge<true> : k_eval_binary_edge<false>)<<<nitems, BIN_T, 0, st>>>(d_items, d_poses, d_partials);
    lc.end(st);
  }
  if (n_pairs > 0) {
    lc.begin("k_bin_pair_sums", st); k_bin_pair_sums<<<n_pairs, 64, 0, st>>>(d_partials, d_pair_item_start, d_pair_sums); lc.end(st);
  }
  GLIO_CUDA_TRY(cudaGetLastError());
}

// ---------------------------------------------------------------------------------------------------------------
// K2p: the batch refinement's pose factors (glio_batch_set_pose_factors), as their AutoDiff functors evaluate them with Eigen:
//   relative  (LidarPoseFactorBatchRelativeAutoDiff, LidarPoseFactor.h:54-95; blocks t_i, q_i, t_j, q_j):
//     E = (dq^-1 q_i^-1) q_j,  r[0..2] = 10 (2 vec(E)),  r[3..5] = 20 (q_i^-1 (t_j - t_i) - dp)
//   attitude  (delta_q_factor_auto, LidarKeyframeFactor.h:281-303; blocks q_i, q_j):  r = 10000 vec(E)
// with q^-1 = conj(q) / |q|^2 (0 for q = 0) and q v = v + 2w (u x v) + 2 u x (u x v), for any (not necessarily unit) q.
// Tangent columns: the directional derivative of r along Ceres' QuaternionParameterization column k, d q = [0, e_k] (x) q, i.e. the
// ambient Jacobian times the 4 x 3 local Jacobian, exact at non-unit quaternions too.
// Layout: one half-warp per distinct pair (a, b); lane l < 12 owns tangent column l of (t_a, d_a, t_b, d_b), walks the pair's
// factors in list order and keeps row l of the pair's 12 x 12 J^T J and entry l of J^T r in registers (12 + 1 doubles); the other
// columns come by shuffle.  k_pair_assemble (PoseLayout) then sums each keyframe's pairs in incidence order.  No floating-point atomics.
// ---------------------------------------------------------------------------------------------------------------
constexpr int NP = GLIO_NACC_POSE;
constexpr int POSE_T = 128;   // 8 pairs per block

__device__ __forceinline__ void qmul(const double a[4], const double b[4], double o[4]) {   // Eigen's quaternion product, (w, x, y, z)
  o[0] = a[0] * b[0] - a[1] * b[1] - a[2] * b[2] - a[3] * b[3];
  o[1] = a[0] * b[1] + a[1] * b[0] + a[2] * b[3] - a[3] * b[2];
  o[2] = a[0] * b[2] + a[2] * b[0] + a[3] * b[1] - a[1] * b[3];
  o[3] = a[0] * b[3] + a[3] * b[0] + a[1] * b[2] - a[2] * b[1];
}
// Eigen's q * v:  uv = 2 (u x v);  v + w uv + u x uv
__device__ __forceinline__ void qrot(const double q[4], const double v[3], double o[3]) {
  const double uv[3] = {2.0 * (q[2] * v[2] - q[3] * v[1]), 2.0 * (q[3] * v[0] - q[1] * v[2]), 2.0 * (q[1] * v[1] - q[2] * v[0])};
  o[0] = v[0] + q[0] * uv[0] + (q[2] * uv[2] - q[3] * uv[1]);
  o[1] = v[1] + q[0] * uv[1] + (q[3] * uv[0] - q[1] * uv[2]);
  o[2] = v[2] + q[0] * uv[2] + (q[1] * uv[1] - q[2] * uv[0]);
}
// derivative of q * v along d q (v fixed): dw uv + w duv + du x uv + u x duv,  duv = 2 (du x v)
__device__ __forceinline__ void qrot_d(const double q[4], const double d[4], const double v[3], double o[3]) {
  const double uv[3] = {2.0 * (q[2] * v[2] - q[3] * v[1]), 2.0 * (q[3] * v[0] - q[1] * v[2]), 2.0 * (q[1] * v[1] - q[2] * v[0])};
  const double du[3] = {2.0 * (d[2] * v[2] - d[3] * v[1]), 2.0 * (d[3] * v[0] - d[1] * v[2]), 2.0 * (d[1] * v[1] - d[2] * v[0])};
  o[0] = d[0] * uv[0] + q[0] * du[0] + (d[2] * uv[2] - d[3] * uv[1]) + (q[2] * du[2] - q[3] * du[1]);
  o[1] = d[0] * uv[1] + q[0] * du[1] + (d[3] * uv[0] - d[1] * uv[2]) + (q[3] * du[0] - q[1] * du[2]);
  o[2] = d[0] * uv[2] + q[0] * du[2] + (d[1] * uv[1] - d[2] * uv[0]) + (q[1] * du[1] - q[2] * du[0]);
}

__device__ __forceinline__ int sym6(int p, int q) { return p * 6 - p * (p - 1) / 2 + (q - p); }   // p <= q

template <bool WANT_JAC>
__global__ void __launch_bounds__(POSE_T) k_pose_pair_sums(const PoseFactor* __restrict__ fl, const int* __restrict__ fstart, int n_pairs,
                                                           const double* __restrict__ poses, double* __restrict__ sums) {
  const int p = blockIdx.x * (POSE_T / 16) + (threadIdx.x >> 4);
  if (p >= n_pairs) return;                       // a half-warp leaves as a whole; the shuffles below stay inside it
  const unsigned mask = 0xffffu << (threadIdx.x & 16);
  const int l = threadIdx.x & 15, comp = l % 6;
  double H[12], gl = 0.0, cost = 0.0;
#pragma unroll
  for (int m = 0; m < 12; ++m) H[m] = 0.0;
  const int f1 = fstart[p + 1];
  for (int k = fstart[p]; k < f1; ++k) {
    const PoseFactor F = fl[k];
    const double* Pi = poses + 7 * F.i;
    const double* Pj = poses + 7 * F.j;
    const double qi[4] = {Pi[3], Pi[4], Pi[5], Pi[6]}, qj[4] = {Pj[3], Pj[4], Pj[5], Pj[6]};
    const double v[3] = {Pj[0] - Pi[0], Pj[1] - Pi[1], Pj[2] - Pi[2]};
    const double nd = F.dq[0] * F.dq[0] + F.dq[1] * F.dq[1] + F.dq[2] * F.dq[2] + F.dq[3] * F.dq[3];
    double A[4] = {0.0, 0.0, 0.0, 0.0};
    if (nd > 0.0) { A[0] = F.dq[0] / nd; A[1] = -F.dq[1] / nd; A[2] = -F.dq[2] / nd; A[3] = -F.dq[3] / nd; }
    const double n2 = qi[0] * qi[0] + qi[1] * qi[1] + qi[2] * qi[2] + qi[3] * qi[3];
    double B[4] = {0.0, 0.0, 0.0, 0.0};
    if (n2 > 0.0) { B[0] = qi[0] / n2; B[1] = -qi[1] / n2; B[2] = -qi[2] / n2; B[3] = -qi[3] / n2; }
    double AB[4], E[4]; qmul(A, B, AB); qmul(AB, qj, E);
    const bool rel = F.kind == 0;
    double r[6];
    if (rel) {
      double Bv[3]; qrot(B, v, Bv);
#pragma unroll
      for (int m = 0; m < 3; ++m) { r[m] = 10.0 * (2.0 * E[1 + m]); r[3 + m] = 20.0 * (Bv[m] - F.dp[m]); }
    } else {
#pragma unroll
      for (int m = 0; m < 3; ++m) { r[m] = 10000.0 * E[1 + m]; r[3 + m] = 0.0; }
    }
    cost += 0.5 * (r[0] * r[0] + r[1] * r[1] + r[2] * r[2] + r[3] * r[3] + r[4] * r[4] + r[5] * r[5]);
    if (WANT_JAC) {
      double c[6] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0};   // column l of J
      const bool is_i = (l < 6) == (F.i < F.j);
      if (l < 12 && comp < 3) {
        if (rel) {
          const double e[3] = {comp == 0 ? 1.0 : 0.0, comp == 1 ? 1.0 : 0.0, comp == 2 ? 1.0 : 0.0};
          double Be[3]; qrot(B, e, Be);
          const double s = is_i ? -20.0 : 20.0;
          c[3] = s * Be[0]; c[4] = s * Be[1]; c[5] = s * Be[2];
        }
      } else if (l < 12) {
        const double w = is_i ? qi[0] : qj[0], x = is_i ? qi[1] : qj[1], y = is_i ? qi[2] : qj[2], z = is_i ? qi[3] : qj[3];
        // [0, e_k] (x) q, k = comp - 3 (the columns of QuaternionParameterization::ComputeJacobian)
        const double d[4] = {comp == 3 ? -x : comp == 4 ? -y : -z, comp == 3 ? w : comp == 4 ? z : -y,
                             comp == 3 ? -z : comp == 4 ? w : x, comp == 3 ? y : comp == 4 ? -x : w};
        double dE[4];
        if (is_i) {
          // d(conj(q) / |q|^2) = (conj(d) - B d|q|^2) / |q|^2, as the Jet quotient forms it
          double dB[4] = {0.0, 0.0, 0.0, 0.0};
          if (n2 > 0.0) {
            const double dn = 2.0 * (qi[0] * d[0] + qi[1] * d[1] + qi[2] * d[2] + qi[3] * d[3]);
            dB[0] = (d[0] - B[0] * dn) / n2; dB[1] = (-d[1] - B[1] * dn) / n2; dB[2] = (-d[2] - B[2] * dn) / n2; dB[3] = (-d[3] - B[3] * dn) / n2;
          }
          double t4[4]; qmul(A, dB, t4); qmul(t4, qj, dE);
          if (rel) { double dBv[3]; qrot_d(B, dB, v, dBv); c[3] = 20.0 * dBv[0]; c[4] = 20.0 * dBv[1]; c[5] = 20.0 * dBv[2]; }
        } else {
          qmul(AB, d, dE);
        }
        const double s = rel ? 20.0 : 10000.0;
        c[0] = s * dE[1]; c[1] = s * dE[2]; c[2] = s * dE[3];
      }
      gl += c[0] * r[0] + c[1] * r[1] + c[2] * r[2] + c[3] * r[3] + c[4] * r[4] + c[5] * r[5];
#pragma unroll
      for (int m = 0; m < 12; ++m) {
        double s = 0.0;
#pragma unroll
        for (int q = 0; q < 6; ++q) s += c[q] * __shfl_sync(mask, c[q], m, 16);
        H[m] += s;
      }
    }
  }
  double* S = sums + (size_t)p * NP;
  if (WANT_JAC) {
    if (l < 6) {
#pragma unroll
      for (int m = 0; m < 6; ++m) if (m >= l) S[sym6(l, m)] = H[m];
#pragma unroll
      for (int m = 0; m < 6; ++m) S[42 + 6 * l + m] = H[6 + m];
    } else if (l < 12) {
#pragma unroll
      for (int m = 6; m < 12; ++m) if (m >= l) S[21 + sym6(l - 6, m - 6)] = H[m];
    }
    if (l < 12) S[78 + l] = gl;
  }
  if (l == 0) S[90] = cost;
}

// K2p: the GLIO_NACC layout per keyframe, the ab blocks per pair
struct PoseLayout {
  static constexpr int NS = NP, ND = GLIO_NACC, NO = 36, COST = 27;
  __device__ static __forceinline__ double diag(const double* s, int role, int e) {
    if (e < 21) return s[21 * role + e];                       // aa | bb
    if (e < 27) return s[78 + 6 * role + (e - 21)];            // g_a | g_b
    return role == 0 ? s[90] : 0.0;                            // the cost goes to a
  }
  __device__ static __forceinline__ double off(const double* s, int e) { return s[42 + e]; }
};

void eval_pose_run(const PoseFactor* d_f, const int* d_fstart, int n_pairs, int K, int n_inc_kf, const int* d_kf_inc_start,
                   const BinIncidence* d_inc, const double* d_poses, bool want_jac, bool add, double* d_sums, double* d_diag, double* d_off,
                   cudaStream_t st, LaunchCounter& lc) {
  if (n_pairs > 0) {
    const int nb = (n_pairs + POSE_T / 16 - 1) / (POSE_T / 16);
    lc.begin(want_jac ? "k_pose_pair_sums" : "k_pose_pair_sums_cost", st);
    (want_jac ? k_pose_pair_sums<true> : k_pose_pair_sums<false>)<<<nb, POSE_T, 0, st>>>(d_f, d_fstart, n_pairs, d_poses, d_sums);
    lc.end(st);
  }
  lc.begin("k_pose_assemble", st);
  pair_assemble_run<PoseLayout>(d_sums, K, n_pairs, n_inc_kf, d_kf_inc_start, d_inc, want_jac, add, d_diag, d_off, st);
  lc.end(st);
}

// ---------------------------------------------------------------------------------------------------------------
// K2g: the batch refinement's double-differenced pseudorange factors (glio_batch_set_dd_psr_factors), as dd_psr_factor_20's
// Evaluate forms them (dd_psr_factor.hpp:25-171; blocks t_i, t_j, and the constant yaw and anchor folded into R and anchor):
//   P = R (ratio t_i + (1 - ratio) t_j) + anchor;  row k <-> satellite s = k + (k >= m), m the master:
//   e_k = (|su_s - P| - |sr_s - st|) - (|su_m - P| - |sr_m - st|) - ((pu_s - pr_s) - (pu_m - pr_m)),  w_k = |e_k| > thr ? 0.05 : 1
//   r_k = w_k e_k,  J_i row k = (-u_s^T R w_k ratio) - (-u_m^T R w_k ratio), J_j the same with (1 - ratio),  u = normalized(su - P)
//   then r = W r, J = W J when the factor has a weight matrix.  normalized() is Eigen 3.3's: d / |d| if |d|^2 > 0, else d.
// Layout: one warp per distinct pair (a, b); lane k owns row k, walks the pair's factors in list order and accumulates its row's
// contributions to the 28 pair sums (aa, bb upper-triangular over t, ab, g, cost) in registers; W is applied by broadcasting the
// raw rows with __shfl_sync in index order; one butterfly reduction over the lanes at the end.  k_pair_assemble (DdLayout) then
// sums each keyframe's pairs in incidence order into the t columns of the K x 28 layout.  No floating-point atomics.
// ---------------------------------------------------------------------------------------------------------------
constexpr int ND = GLIO_NACC_DD;
constexpr int PSR_T = 128;   // 4 pairs per block

// d = a - b and |d|^2 with the roundings pinned: equal arguments give equal bits wherever they are formed
__device__ __forceinline__ double psr_diff_sq(const double a[3], const double b[3], double d[3]) {
  d[0] = __dsub_rn(a[0], b[0]); d[1] = __dsub_rn(a[1], b[1]); d[2] = __dsub_rn(a[2], b[2]);
  return __fma_rn(d[2], d[2], __fma_rn(d[1], d[1], __dmul_rn(d[0], d[0])));
}

template <bool WANT_JAC>
__global__ void __launch_bounds__(PSR_T) k_psr_pair_sums(const DdPsrFactor* __restrict__ fl, const int* __restrict__ fstart,
                                                         const DdPsrSat* __restrict__ sats, const double* __restrict__ Wm, const DdPsrFrame fr,
                                                         int n_pairs, const double* __restrict__ poses, double* __restrict__ sums) {
  const int p = blockIdx.x * (PSR_T / 32) + (threadIdx.x >> 5);
  if (p >= n_pairs) return;                       // a warp leaves as a whole; the shuffles below use the full mask
  const int k = threadIdx.x & 31;
  double acc[ND];
#pragma unroll
  for (int e = 0; e < ND; ++e) acc[e] = 0.0;
  const int f1 = fstart[p];
  for (int f = f1, f2 = fstart[p + 1]; f < f2; ++f) {
    const DdPsrFactor F = fl[f];
    const double* ti = poses + 7 * F.i;
    const double* tj = poses + 7 * F.j;
    const double ra = F.ratio, rb = 1.0 - F.ratio;
    double loc[3], P[3];
#pragma unroll
    for (int c = 0; c < 3; ++c) loc[c] = ra * ti[c] + rb * tj[c];
#pragma unroll
    for (int c = 0; c < 3; ++c) P[c] = fr.R[3 * c] * loc[0] + fr.R[3 * c + 1] * loc[1] + fr.R[3 * c + 2] * loc[2] + fr.anchor[c];
    const int nr = F.n_sat - 1, m = F.master;
    const DdPsrSat* S = sats + F.sat_offset;
    double r = 0.0, J[6] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
    if (k < nr) {
      const DdPsrSat Sm = S[m], Ss = S[k + (k >= m ? 1 : 0)];
      double dus[3], dum[3], drs[3], drm[3];
      const double zus = psr_diff_sq(Ss.sat_user, P, dus), zum = psr_diff_sq(Sm.sat_user, P, dum);
      const double zrs = psr_diff_sq(Ss.sat_ref, F.station, drs), zrm = psr_diff_sq(Sm.sat_ref, F.station, drm);
      const double nus = sqrt(zus), num = sqrt(zum);
      const double dd_est = (nus - sqrt(zrs)) - (num - sqrt(zrm));
      const double dd_psr = (Ss.psr_user - Ss.psr_ref) - (Sm.psr_user - Sm.psr_ref);
      const double e = dd_est - dd_psr;
      const double w = fabs(e) > F.threshold ? 0.05 : 1.0;
      r = w * e;
      if (WANT_JAC) {
#pragma unroll
        for (int c = 0; c < 3; ++c) {
          if (zus > 0.0) dus[c] = dus[c] / nus;
          if (zum > 0.0) dum[c] = dum[c] / num;
        }
#pragma unroll
        for (int c = 0; c < 3; ++c) {
          const double as = -dus[0] * fr.R[c] - dus[1] * fr.R[3 + c] - dus[2] * fr.R[6 + c];   // (-u_s^T R)[c]
          const double am = -dum[0] * fr.R[c] - dum[1] * fr.R[3 + c] - dum[2] * fr.R[6 + c];   // (-u_m^T R)[c]
          J[c] = as * w * ra - am * w * ra;
          J[3 + c] = as * w * rb - am * w * rb;
        }
      }
    }
    if (F.w_offset >= 0) {                        // r = W r, J = W J: row l broadcast from lane l, in index order
      const double* Wf = Wm + F.w_offset;
      double rw = 0.0, Jw[6] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
      for (int l = 0; l < nr; ++l) {
        const double wl = k < nr ? Wf[k * nr + l] : 0.0;
        rw += wl * __shfl_sync(0xffffffffu, r, l);
        if (WANT_JAC) {
#pragma unroll
          for (int q = 0; q < 6; ++q) Jw[q] += wl * __shfl_sync(0xffffffffu, J[q], l);
        }
      }
      r = rw;
#pragma unroll
      for (int q = 0; q < 6; ++q) J[q] = Jw[q];
    }
    acc[27] += 0.5 * r * r;
    if (WANT_JAC) {
      const bool ilo = F.i < F.j;
      const double Ja[3] = {ilo ? J[0] : J[3], ilo ? J[1] : J[4], ilo ? J[2] : J[5]};
      const double Jb[3] = {ilo ? J[3] : J[0], ilo ? J[4] : J[1], ilo ? J[5] : J[2]};
      int s = 0;
#pragma unroll
      for (int a = 0; a < 3; ++a)
#pragma unroll
        for (int b = a; b < 3; ++b, ++s) { acc[s] += Ja[a] * Ja[b]; acc[6 + s] += Jb[a] * Jb[b]; }
#pragma unroll
      for (int a = 0; a < 3; ++a) {
#pragma unroll
        for (int b = 0; b < 3; ++b) acc[12 + 3 * a + b] += Ja[a] * Jb[b];
        acc[21 + a] += Ja[a] * r;
        acc[24 + a] += Jb[a] * r;
      }
    }
  }
  // butterfly over the 32 lanes: a lane and its partner add the same two values, so every lane ends with the same bits
#pragma unroll
  for (int e = WANT_JAC ? 0 : 27; e < ND; ++e)
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) acc[e] += __shfl_xor_sync(0xffffffffu, acc[e], o);
  double* Sp = sums + (size_t)p * ND;
#pragma unroll
  for (int e = WANT_JAC ? 0 : 27; e < ND; ++e)
    if (k == e) Sp[e] = acc[e];
}

// K2g: the GLIO_NACC layout per keyframe, the t rows and columns only; the 6 x 6 ab blocks per pair, zero outside t x t
struct DdLayout {
  static constexpr int NS = GLIO_NACC_DD, ND = GLIO_NACC, NO = 36, COST = 27;
  __device__ static __forceinline__ double diag(const double* s, int role, int e) {
    // 6 x 6 upper triangle -> the 3 x 3 t block: (0,0..2) = 0..2, (1,1..2) = 6..7, (2,2) = 11; g_t = 21..23; cost = 27
    const int src = e <= 2 ? e : e == 6 || e == 7 ? e - 3 : e == 11 ? 5 : -1;
    if (e < 21) return src >= 0 ? s[6 * role + src] : 0.0;    // aa | bb
    if (e < 24) return s[21 + 3 * role + (e - 21)];            // g_a | g_b
    if (e < 27) return 0.0;
    return role == 0 ? s[27] : 0.0;                            // the cost goes to a
  }
  __device__ static __forceinline__ double off(const double* s, int e) {
    const int row = e / 6, col = e - 6 * row;
    return row < 3 && col < 3 ? s[12 + 3 * row + col] : 0.0;
  }
};

void eval_dd_psr_run(const DdPsrFactor* d_f, const int* d_fstart, const DdPsrSat* d_sats, const double* d_w, const DdPsrFrame& frame,
                     int n_pairs, int K, int n_inc_kf, const int* d_kf_inc_start, const BinIncidence* d_inc, const double* d_poses,
                     bool want_jac, bool add, double* d_sums, double* d_diag, double* d_off, cudaStream_t st, LaunchCounter& lc) {
  if (n_pairs > 0) {
    const int nb = (n_pairs + PSR_T / 32 - 1) / (PSR_T / 32);
    lc.begin(want_jac ? "k_psr_pair_sums" : "k_psr_pair_sums_cost", st);
    (want_jac ? k_psr_pair_sums<true> : k_psr_pair_sums<false>)<<<nb, PSR_T, 0, st>>>(d_f, d_fstart, d_sats, d_w, frame, n_pairs,
                                                                                     d_poses, d_sums);
    lc.end(st);
  }
  lc.begin("k_psr_assemble", st);
  pair_assemble_run<DdLayout>(d_sums, K, n_pairs, n_inc_kf, d_kf_inc_start, d_inc, want_jac, add, d_diag, d_off, st);
  lc.end(st);
}

// ---------------------------------------------------------------------------------------------------------------
// K2i: the batch refinement's IMU factors (glio_batch_set_imu_factors), as ImuFactor::Evaluate writes them (ImuFactor.h:21-171,
// the residual of Preintegration::evaluate, Preintegration.h:196-235; blocks P_i, Q_i, SB_i, P_j, Q_j, SB_j), from the caller's
// pre-integration.  Q_i and Q_j are normalised first; inverse() = conj / |q|^2 and q v are Eigen's; deltaQ(theta) = (1, theta / 2):
//   dba = Ba_i - lin_ba,  dbg = Bg_i - lin_bg,  cdq = delta_q deltaQ(dq_dbg dbg),  cdv / cdp = delta_v / delta_p + dv_dba / dp_dba dba
//   + dv_dbg / dp_dbg dbg;  r_P = Q_i^-1 (-g T^2 / 2 + P_j - P_i - V_i T) - cdp,  r_R = 2 vec(normalized(cdq^-1 (Q_i^-1 Q_j))),
//   r_V = Q_i^-1 (-g T + V_j - V_i) - cdv,  r_BA = Ba_j - Ba_i,  r_BG = Bg_j - Bg_i,  r = sqrt_info r_raw,  cost = |r|^2 / 2.
// The Jacobian is ImuFactor's analytic one (not the derivative of r): its ambient 15 x 4 quaternion blocks times Ceres'
// QuaternionParameterization local Jacobian at the unnormalised parameter, [0, e_k] (x) q, then sqrt_info times every column.
// Layout: one warp per distinct pair (a, b); lane l < 30 owns tangent column l of (x_a, x_b), x = [t, delta, v, ba, bg], walks the
// pair's factors in list order and keeps row l of the pair's 30 x 30 J^T J and entry l of J^T r in registers; the other columns,
// and row a of r from lane a, come by shuffle; the lanes' cost shares are summed by one butterfly at the end.  k_pair_assemble (ImuLayout) then sums each keyframe's pairs in incidence order.  No floating-point atomics.
// ---------------------------------------------------------------------------------------------------------------
constexpr int NI = GLIO_NACC_IMU, NIK = GLIO_NACC_IMU_KF;
constexpr int IMU_T = 128;   // 4 pairs per block

__device__ __forceinline__ void qnormalize(const double q[4], double o[4]) {   // Eigen's normalize(): unchanged when |q|^2 = 0
  const double n2 = q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3];
  const double n = n2 > 0.0 ? sqrt(n2) : 1.0;
#pragma unroll
  for (int m = 0; m < 4; ++m) o[m] = n2 > 0.0 ? q[m] / n : q[m];
}
__device__ __forceinline__ void qinverse(const double q[4], double o[4]) {     // Eigen's inverse(): conj / |q|^2, 0 for q = 0
  const double n2 = q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3];
  o[0] = n2 > 0.0 ? q[0] / n2 : 0.0; o[1] = n2 > 0.0 ? -q[1] / n2 : 0.0; o[2] = n2 > 0.0 ? -q[2] / n2 : 0.0; o[3] = n2 > 0.0 ? -q[3] / n2 : 0.0;
}
// y = M x for a row-major 3 x 3 M
__device__ __forceinline__ void mat3v(const double* M, const double x[3], double y[3]) {
#pragma unroll
  for (int m = 0; m < 3; ++m) y[m] = M[3 * m] * x[0] + M[3 * m + 1] * x[1] + M[3 * m + 2] * x[2];
}
// column e of Eigen's toRotationMatrix() of q
__device__ __forceinline__ void rotmat_col(const double q[4], int e, double o[3]) {
  const double tx = 2.0 * q[1], ty = 2.0 * q[2], tz = 2.0 * q[3];
  const double twx = tx * q[0], twy = ty * q[0], twz = tz * q[0], txx = tx * q[1], txy = ty * q[1], txz = tz * q[1];
  const double tyy = ty * q[2], tyz = tz * q[2], tzz = tz * q[3];
  if (e == 0) { o[0] = 1.0 - (tyy + tzz); o[1] = txy + twz; o[2] = txz - twy; }
  else if (e == 1) { o[0] = txy - twz; o[1] = 1.0 - (txx + tzz); o[2] = tyz + twx; }
  else { o[0] = txz + twy; o[1] = tyz - twx; o[2] = 1.0 - (txx + tyy); }
}
// ImuFactor's P / V rows of the Q_i block along d:  2 (d_w (w t + u x t) + (u.t) d_u + u (t.d_u) - t (u.d_u) - w (t x d_u))
__device__ __forceinline__ void imu_qi_rows(const double q[4], const double t[3], const double d[4], double o[3]) {
  const double ut = q[1] * t[0] + q[2] * t[1] + q[3] * t[2], td = t[0] * d[1] + t[1] * d[2] + t[2] * d[3];
  const double ud = q[1] * d[1] + q[2] * d[2] + q[3] * d[3];
  const double uxt[3] = {q[2] * t[2] - q[3] * t[1], q[3] * t[0] - q[1] * t[2], q[1] * t[1] - q[2] * t[0]};
  const double txd[3] = {t[1] * d[3] - t[2] * d[2], t[2] * d[1] - t[0] * d[3], t[0] * d[2] - t[1] * d[1]};
#pragma unroll
  for (int m = 0; m < 3; ++m) o[m] = 2.0 * (d[0] * (q[0] * t[m] + uxt[m]) + ut * d[1 + m] + q[1 + m] * td - t[m] * ud - q[0] * txd[m]);
}

// JAC_KIND 0: the tangent columns above.  JAC_KIND 1 (the window marginalisation, MarginalizationFactor.cpp:3-29): the delta lanes
// take the ambient x, y, z columns of the 4-vector parameter, d = e_{1+k}, in place of [0, e_k] (x) q; every other column is the same.
template <bool WANT_JAC, int JAC_KIND>
__global__ void __launch_bounds__(IMU_T) k_imu_pair_sums(const ImuFactor* __restrict__ fl, const int* __restrict__ fstart, int n_pairs,
                                                         const double* __restrict__ poses, const double* __restrict__ sb,
                                                         double* __restrict__ sums) {
  const int p = blockIdx.x * (IMU_T / 32) + (threadIdx.x >> 5);
  if (p >= n_pairs) return;                       // a warp leaves as a whole
  const int l = threadIdx.x & 31, half = l >= 15 ? 1 : 0, comp = l - 15 * half, blk = comp / 3, e = comp - 3 * blk;
  double H[30], gl = 0.0, cost = 0.0;
#pragma unroll
  for (int m = 0; m < 30; ++m) H[m] = 0.0;
  const int f1 = fstart[p + 1];
  for (int k = fstart[p]; k < f1; ++k) {
    const ImuFactor& F = fl[k];
    const double* Pi = poses + 7 * F.i;
    const double* Pj = poses + 7 * F.j;
    const double* Si = sb + 9 * F.i;
    const double* Sj = sb + 9 * F.j;
    double qi[4], qj[4], qii[4];
    { const double a[4] = {Pi[3], Pi[4], Pi[5], Pi[6]}, b[4] = {Pj[3], Pj[4], Pj[5], Pj[6]}; qnormalize(a, qi); qnormalize(b, qj); }
    qinverse(qi, qii);
    const double T = F.sum_dt;
    double dba[3], dbg[3], th[3], ca[3], cb[3];
#pragma unroll
    for (int m = 0; m < 3; ++m) { dba[m] = Si[3 + m] - F.linearized_ba[m]; dbg[m] = Si[6 + m] - F.linearized_bg[m]; }
    mat3v(F.dq_dbg, dbg, th);
    const double dQ[4] = {1.0, th[0] / 2.0, th[1] / 2.0, th[2] / 2.0};
    double cdq[4]; qmul(F.delta_q, dQ, cdq);
    double raw[15], tmp[3], tmp1[3];
#pragma unroll
    for (int m = 0; m < 3; ++m) {
      tmp[m] = -0.5 * F.g_vec[m] * T * T + Pj[m] - Pi[m] - Si[m] * T;
      tmp1[m] = -F.g_vec[m] * T + Sj[m] - Si[m];
    }
    {
      double rp[3], rv[3];
      qrot(qii, tmp, rp); qrot(qii, tmp1, rv);
      mat3v(F.dp_dba, dba, ca); mat3v(F.dp_dbg, dbg, cb);
#pragma unroll
      for (int m = 0; m < 3; ++m) raw[m] = rp[m] - (F.delta_p[m] + ca[m] + cb[m]);
      mat3v(F.dv_dba, dba, ca); mat3v(F.dv_dbg, dbg, cb);
#pragma unroll
      for (int m = 0; m < 3; ++m) raw[6 + m] = rv[m] - (F.delta_v[m] + ca[m] + cb[m]);
      double cinv[4], qij[4], E[4], En[4];
      qinverse(cdq, cinv); qmul(qii, qj, qij); qmul(cinv, qij, E); qnormalize(E, En);
#pragma unroll
      for (int m = 0; m < 3; ++m) {
        raw[3 + m] = 2.0 * En[1 + m];
        raw[9 + m] = Sj[3 + m] - Si[3 + m];
        raw[12 + m] = Sj[6 + m] - Si[6 + m];
      }
    }
    // lane l < 15 owns row l of r = sqrt_info r_raw (the other rows come by shuffle); its cost share is summed over the lanes
    // once, at the end
    double rl = 0.0;
    if (l < 15) {
#pragma unroll
      for (int b = 0; b < 15; ++b) rl += F.sqrt_info[15 * l + b] * raw[b];
    }
    cost += 0.5 * (rl * rl);
    if (WANT_JAC) {
      double u[15];   // column l of the Jacobian before sqrt_info
#pragma unroll
      for (int m = 0; m < 15; ++m) u[m] = 0.0;
      const bool is_i = (half == 0) == (F.i < F.j);
      if (l < 30) {
        if (blk == 0 || blk == 2) {                                  // t, v: columns of +-R(Q_i^-1) (times T for v in the P rows)
          double c3[3]; rotmat_col(qii, e, c3);
          const double s = is_i ? -1.0 : 1.0;
#pragma unroll
          for (int m = 0; m < 3; ++m) {
            if (blk == 0) u[m] = s * c3[m];
            else if (is_i) { u[m] = -c3[m] * T; u[6 + m] = -c3[m]; }
            else u[6 + m] = c3[m];
          }
        } else if (blk == 1) {                                       // delta: the ambient block along [0, e_k] (x) q, or e_{1+k}
          double d[4];
          if (JAC_KIND == 1) {
            d[0] = 0.0; d[1] = e == 0 ? 1.0 : 0.0; d[2] = e == 1 ? 1.0 : 0.0; d[3] = e == 2 ? 1.0 : 0.0;
          } else {
            const double* qr = is_i ? Pi + 3 : Pj + 3;
            const double w = qr[0], x = qr[1], y = qr[2], z = qr[3];
            d[0] = e == 0 ? -x : e == 1 ? -y : -z; d[1] = e == 0 ? w : e == 1 ? z : -y;
            d[2] = e == 0 ? -z : e == 1 ? w : x; d[3] = e == 0 ? y : e == 1 ? -x : w;
          }
          double t4[4], o4[4];
          if (is_i) {
            imu_qi_rows(qi, tmp, d, u); imu_qi_rows(qi, tmp1, d, u + 6);
            double qji[4]; qinverse(qj, qji);
            qmul(d, cdq, t4); qmul(qji, t4, o4);                     // Qleft(Q_j^-1) Qright(cdq) d
#pragma unroll
            for (int m = 0; m < 3; ++m) u[3 + m] = -2.0 * o4[1 + m];
          } else {
            double cinv[4]; qinverse(cdq, cinv); qmul(cinv, qii, t4); qmul(t4, d, o4);   // Qleft(cdq^-1 Q_i^-1) d
#pragma unroll
            for (int m = 0; m < 3; ++m) u[3 + m] = 2.0 * o4[1 + m];
          }
        } else if (blk == 3) {                                       // ba
          if (is_i) {
#pragma unroll
            for (int m = 0; m < 3; ++m) { u[m] = -F.dp_dba[3 * m + e]; u[6 + m] = -F.dv_dba[3 * m + e]; }
            u[9 + e] = -1.0;
          } else {
            u[9 + e] = 1.0;
          }
        } else {                                                     // bg
          if (is_i) {
            double qji[4], t4[4], M[4]; qinverse(qj, qji); qmul(qji, qi, t4); qmul(t4, cdq, M);
            const double c3[3] = {F.dq_dbg[e], F.dq_dbg[3 + e], F.dq_dbg[6 + e]};
            // -(w I + [v]x) c:  LeftQuatMatrix's top-left 3 x 3
            u[3] = -(M[0] * c3[0] + (M[2] * c3[2] - M[3] * c3[1]));
            u[4] = -(M[0] * c3[1] + (M[3] * c3[0] - M[1] * c3[2]));
            u[5] = -(M[0] * c3[2] + (M[1] * c3[1] - M[2] * c3[0]));
#pragma unroll
            for (int m = 0; m < 3; ++m) { u[m] = -F.dp_dbg[3 * m + e]; u[6 + m] = -F.dv_dbg[3 * m + e]; }
            u[12 + e] = -1.0;
          } else {
            u[12 + e] = 1.0;
          }
        }
      }
      double c[15];
#pragma unroll
      for (int a = 0; a < 15; ++a) {
        double s = 0.0;
#pragma unroll
        for (int b = 0; b < 15; ++b) s += F.sqrt_info[15 * a + b] * u[b];
        c[a] = s;
      }
#pragma unroll
      for (int a = 0; a < 15; ++a) gl += c[a] * __shfl_sync(0xffffffffu, rl, a);
#pragma unroll
      for (int m = 0; m < 30; ++m) {
        double s = 0.0;
#pragma unroll
        for (int a = 0; a < 15; ++a) s += c[a] * __shfl_sync(0xffffffffu, c[a], m);
        H[m] += s;
      }
    }
  }
  double* S = sums + (size_t)p * NI;
  if (WANT_JAC) {
    if (l < 15) {
#pragma unroll
      for (int m = 0; m < 15; ++m) { S[15 * l + m] = H[m]; S[450 + 15 * l + m] = H[15 + m]; }
    } else if (l < 30) {
#pragma unroll
      for (int m = 0; m < 15; ++m) S[225 + 15 * (l - 15) + m] = H[15 + m];
    }
    if (l < 30) S[675 + l] = gl;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) cost += __shfl_xor_sync(0xffffffffu, cost, o);
  if (l == 0) S[705] = cost;
}

// K2i: per keyframe its 15 x 15 block, g and cost (GLIO_NACC_IMU_KF), the ab blocks per pair
struct ImuLayout {
  static constexpr int NS = NI, ND = NIK, NO = 225, COST = 240;
  __device__ static __forceinline__ double diag(const double* s, int role, int e) {
    if (e < 225) return s[225 * role + e];                     // aa | bb
    if (e < 240) return s[675 + 15 * role + (e - 225)];        // g_a | g_b
    return role == 0 ? s[705] : 0.0;                           // the cost goes to a
  }
  __device__ static __forceinline__ double off(const double* s, int e) { return s[450 + e]; }
};

// the pair sums alone: n_pairs pairs from d_fstart, JAC_KIND jac_kind with want_jac, the cost otherwise
void eval_imu_pair_sums_run(const ImuFactor* d_f, const int* d_fstart, int n_pairs, const double* d_poses, const double* d_sb, int jac_kind,
                            bool want_jac, double* d_sums, cudaStream_t st, LaunchCounter& lc) {
  if (n_pairs <= 0) return;
  const int nb = (n_pairs + IMU_T / 32 - 1) / (IMU_T / 32);
  lc.begin(want_jac ? (jac_kind == 1 ? "k_imu_pair_sums_ambient" : "k_imu_pair_sums") : "k_imu_pair_sums_cost", st);
  (want_jac ? (jac_kind == 1 ? k_imu_pair_sums<true, 1> : k_imu_pair_sums<true, 0>) : k_imu_pair_sums<false, 0>)<<<nb, IMU_T, 0, st>>>(
      d_f, d_fstart, n_pairs, d_poses, d_sb, d_sums);
  lc.end(st);
  GLIO_CUDA_TRY(cudaGetLastError());
}

void eval_imu_run(const ImuFactor* d_f, const int* d_fstart, int n_pairs, int K, int n_inc_kf, const int* d_kf_inc_start,
                  const BinIncidence* d_inc, const double* d_poses, const double* d_sb, int jac_kind, bool want_jac, double* d_sums,
                  double* d_diag, double* d_off, cudaStream_t st, LaunchCounter& lc) {
  eval_imu_pair_sums_run(d_f, d_fstart, n_pairs, d_poses, d_sb, jac_kind, want_jac, d_sums, st, lc);
  lc.begin("k_imu_assemble", st);
  pair_assemble_run<ImuLayout>(d_sums, K, n_pairs, n_inc_kf, d_kf_inc_start, d_inc, want_jac, false, d_diag, d_off, st);
  lc.end(st);
}

}  // namespace glio
