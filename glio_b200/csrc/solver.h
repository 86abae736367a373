// solver.h — host-side trust-region minimizer (dogleg and Levenberg-Marquardt strategies) over normal equations, with
// Ceres 2.0.0 semantics.
//
// The LiDAR residual blocks are evaluated on the device into 6x6 pose blocks; everything else the reference
// adds to the same ceres::Problem (IMU, marginalisation prior, GNSS — host C++ CostFunctions by north_star)
// arrives through a callback that accumulates into the same dense J^T J / J^T r.  This file restates, on the
// normal equations, what ceres::Solve does for the options the reference sets (Estimator.cpp:2424-2433,
// 3275-3284): TrustRegionMinimizer (ceres.tgz::internal/ceres/trust_region_minimizer.cc) with Jacobi scaling
// (:231-263), DoglegStrategy (dogleg_strategy.cc:79-340,517-697; traditional and subspace), LevenbergMarquardtStrategy
// (levenberg_marquardt_strategy.cc:69-160: D = sqrt(clamp(diag(J^T J)) / radius), radius / max(1/3, 1 - (2 rho - 1)^3) on
// acceptance, radius / decrease_factor with the factor doubling on rejection),
// normal-equation Cholesky (sparse_normal_cholesky_solver.cc:59-113), TrustRegionStepEvaluator
// (trust_region_step_evaluator.cc) and QuaternionParameterization::Plus (local_parameterization.cc:163-182).
// Quantities Ceres computes from the Jacobian itself (|J v|^2, (J s).(r + J s/2)) are computed from H = J^T J,
// g = J^T r: identical in exact arithmetic, equal to rounding in floating point.
#pragma once
#include <algorithm>
#include <cmath>
#include <cstring>
#include <functional>
#include <limits>
#include <string>
#include <vector>

namespace glio {

struct ParamBlock {
  int amb_off, amb_size;   // offset/size in the ambient state vector
  int tan_off, tan_size;   // offset/size in the tangent vector
  bool quaternion;         // amb 4 (w,x,y,z) / tan 3, Ceres QuaternionParameterization
  // optional custom LocalParameterization::Plus(x, delta, x_plus_delta) (Ceres shim); empty -> the two built-ins
  std::function<void(const double*, const double*, double*)> plus_fn;
};

struct SolverOptions {
  int max_num_iterations = 15;
  double max_solver_time_in_seconds = 1e9;   // Solver::Options::max_solver_time_in_seconds (LidarOdometry.cpp:527 sets 0.015)
  int trust_region_strategy = 0;   // 0 DOGLEG (what Estimator.cpp:2427 / :3278 select), 1 LEVENBERG_MARQUARDT (Ceres' default, used by
                                   // the front end's scan matcher, LidarOdometry.cpp:521-530)
  int dogleg_type = 0;  // 0 TRADITIONAL_DOGLEG, 1 SUBSPACE_DOGLEG
  bool use_nonmonotonic_steps = false;
  int max_consecutive_nonmonotonic_steps = 5;
  double initial_trust_region_radius = 1e4;
  double max_trust_region_radius = 1e16;
  double min_trust_region_radius = 1e-32;
  double min_relative_decrease = 1e-3;
  double min_lm_diagonal = 1e-6;
  double max_lm_diagonal = 1e32;
  int max_num_consecutive_invalid_steps = 5;
  double function_tolerance = 1e-6;
  double gradient_tolerance = 1e-10;
  double parameter_tolerance = 1e-8;
  bool jacobi_scaling = true;
  bool fuse_candidate_jacobian = true;  // evaluate J together with the candidate cost, reuse on acceptance
};

struct IterationRecord {
  int iteration;
  double cost, cost_change, gradient_max_norm, gradient_norm, step_norm, relative_decrease, trust_region_radius, mu;
  int step_is_valid, step_is_successful;
};

enum Termination { TERM_CONVERGENCE = 0, TERM_NO_CONVERGENCE = 1, TERM_FAILURE = 2 };

struct SolverSummary {
  int termination = TERM_NO_CONVERGENCE;
  std::string message;
  double initial_cost = 0, final_cost = 0;
  int num_successful_steps = 0, num_unsuccessful_steps = 0;
  std::vector<IterationRecord> iterations;
  std::vector<double> steps;   // tangent delta of every iteration that produced a valid step (n each), in order
  int num_evaluations = 0, num_jacobian_evaluations = 0, num_linear_solves = 0;
  double eval_seconds = 0, linear_solver_seconds = 0, total_seconds = 0;   // wall-clock split (like Ceres' Summary timers)
};

// Symmetric matrix in lower-band storage: entry (i,j), i-hb <= j <= i, lives at a[i*(hb+1) + (j-i+hb)].
// hb = n-1 is a dense lower triangle.  The block structure of the problems here is fixed, so the band is too:
// window = block tridiagonal (prior + IMU chain + unary LiDAR), batch = (2*search_range+1) block band.
struct BandMat {
  int n = 0, hb = 0;
  std::vector<double> a;
  void reset(int n_, int hb_) { n = n_; hb = std::min(hb_, std::max(n_ - 1, 0)); a.assign((size_t)n * (hb + 1), 0.0); }
  inline double& at(int i, int j) { return a[(size_t)i * (hb + 1) + (j - i + hb)]; }          // requires i-hb <= j <= i
  inline double at(int i, int j) const { return a[(size_t)i * (hb + 1) + (j - i + hb)]; }
  inline double sym(int i, int j) const { return i >= j ? (i - j <= hb ? at(i, j) : 0.0) : (j - i <= hb ? at(j, i) : 0.0); }
  inline void add_sym(int i, int j, double v) { if (i >= j) at(i, j) += v; else at(j, i) += v; }   // one triangle only
};

// evaluate(x_ambient, want_jac, &cost, H, g) -> ok.  When want_jac the evaluator calls H->reset(n, hb) itself (the band
// it needs; it must be the same on every call) and fills the lower band + g (n, overwritten).
using EvalFn = std::function<bool(const double*, bool, double*, BandMat*, double*)>;

namespace detail {

inline void quat_plus(const double* x, const double* d, double* o) {
  const double nd = std::sqrt(d[0] * d[0] + d[1] * d[1] + d[2] * d[2]);
  if (nd > 0.0) {
    const double s = std::sin(nd) / nd;
    const double z0 = std::cos(nd), z1 = s * d[0], z2 = s * d[1], z3 = s * d[2];
    // ceres::QuaternionProduct(z, x)
    o[0] = z0 * x[0] - z1 * x[1] - z2 * x[2] - z3 * x[3];
    o[1] = z0 * x[1] + z1 * x[0] + z2 * x[3] - z3 * x[2];
    o[2] = z0 * x[2] - z1 * x[3] + z2 * x[0] + z3 * x[1];
    o[3] = z0 * x[3] + z1 * x[2] - z2 * x[1] + z3 * x[0];
  } else {
    o[0] = x[0]; o[1] = x[1]; o[2] = x[2]; o[3] = x[3];
  }
}

// In-place band Cholesky A = L L^T (lower band storage) and solve L L^T x = b (solver.cpp, right-looking).  Returns false if a pivot is not positive / finite (Ceres: LINEAR_SOLVER_FAILURE -> mu escalation).
bool cholesky_solve(BandMat& A, const double* b, double* x);
bool cholesky_solve_scalar(BandMat& A, const double* b, double* x);   // portable path
#if defined(__x86_64__)
bool cholesky_solve_avx2(BandMat& A, const double* b, double* x);     // band_chol_avx2.cpp; call only when the CPU has AVX2 + FMA
void symv_avx2(const BandMat& A, const double* x, double* y);          // band_chol_avx2.cpp; y = A x (differs from the scalar loop by rounding only)
#endif

// real roots of a polynomial of degree <= 4 (highest power first), for the subspace dogleg
// (dogleg_strategy.cc:421-446 uses FindPolynomialRoots; here: Durand-Kerner + Newton polish in long double).
bool real_roots_deg4(const double* poly5, std::vector<double>* roots);

}  // namespace detail

// The band operations of the minimizer, behind one seam so the same trust-region control flow runs with its band matrices in host
// memory (HostBandOps, below) or on the device (glio_batch_solve with glio_batch_use_device_solver).  Bands: H (slot 0) and the
// candidate's Hc (slot 1) from the evaluator, the scaled Hs = S H S, and the shifted A = Hs + diag(v*v) that is factored.  Only
// n-vectors cross the seam.
struct BandOps {
  virtual ~BandOps() = default;
  // evaluate at x; with want_jac fill band `slot` and g (n, overwritten).  false: evaluation failed
  virtual bool eval(const double* x, bool want_jac, double* cost, int slot, double* g) = 0;
  virtual bool shape_ok(int n) const = 0;                  // after the first Jacobian evaluation: the band has n rows
  virtual void diag(double* d) = 0;                        // d = diag(H)
  virtual void scale(const double* s, double* hs_diag) = 0;  // Hs = S H S, hs_diag = diag(Hs)
  virtual bool shifted_solve(const double* v, const double* rhs, double* y) = 0;   // A = Hs + diag(v*v); A y = rhs; false: not SPD
  virtual void symv(const double* x, double* y) = 0;       // y = Hs x
  virtual void swap() = 0;                                 // H <-> Hc (an accepted fused candidate)
};

class TrustRegionDogleg {
 public:
  TrustRegionDogleg(const std::vector<ParamBlock>& blocks, const SolverOptions& opt) : blocks_(blocks), opt_(opt) {
    n_amb_ = 0; n_ = 0;
    for (auto& b : blocks_) { n_amb_ = std::max(n_amb_, b.amb_off + b.amb_size); n_ = std::max(n_, b.tan_off + b.tan_size); }
  }
  int num_tangent() const { return n_; }
  int num_ambient() const { return n_amb_; }

  void plus(const double* x, const double* delta, double* out) const {
    for (auto& b : blocks_) {
      if (b.plus_fn) { b.plus_fn(x + b.amb_off, delta + b.tan_off, out + b.amb_off); continue; }
      if (b.quaternion) detail::quat_plus(x + b.amb_off, delta + b.tan_off, out + b.amb_off);
      else for (int k = 0; k < b.amb_size; ++k) out[b.amb_off + k] = x[b.amb_off + k] + delta[b.tan_off + k];
    }
  }

  // x: ambient state, in/out (on return: the lowest-cost accepted point, like Ceres' `parameters`)
  void solve(double* x_inout, const EvalFn& eval, SolverSummary* sum);
  // the same minimizer over any band implementation
  void solve(double* x_inout, BandOps& ops, SolverSummary* sum);

 private:
  std::vector<ParamBlock> blocks_;
  SolverOptions opt_;
  int n_amb_ = 0, n_ = 0;
};

}  // namespace glio
