// ceres/ceres.h — glio_b200's Ceres-API shim: the subset of the Ceres 2.0.0 public API that GLIO uses
// (census: `grep -ohE "ceres::[A-Za-z_:]+" GLIO/src GLIO/include`), with the same names, signatures, ownership
// and error conventions, so Estimator.cpp / LidarOdometry.cpp / MarginalizationFactor.cpp and the factor headers
// compile against it unchanged (they additionally need Eigen, which this repository does not ship).
//
//   ceres::CostFunction / SizedCostFunction / AutoDiffCostFunction     ceres.tgz::include/ceres/{cost_function,sized_cost_function,autodiff_cost_function}.h
//   ceres::LossFunction / HuberLoss / CauchyLoss / TrivialLoss          .../loss_function.h
//   ceres::LocalParameterization / QuaternionParameterization / ...     .../local_parameterization.h
//   ceres::Problem, ceres::Solver::{Options,Summary}, ceres::Solve      .../problem.h, .../solver.h
//
// What is different underneath: ceres::Solve runs glio's trust-region / dogleg restatement (glio_b200/csrc/solver.h)
// on the normal equations, and residual blocks whose cost function can describe itself as one of GLIO's LiDAR factors
// (glio::DeviceFactorTraits<Functor>, see INTEGRATION.md) are not evaluated one virtual call at a time on the host:
// they are uploaded once to a glio_ctx and evaluated by the CUDA kernels, which return 6x6 pose blocks: K2 for the plane
// factors (LidarPlaneNormFactor, and LidarPlaneNormIncreFactor in a front-end context), K2e for LidarEdgeFactor, K2b for
// BinaryLidarPlaneNormFactor, K2p for the batch refinement's pose factors (LidarPoseFactorBatchRelativeAutoDiff,
// delta_q_factor_auto), K2g for its GNSS double-differenced pseudorange factor dd_psr_factor_20 and K2i for its IMU factor
// ImuFactor: SizedCostFunctions that describe themselves through glio::DeviceCostTraits<Cost>, looked up by the static type
// AddResidualBlock is given.  Every other cost function (marginalisation prior, the window's GNSS factors, speed-bias priors
// ...) is evaluated on the host through its own Evaluate(), exactly as Ceres would.  Without a glio_ctx attached everything
// runs on the host (used by CPU tests).
#ifndef GLIO_SHIM_CERES_CERES_H_
#define GLIO_SHIM_CERES_CERES_H_

#include <algorithm>
#include <cmath>
#include <cstddef>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <limits>
#include <map>
#include <memory>
#include <set>
#include <string>
#include <type_traits>
#include <utility>
#include <vector>

#include "../../../include/glio_b200.h"
#include "../../csrc/solver.h"
#include "jet.h"

namespace ceres { class CostFunction; }

namespace glio {
// ---- self-description of device-evaluable LiDAR factors --------------------------------------------------------
enum FactorKind { FACTOR_NONE = 0, FACTOR_PLANE_UNARY = 1, FACTOR_PLANE_BINARY = 2, FACTOR_EDGE_UNARY = 3, FACTOR_PLANE_INCRE = 4,
                  FACTOR_POSE_RELATIVE = 5, FACTOR_POSE_DELTA_Q = 6 };
struct FactorDesc {
  int kind = FACTOR_NONE;
  double cp[3] = {0, 0, 0};           // current point (scan / body frame)
  double n[3] = {0, 0, 0}, d = 0;     // unary / incre: weight*normal, weight*d  (LidarPlaneNormFactor, LidarPlaneNormIncreFactor)
  double q_lb[4] = {1, 0, 0, 0}, t_lb[3] = {0, 0, 0};
  double nc[6] = {0, 0, 0, 0, 0, 0};  // binary: local normal + centroid (BinaryLidarPlaneNormFactor)
  double score = 0;                   // unary / binary: score; edge: the weight s
  double pa[3] = {0, 0, 0}, pb[3] = {0, 0, 0};   // edge: two points of the map line (LidarEdgeFactor last_point_a / _b)
  double dq[4] = {1, 0, 0, 0}, dp[3] = {0, 0, 0};  // pose factors: the measured delta_q (w, x, y, z) and, relative kind, delta_p
};
// Specialise for the reference's functors (INTEGRATION.md shows the lines for each LiDAR functor):
//   template <> struct glio::DeviceFactorTraits<LidarPlaneNormFactor> { static bool describe(const LidarPlaneNormFactor&, FactorDesc*); };
template <class Functor> struct DeviceFactorTraits { static bool describe(const Functor&, FactorDesc*) { return false; } };

// ---- self-description of device-evaluable cost functions that are not AutoDiffCostFunctions ----------------------------
// dd_psr_factor_20 (dd_psr_factor.hpp) is a SizedCostFunction<19, 3, 3, 1, 3> with its own Evaluate: blocks t_i, t_j, yaw, anchor.
// Its description is the factor's data; the rows it evaluates are those of K2g (glio_batch_set_dd_psr_factors in glio_b200.h).
struct DdPsrDesc {
  int n_sat = 0, master = -1;         // satellites (the rows of GNSS_Raws); master: the reference's mPrn, an index into them
  double ratio = 0, threshold = 0, station[3] = {0, 0, 0};
  double sat_user[GLIO_DD_PSR_MAX_SAT][3], sat_ref[GLIO_DD_PSR_MAX_SAT][3];   // ECEF satellite positions: rover, station
  double psr_user[GLIO_DD_PSR_MAX_SAT], psr_ref[GLIO_DD_PSR_MAX_SAT];         // raw pseudoranges: rover, station
  double W[(GLIO_DD_PSR_MAX_SAT - 1) * (GLIO_DD_PSR_MAX_SAT - 1)];             // the (n_sat-1) x (n_sat-1) weight, row-major
  int w_identity = 0;                 // 1: W is exactly the identity (uploaded as w_offset = -1)
};
// Specialise for the cost function's class, next to its header (INTEGRATION.md shows the lines for dd_psr_factor_20 and
// ImuFactor).  A specialisation provides one of two kinds of description:
//   template <> struct glio::DeviceCostTraits<dd_psr_factor_20> {
//     static bool describe(const dd_psr_factor_20&, DdPsrDesc*);                 // false: the block stays on the host
//     static void frame(const double* yaw, const double* anchor, double R_ecef_local[9]);   // row-major, the factor's own R
//   };
//   template <> struct glio::DeviceCostTraits<ImuFactor> {
//     static bool describe(const ImuFactor&, glio_imu_factor*);                  // false: the block stays on the host
//   };
// The IMU description is K2i's record (glio_imu_factor in glio_b200.h) without i, j and active, which the shim sets: the
// pre-integrated deltas, the five jacobian_ blocks and sqrt_info, formed on the caller's side from the covariance as the
// factor forms it.  Problem::AddResidualBlock looks the traits up by the cost function's static type.  The default describes
// nothing.
template <class Cost> struct DeviceCostTraits {};

// what AddResidualBlock records for a cost function whose static type has a DeviceCostTraits specialisation: the calls of its
// kind, the others NULL
struct CostDescriber {
  bool (*describe_dd_psr)(const ceres::CostFunction* cost, DdPsrDesc*);
  void (*frame)(const double* yaw, const double* anchor, double R_ecef_local[9]);
  bool (*describe_imu)(const ceres::CostFunction* cost, glio_imu_factor*);
};
namespace detail {
template <class Cost, class = void> struct HasDdPsrTraits : std::false_type {};
template <class Cost>
struct HasDdPsrTraits<Cost, decltype((void)DeviceCostTraits<Cost>::describe(std::declval<const Cost&>(), (DdPsrDesc*)nullptr),
                                     (void)&DeviceCostTraits<Cost>::frame)> : std::true_type {};
template <class Cost, class = void> struct HasImuTraits : std::false_type {};
template <class Cost>
struct HasImuTraits<Cost, decltype((void)DeviceCostTraits<Cost>::describe(std::declval<const Cost&>(), (glio_imu_factor*)nullptr))>
    : std::true_type {};
template <class Cost> struct HasCostTraits : std::integral_constant<bool, HasDdPsrTraits<Cost>::value || HasImuTraits<Cost>::value> {};
template <class Cost> CostDescriber make_describer(std::true_type /* DD */) {
  return CostDescriber{[](const ceres::CostFunction* c, DdPsrDesc* out) { return DeviceCostTraits<Cost>::describe(*static_cast<const Cost*>(c), out); },
                       &DeviceCostTraits<Cost>::frame, nullptr};
}
template <class Cost> CostDescriber make_describer(std::false_type /* IMU */) {
  return CostDescriber{nullptr, nullptr, [](const ceres::CostFunction* c, glio_imu_factor* out) {
                         return DeviceCostTraits<Cost>::describe(*static_cast<const Cost*>(c), out);
                       }};
}
template <class Cost> const CostDescriber* cost_describer() {
  static const CostDescriber d = make_describer<Cost>(HasDdPsrTraits<Cost>());
  return &d;
}
}  // namespace detail
}  // namespace glio

namespace ceres {

// ---- types.h ----------------------------------------------------------------------------------------------------
enum Ownership { DO_NOT_TAKE_OWNERSHIP, TAKE_OWNERSHIP };
enum LinearSolverType { DENSE_NORMAL_CHOLESKY, DENSE_QR, SPARSE_NORMAL_CHOLESKY, DENSE_SCHUR, SPARSE_SCHUR, ITERATIVE_SCHUR, CGNR };
enum MinimizerType { LINE_SEARCH, TRUST_REGION };
enum TrustRegionStrategyType { LEVENBERG_MARQUARDT, DOGLEG };
enum DoglegType { TRADITIONAL_DOGLEG, SUBSPACE_DOGLEG };
enum TerminationType { CONVERGENCE, NO_CONVERGENCE, FAILURE, USER_SUCCESS, USER_FAILURE };
enum LoggingType { SILENT, PER_MINIMIZER_ITERATION };
enum { DYNAMIC = -1 };
typedef void* ResidualBlockId;

// ---- cost_function.h ----------------------------------------------------------------------------------------------
class CostFunction {
 public:
  CostFunction() : num_residuals_(0) {}
  CostFunction(const CostFunction&) = delete;
  void operator=(const CostFunction&) = delete;
  virtual ~CostFunction() {}
  virtual bool Evaluate(double const* const* parameters, double* residuals, double** jacobians) const = 0;
  const std::vector<int32_t>& parameter_block_sizes() const { return parameter_block_sizes_; }
  int num_residuals() const { return num_residuals_; }
  // glio extension: a LiDAR factor that the device kernels can evaluate describes itself here
  virtual bool GlioDescribe(glio::FactorDesc*) const { return false; }

 protected:
  std::vector<int32_t>* mutable_parameter_block_sizes() { return &parameter_block_sizes_; }
  void set_num_residuals(int n) { num_residuals_ = n; }

 private:
  std::vector<int32_t> parameter_block_sizes_;
  int num_residuals_;
};

template <int kNumResiduals, int... Ns>
class SizedCostFunction : public CostFunction {
 public:
  SizedCostFunction() {
    set_num_residuals(kNumResiduals);
    *mutable_parameter_block_sizes() = std::vector<int32_t>{Ns...};
  }
  virtual ~SizedCostFunction() {}
};

// ---- autodiff_cost_function.h -----------------------------------------------------------------------------------
namespace internal {
template <int... Ns> struct Sum { static constexpr int value = 0; };
template <int N, int... Ns> struct Sum<N, Ns...> { static constexpr int value = N + Sum<Ns...>::value; };
template <typename F, typename T, size_t... I>
inline bool CallFunctor(const F& f, T const* const* p, T* r, std::index_sequence<I...>) { return f(p[I]..., r); }
}  // namespace internal

template <typename CostFunctor, int kNumResiduals, int... Ns>
class AutoDiffCostFunction : public SizedCostFunction<kNumResiduals, Ns...> {
 public:
  explicit AutoDiffCostFunction(CostFunctor* functor) : functor_(functor) {
    static_assert(kNumResiduals != DYNAMIC, "use the (functor, num_residuals) constructor for DYNAMIC residuals");
  }
  AutoDiffCostFunction(CostFunctor* functor, int num_residuals) : functor_(functor) { this->set_num_residuals(num_residuals); }
  virtual ~AutoDiffCostFunction() {}
  const CostFunctor& functor() const { return *functor_; }

  bool Evaluate(double const* const* parameters, double* residuals, double** jacobians) const override {
    constexpr int kB = sizeof...(Ns);
    if (!jacobians) return internal::CallFunctor(*functor_, parameters, residuals, std::make_index_sequence<kB>());
    constexpr int kN = internal::Sum<Ns...>::value;
    typedef Jet<double, kN> JetT;
    const int sizes[kB] = {Ns...};
    std::vector<JetT> x(kN);
    const JetT* ptrs[kB];
    int off = 0;
    for (int b = 0; b < kB; ++b) {
      ptrs[b] = x.data() + off;
      for (int k = 0; k < sizes[b]; ++k) x[off + k] = JetT(parameters[b][k], off + k);
      off += sizes[b];
    }
    const int nr = this->num_residuals();
    std::vector<JetT> out(nr);
    if (!internal::CallFunctor(*functor_, ptrs, out.data(), std::make_index_sequence<kB>())) return false;
    off = 0;
    for (int b = 0; b < kB; ++b) {
      if (jacobians[b])
        for (int r = 0; r < nr; ++r)
          for (int k = 0; k < sizes[b]; ++k) jacobians[b][r * sizes[b] + k] = out[r].v[off + k];
      off += sizes[b];
    }
    for (int r = 0; r < nr; ++r) residuals[r] = out[r].a;
    return true;
  }
  bool GlioDescribe(glio::FactorDesc* d) const override { return glio::DeviceFactorTraits<CostFunctor>::describe(*functor_, d); }

 private:
  std::unique_ptr<CostFunctor> functor_;
};

// ---- loss_function.h ----------------------------------------------------------------------------------------------
class LossFunction {
 public:
  virtual ~LossFunction() {}
  virtual void Evaluate(double sq_norm, double out[3]) const = 0;
};
class TrivialLoss : public LossFunction {
 public:
  void Evaluate(double s, double rho[3]) const override { rho[0] = s; rho[1] = 1.0; rho[2] = 0.0; }
};
class HuberLoss : public LossFunction {
 public:
  explicit HuberLoss(double a) : a_(a), b_(a * a) {}
  void Evaluate(double s, double rho[3]) const override {
    if (s > b_) {
      const double r = std::sqrt(s);
      rho[0] = 2.0 * a_ * r - b_;
      rho[1] = std::max(std::numeric_limits<double>::min(), a_ / r);
      rho[2] = -rho[1] / (2.0 * s);
    } else { rho[0] = s; rho[1] = 1.0; rho[2] = 0.0; }
  }
  double a() const { return a_; }
 private:
  const double a_, b_;
};
class CauchyLoss : public LossFunction {
 public:
  explicit CauchyLoss(double a) : b_(a * a), c_(1.0 / b_) {}
  void Evaluate(double s, double rho[3]) const override {
    const double sum = 1.0 + s * c_, inv = 1.0 / sum;
    rho[0] = b_ * std::log(sum);
    rho[1] = std::max(std::numeric_limits<double>::min(), inv);
    rho[2] = -c_ * (inv * inv);
  }
 private:
  const double b_, c_;
};

// ---- local_parameterization.h -----------------------------------------------------------------------------------
class LocalParameterization {
 public:
  virtual ~LocalParameterization() {}
  virtual bool Plus(const double* x, const double* delta, double* x_plus_delta) const = 0;
  virtual bool ComputeJacobian(const double* x, double* jacobian) const = 0;   // GlobalSize x LocalSize, row-major
  virtual int GlobalSize() const = 0;
  virtual int LocalSize() const = 0;
};
class IdentityParameterization : public LocalParameterization {
 public:
  explicit IdentityParameterization(int size) : size_(size) {}
  bool Plus(const double* x, const double* d, double* o) const override { for (int i = 0; i < size_; ++i) o[i] = x[i] + d[i]; return true; }
  bool ComputeJacobian(const double*, double* J) const override { for (int i = 0; i < size_ * size_; ++i) J[i] = 0; for (int i = 0; i < size_; ++i) J[i * size_ + i] = 1; return true; }
  int GlobalSize() const override { return size_; }
  int LocalSize() const override { return size_; }
 private:
  int size_;
};
class QuaternionParameterization : public LocalParameterization {      // (w,x,y,z), q <- [cos|d|, sin|d|/|d| d] (x) q
 public:
  bool Plus(const double* x, const double* delta, double* o) const override { glio::detail::quat_plus(x, delta, o); return true; }
  bool ComputeJacobian(const double* x, double* J) const override {
    J[0] = -x[1]; J[1] = -x[2]; J[2] = -x[3];
    J[3] = x[0];  J[4] = x[3];  J[5] = -x[2];
    J[6] = -x[3]; J[7] = x[0];  J[8] = x[1];
    J[9] = x[2];  J[10] = -x[1]; J[11] = x[0];
    return true;
  }
  int GlobalSize() const override { return 4; }
  int LocalSize() const override { return 3; }
};

// ---- solver.h -----------------------------------------------------------------------------------------------------
struct IterationSummary {
  int iteration = 0;
  bool step_is_valid = false, step_is_nonmonotonic = false, step_is_successful = false;
  double cost = 0, cost_change = 0, gradient_max_norm = 0, gradient_norm = 0, step_norm = 0, relative_decrease = 0, trust_region_radius = 0;
};

class Problem;

class Solver {
 public:
  struct Options {
    MinimizerType minimizer_type = TRUST_REGION;
    TrustRegionStrategyType trust_region_strategy_type = LEVENBERG_MARQUARDT;
    DoglegType dogleg_type = TRADITIONAL_DOGLEG;
    bool use_nonmonotonic_steps = false;
    int max_consecutive_nonmonotonic_steps = 5;
    int max_num_iterations = 50;
    double max_solver_time_in_seconds = 1e9;
    int num_threads = 1;
    double initial_trust_region_radius = 1e4, max_trust_region_radius = 1e16, min_trust_region_radius = 1e-32;
    double min_relative_decrease = 1e-3, min_lm_diagonal = 1e-6, max_lm_diagonal = 1e32;
    int max_num_consecutive_invalid_steps = 5;
    double function_tolerance = 1e-6, gradient_tolerance = 1e-10, parameter_tolerance = 1e-8;
    LinearSolverType linear_solver_type = SPARSE_NORMAL_CHOLESKY;
    bool jacobi_scaling = true;
    LoggingType logging_type = PER_MINIMIZER_ITERATION;
    bool minimizer_progress_to_stdout = false;
    bool check_gradients = false;
    double gradient_check_relative_precision = 1e-8;
    bool update_state_every_iteration = false;
    bool IsValid(std::string*) const { return true; }
  };
  struct Summary {
    TerminationType termination_type = FAILURE;
    std::string message = "ceres::Solve was not called.";
    double initial_cost = -1.0, final_cost = -1.0, fixed_cost = -1.0;
    std::vector<IterationSummary> iterations;
    int num_successful_steps = -1, num_unsuccessful_steps = -1;
    double total_time_in_seconds = -1.0;
    int num_parameter_blocks = -1, num_parameters = -1, num_effective_parameters = -1, num_residual_blocks = -1, num_residuals = -1;
    int num_device_residual_blocks = 0;     // glio extension: residual blocks evaluated by the CUDA kernels
    int num_device_edge_residual_blocks = 0;   // glio extension: the LidarEdgeFactor blocks among them (K2e)
    int num_device_pose_residual_blocks = 0;   // glio extension: the relative-pose and delta_q blocks among them (K2p)
    int num_device_dd_psr_residual_blocks = 0;   // glio extension: the dd_psr_factor_20 blocks among them (K2g)
    int num_device_imu_residual_blocks = 0;   // glio extension: the ImuFactor blocks among them (K2i)
    bool IsSolutionUsable() const { return termination_type == CONVERGENCE || termination_type == NO_CONVERGENCE || termination_type == USER_SUCCESS; }
    std::string BriefReport() const {
      char b[256];
      snprintf(b, sizeof(b), "Ceres(glio shim) Solver Report: Iterations: %d, Initial cost: %e, Final cost: %e, Termination: %s",
               (int)iterations.size(), initial_cost, final_cost, termination_type == CONVERGENCE ? "CONVERGENCE" : termination_type == NO_CONVERGENCE ? "NO_CONVERGENCE" : "FAILURE");
      return b;
    }
    std::string FullReport() const { return BriefReport() + "\n" + message + "\n"; }
  };
};

// ---- problem.h ------------------------------------------------------------------------------------------------------
class Problem {
 public:
  struct Options {
    Ownership cost_function_ownership = TAKE_OWNERSHIP;
    Ownership loss_function_ownership = TAKE_OWNERSHIP;
    Ownership local_parameterization_ownership = TAKE_OWNERSHIP;
    bool enable_fast_removal = false;
    bool disable_all_safety_checks = false;
  };
  struct EvaluateOptions {
    bool apply_loss_function = true;
  };

  Problem() {}
  explicit Problem(const Options& o) : options_(o) {}
  Problem(const Problem&) = delete;
  void operator=(const Problem&) = delete;
  ~Problem() {
    std::set<const void*> done;
    for (auto& rb : residual_blocks_) {
      if (options_.cost_function_ownership == TAKE_OWNERSHIP && rb->cost && done.insert(rb->cost).second) delete rb->cost;
      if (options_.loss_function_ownership == TAKE_OWNERSHIP && rb->loss && done.insert(rb->loss).second) delete rb->loss;
    }
    if (options_.local_parameterization_ownership == TAKE_OWNERSHIP)
      for (auto& pb : blocks_) if (pb.second.param && done.insert(pb.second.param).second) delete pb.second.param;
    for (auto p : extra_params_) if (options_.local_parameterization_ownership == TAKE_OWNERSHIP && done.insert(p).second) delete p;
  }

  void AddParameterBlock(double* values, int size) { AddParameterBlock(values, size, nullptr); }
  void AddParameterBlock(double* values, int size, LocalParameterization* lp) {
    auto it = blocks_.find(values);
    if (it == blocks_.end()) {
      Block b; b.values = values; b.size = size; b.param = lp; b.order = (int)order_.size();
      blocks_[values] = b; order_.push_back(values);
    } else if (lp) {
      if (it->second.param && it->second.param != lp) extra_params_.push_back(it->second.param);
      it->second.param = lp;
    }
  }
  void SetParameterization(double* values, LocalParameterization* lp) { AddParameterBlock(values, blocks_.at(values).size, lp); }
  void SetParameterBlockConstant(double* values) { blocks_.at(values).constant = true; }
  void SetParameterBlockVariable(double* values) { blocks_.at(values).constant = false; }
  bool IsParameterBlockConstant(double* values) const { return blocks_.at(values).constant; }
  bool HasParameterBlock(const double* values) const { return blocks_.count(const_cast<double*>(values)) != 0; }

  ResidualBlockId AddResidualBlock(CostFunction* cost, LossFunction* loss, const std::vector<double*>& parameter_blocks) {
    return AddResidual(cost, loss, parameter_blocks, nullptr);
  }
  template <typename... Ts>
  ResidualBlockId AddResidualBlock(CostFunction* cost, LossFunction* loss, double* x0, Ts*... xs) {
    return AddResidual(cost, loss, std::vector<double*>{x0, xs...}, nullptr);
  }
  // glio extension: a cost function whose static type has a glio::DeviceCostTraits specialisation (dd_psr_factor_20, ImuFactor) is
  // recorded with its describer.  These overloads exist only for such types, so every other call resolves as above; a
  // described cost function passed as a plain CostFunction* is recorded without one and stays on the host.
  template <class Cost, typename std::enable_if<glio::detail::HasCostTraits<Cost>::value, int>::type = 0>
  ResidualBlockId AddResidualBlock(Cost* cost, LossFunction* loss, const std::vector<double*>& parameter_blocks) {
    return AddResidual(cost, loss, parameter_blocks, glio::detail::cost_describer<Cost>());
  }
  template <class Cost, typename... Ts, typename std::enable_if<glio::detail::HasCostTraits<Cost>::value, int>::type = 0>
  ResidualBlockId AddResidualBlock(Cost* cost, LossFunction* loss, double* x0, Ts*... xs) {
    return AddResidual(cost, loss, std::vector<double*>{x0, xs...}, glio::detail::cost_describer<Cost>());
  }

  int NumParameterBlocks() const { return (int)blocks_.size(); }
  int NumResidualBlocks() const { return (int)residual_blocks_.size(); }
  int NumParameters() const { int n = 0; for (auto& b : blocks_) n += b.second.size; return n; }
  int NumResiduals() const { int n = 0; for (auto& r : residual_blocks_) n += r->cost->num_residuals(); return n; }

  // glio extension: attach the device context that evaluates self-describing LiDAR factors (NULL: host only)
  void SetGlioContext(glio_ctx* ctx) { ctx_ = ctx; }
  glio_ctx* glio_context() const { return ctx_; }

  // cost (and optionally the gradient in tangent space, parameter blocks in insertion order) at the current state
  bool Evaluate(const EvaluateOptions&, double* cost, std::vector<double>* residuals, std::vector<double>* gradient, void* jacobian);

 private:
  friend void Solve(const Solver::Options&, Problem*, Solver::Summary*);
  struct Block { double* values = nullptr; int size = 0; LocalParameterization* param = nullptr; bool constant = false; int order = 0; };
  struct Residual { CostFunction* cost = nullptr; LossFunction* loss = nullptr; std::vector<double*> params; const glio::CostDescriber* describer = nullptr; };
  ResidualBlockId AddResidual(CostFunction* cost, LossFunction* loss, const std::vector<double*>& parameter_blocks, const glio::CostDescriber* describer) {
    const std::vector<int32_t>& sizes = cost->parameter_block_sizes();
    if (sizes.size() != parameter_blocks.size()) { fprintf(stderr, "ceres(glio shim): parameter block count mismatch\n"); return nullptr; }
    for (size_t i = 0; i < sizes.size(); ++i) AddParameterBlock(parameter_blocks[i], sizes[i], nullptr);
    std::unique_ptr<Residual> rb(new Residual());
    rb->cost = cost; rb->loss = loss; rb->params = parameter_blocks; rb->describer = describer;
    residual_blocks_.push_back(std::move(rb));
    return residual_blocks_.back().get();
  }
  Options options_;
  std::map<double*, Block> blocks_;
  std::vector<double*> order_;
  std::vector<std::unique_ptr<Residual>> residual_blocks_;
  std::vector<LocalParameterization*> extra_params_;
  glio_ctx* ctx_ = nullptr;
};

void Solve(const Solver::Options& options, Problem* problem, Solver::Summary* summary);

}  // namespace ceres

#include "shim_solve.h"

#endif  // GLIO_SHIM_CERES_CERES_H_
