// solver.cpp — see solver.h.  Host C++ only (no CUDA): the iteration driver around the device evaluation.
#include "solver.h"

#include <chrono>
#include <complex>
#include <cstdlib>

namespace glio {
namespace detail {

// All (complex) roots of a polynomial of degree <= 4, highest power first; returns the REAL PARTS of all of them,
// which is what ceres::internal::FindPolynomialRoots(poly, &real, NULL) hands to the subspace dogleg
// (polynomial.cc: companion-matrix eigenvalues; dogleg_strategy.cc:473-507 uses every real part).
bool real_roots_deg4(const double* poly5, std::vector<double>* roots) {
  roots->clear();
  int lead = 0;
  while (lead < 5 && poly5[lead] == 0.0) ++lead;
  const int deg = 4 - lead;
  if (deg < 1) return false;
  const double* p = poly5 + lead;
  if (deg == 1) { roots->push_back(-p[1] / p[0]); return true; }
  if (deg == 2) {
    const double a = p[0], b = p[1], c = p[2];
    const double D = b * b - 4 * a * c;
    if (D >= 0) {
      const double sq = std::sqrt(D);
      // numerically stable form
      if (b >= 0) { roots->push_back((-b - sq) / (2 * a)); roots->push_back((2 * c) / (-b - sq)); }
      else { roots->push_back((2 * c) / (-b + sq)); roots->push_back((-b + sq) / (2 * a)); }
    } else { roots->push_back(-b / (2 * a)); roots->push_back(-b / (2 * a)); }
    return true;
  }
  typedef std::complex<double> cd;
  std::vector<cd> c(deg + 1);
  for (int i = 0; i <= deg; ++i) c[i] = p[i] / p[0];
  // Cauchy bound for the initial radius
  double bound = 0; for (int i = 1; i <= deg; ++i) bound = std::max(bound, std::abs(c[i]));
  bound = 1.0 + bound;
  std::vector<cd> z(deg);
  for (int i = 0; i < deg; ++i) z[i] = std::polar(bound * 0.7, 0.4 + 2.0 * M_PI * i / deg);
  auto evalp = [&](cd x) { cd v = c[0]; for (int i = 1; i <= deg; ++i) v = v * x + c[i]; return v; };
  for (int it = 0; it < 500; ++it) {
    double change = 0;
    for (int i = 0; i < deg; ++i) {
      cd den = 1.0;
      for (int j = 0; j < deg; ++j) if (j != i) den *= (z[i] - z[j]);
      if (std::abs(den) == 0) den = 1e-300;
      const cd dz = evalp(z[i]) / den;
      z[i] -= dz;
      change = std::max(change, std::abs(dz) / std::max(1.0, std::abs(z[i])));
    }
    if (change < 1e-15) break;
  }
  // Newton polish
  auto evald = [&](cd x) { cd v = double(deg) * c[0]; for (int i = 1; i < deg; ++i) v = v * x + double(deg - i) * c[i]; return v; };
  for (int i = 0; i < deg; ++i)
    for (int k = 0; k < 3; ++k) { cd d = evald(z[i]); if (std::abs(d) > 0) z[i] -= evalp(z[i]) / d; }
  for (int i = 0; i < deg; ++i) {
    if (!std::isfinite(z[i].real())) return false;
    roots->push_back(z[i].real());
  }
  return true;
}

bool cholesky_solve_scalar(BandMat& A, const double* b, double* x) {
  const int n = A.n, hb = A.hb, w = hb + 1;
  double* a = A.a.data();
  // right-looking band Cholesky: after column j is scaled, the trailing rows inside the band get a rank-1 update.
  // The updates are contiguous AXPYs over row segments (SIMD without re-associating any sum).
  std::vector<double> colv((size_t)hb + 2);
  double* col = colv.data();
  for (int j = 0; j < n; ++j) {
    const double d = a[(size_t)j * w + hb];
    if (!(d > 0.0) || !std::isfinite(d)) return false;
    const double l = std::sqrt(d);
    a[(size_t)j * w + hb] = l;
    const int m = std::min(hb, n - 1 - j);
    const double linv = 1.0 / l;                          // one division per column
    for (int t = 1; t <= m; ++t) {
      double& e = a[(size_t)(j + t) * w + hb - t];      // A(j+t, j)
      e *= linv; col[t] = e;
    }
    for (int t = 1; t <= m; ++t) {
      double* __restrict ri = a + (size_t)(j + t) * w + hb - t + 1;  // A(j+t, j+1) ... A(j+t, j+t)
      const double* __restrict cu = col + 1;
      const double c = col[t];
#pragma GCC ivdep
      for (int u = 0; u < t; ++u) ri[u] -= c * cu[u];
    }
  }
  for (int i = 0; i < n; ++i) {
    const double* ri = a + (size_t)i * w + hb - i;
    double s = b[i];
    for (int k = std::max(0, i - hb); k < i; ++k) s -= ri[k] * x[k];
    x[i] = s / ri[i];
  }
  for (int i = n - 1; i >= 0; --i) {
    double s = x[i];
    const int kmax = std::min(n, i + hb + 1);
    for (int k = i + 1; k < kmax; ++k) s -= a[(size_t)k * w + hb - k + i] * x[k];
    x[i] = s / a[(size_t)i * w + hb];
  }
  for (int i = 0; i < n; ++i) if (!std::isfinite(x[i])) return false;
  return true;
}

// dispatcher: the AVX2/FMA panel version (band_chol_avx2.cpp) when the CPU has it, else the portable one
bool cholesky_solve(BandMat& A, const double* b, double* x) {
#if defined(__x86_64__)
  static const bool fast = __builtin_cpu_supports("avx2") && __builtin_cpu_supports("fma") && std::getenv("GLIO_NO_AVX2") == nullptr;
  if (fast && A.hb >= 4 && A.n >= 8) return cholesky_solve_avx2(A, b, x);
#endif
  return cholesky_solve_scalar(A, b, x);
}

}  // namespace detail

namespace {

inline double dot(const std::vector<double>& a, const std::vector<double>& b) { double s = 0; for (size_t i = 0; i < a.size(); ++i) s += a[i] * b[i]; return s; }
inline double norm(const std::vector<double>& a) { return std::sqrt(dot(a, a)); }
// y = A x for a symmetric matrix in lower-band storage
inline void symv(const BandMat& A, const double* x, double* y) {
  const int n = A.n, hb = A.hb, w = hb + 1;
#if defined(__x86_64__)
  static const bool fast = __builtin_cpu_supports("avx2") && __builtin_cpu_supports("fma") && std::getenv("GLIO_NO_AVX2") == nullptr;
  if (fast && hb >= 4) { detail::symv_avx2(A, x, y); return; }
#endif
  for (int i = 0; i < n; ++i) y[i] = 0.0;
  for (int i = 0; i < n; ++i) {
    const double* ri = A.a.data() + (size_t)i * w + hb - i;
    double s = ri[i] * x[i];
    for (int j = std::max(0, i - hb); j < i; ++j) { s += ri[j] * x[j]; y[j] += ri[j] * x[i]; }
    y[i] += s;
  }
}

// trust_region_step_evaluator.cc
struct StepEvaluator {
  int max_consec; double minimum_cost, current_cost, reference_cost, candidate_cost, acc_ref = 0, acc_cand = 0; int num_consec = 0;
  StepEvaluator(double c0, int m) : max_consec(m), minimum_cost(c0), current_cost(c0), reference_cost(c0), candidate_cost(c0) {}
  double quality(double cost, double model_change) const {
    if (cost >= std::numeric_limits<double>::max()) return std::numeric_limits<double>::lowest();
    const double rd = (current_cost - cost) / model_change;
    const double hist = (reference_cost - cost) / (acc_ref + model_change);
    return std::max(rd, hist);
  }
  void accepted(double cost, double model_change) {
    current_cost = cost; acc_cand += model_change; acc_ref += model_change;
    if (current_cost < minimum_cost) { minimum_cost = current_cost; num_consec = 0; candidate_cost = current_cost; acc_cand = 0.0; }
    else { ++num_consec; if (current_cost > candidate_cost) { candidate_cost = current_cost; acc_cand = 0.0; } }
    if (num_consec == max_consec) { reference_cost = candidate_cost; acc_ref = acc_cand; }
  }
};

// the band operations in host memory: the evaluator's BandMat, the band Cholesky and symv above
struct HostBandOps : BandOps {
  const EvalFn& fn;
  BandMat H, Hc, Hs, A;
  explicit HostBandOps(const EvalFn& f) : fn(f) {}
  bool eval(const double* x, bool want_jac, double* cost, int slot, double* g) override {
    return fn(x, want_jac, cost, want_jac ? (slot ? &Hc : &H) : nullptr, g);
  }
  bool shape_ok(int n) const override { return H.n == n; }
  void diag(double* d) override { for (int i = 0; i < H.n; ++i) d[i] = H.at(i, i); }
  void scale(const double* scale, double* hs_diag) override {
    const int n = H.n, hb = H.hb, w = hb + 1;
    Hs.n = H.n; Hs.hb = H.hb; Hs.a.resize(H.a.size());
    for (int i = 0; i < n; ++i) {
      const double si = scale[i];
      for (int j = std::max(0, i - hb); j <= i; ++j) Hs.a[(size_t)i * w + (j - i + hb)] = H.a[(size_t)i * w + (j - i + hb)] * si * scale[j];
      hs_diag[i] = Hs.at(i, i);
    }
  }
  bool shifted_solve(const double* v, const double* rhs, double* y) override {
    A = Hs;
    for (int i = 0; i < A.n; ++i) A.at(i, i) += v[i] * v[i];
    return detail::cholesky_solve(A, rhs, y);
  }
  void symv(const double* x, double* y) override { glio::symv(Hs, x, y); }
  void swap() override { std::swap(H, Hc); }
};

}  // namespace

void TrustRegionDogleg::solve(double* x_io, const EvalFn& eval_user, SolverSummary* sum) {
  HostBandOps ops(eval_user);
  solve(x_io, ops, sum);
}

void TrustRegionDogleg::solve(double* x_io, BandOps& ops, SolverSummary* sum) {
  const int n = n_, na = n_amb_;
  SolverSummary& S = *sum;
  S = SolverSummary();
  typedef std::chrono::steady_clock clk;
  const auto t_begin = clk::now();
  auto eval = [&](const double* xx, bool wj, double* cst, int slot, double* gg) -> bool {
    const auto t0 = clk::now();
    const bool ok = ops.eval(xx, wj, cst, slot, gg);
    S.eval_seconds += std::chrono::duration<double>(clk::now() - t0).count();
    return ok;
  };
  struct Fin { SolverSummary& s; clk::time_point t; ~Fin() { s.total_seconds = std::chrono::duration<double>(clk::now() - t).count(); } } fin{S, t_begin};
  std::vector<double> x(x_io, x_io + na), cand(na), proj(na);
  std::vector<double> g(n), gs(n), gc(n), hs_diag(n), hdiag(n), shift(n);
  std::vector<double> scale(n, 1.0), diag(n), grad_d(n), gn(n), step(n), delta(n), tmp(n), tmp2(n), y(n), negg(n);
  double x_cost = 0, cand_cost = 0, minimum_cost = std::numeric_limits<double>::max(), model_cost_change = 0;
  double x_norm = -1;  // trust_region_minimizer.cc:175 "Invalid value"
  double radius = opt_.initial_trust_region_radius, mu = 1e-8, alpha = 0, dogleg_step_norm = 0;
  const double min_mu = 1e-8, max_mu = 1.0, mu_inc = 10.0;
  bool reuse = false;
  int num_consecutive_invalid = 0;
  // subspace model
  std::vector<double> basis0(n), basis1(n);
  double sub_B[4] = {0, 0, 0, 0}, sub_g[2] = {0, 0};
  bool sub_1d = false;

  auto apply_scaling = [&]() {
    ops.scale(scale.data(), hs_diag.data());
    for (int i = 0; i < n; ++i) gs[i] = g[i] * scale[i];
  };
  auto gradient_norms = [&](IterationRecord& it) {
    for (int i = 0; i < n; ++i) negg[i] = -g[i];
    plus(x.data(), negg.data(), proj.data());
    double mx = 0, s2 = 0;
    for (int i = 0; i < na; ++i) { const double d = x[i] - proj[i]; mx = std::max(mx, std::fabs(d)); s2 += d * d; }
    it.gradient_max_norm = mx; it.gradient_norm = std::sqrt(s2);
  };

  // ---- dogleg pieces (dogleg_strategy.cc) ----
  auto traditional = [&]() {
    const double gnorm = norm(grad_d), gnn = norm(gn);
    if (gnn <= radius) { step = gn; dogleg_step_norm = gnn; for (int i = 0; i < n; ++i) step[i] /= diag[i]; return; }
    if (gnorm * alpha >= radius) {
      for (int i = 0; i < n; ++i) step[i] = -(radius / gnorm) * grad_d[i];
      dogleg_step_norm = radius; for (int i = 0; i < n; ++i) step[i] /= diag[i]; return;
    }
    const double b_dot_a = -alpha * dot(grad_d, gn);
    const double a_sq = std::pow(alpha * gnorm, 2.0);
    const double bma_sq = a_sq - 2 * b_dot_a + std::pow(gnn, 2);
    const double c = b_dot_a - a_sq;
    const double d = std::sqrt(c * c + bma_sq * (std::pow(radius, 2.0) - a_sq));
    const double beta = (c <= 0) ? (d - c) / bma_sq : (radius * radius - a_sq) / (d + c);
    for (int i = 0; i < n; ++i) step[i] = (-alpha * (1.0 - beta)) * grad_d[i] + beta * gn[i];
    dogleg_step_norm = norm(step);
    for (int i = 0; i < n; ++i) step[i] /= diag[i];
  };
  auto sub_eval = [&](const double v[2]) { return 0.5 * (v[0] * (sub_B[0] * v[0] + sub_B[1] * v[1]) + v[1] * (sub_B[2] * v[0] + sub_B[3] * v[1])) + sub_g[0] * v[0] + sub_g[1] * v[1]; };
  auto subspace = [&]() {
    const double gnn = norm(gn);
    if (gnn <= radius) { step = gn; dogleg_step_norm = gnn; for (int i = 0; i < n; ++i) step[i] /= diag[i]; return; }
    if (sub_1d) {
      const double gnorm = norm(grad_d);
      for (int i = 0; i < n; ++i) step[i] = -(radius / gnorm) * grad_d[i];
      dogleg_step_norm = radius; for (int i = 0; i < n; ++i) step[i] /= diag[i]; return;
    }
    // polynomial of the boundary-constrained problem (dogleg_strategy.cc:366-385)
    const double detB = sub_B[0] * sub_B[3] - sub_B[1] * sub_B[2], trB = sub_B[0] + sub_B[3], r2 = radius * radius;
    const double Badj[4] = {sub_B[3], -sub_B[1], -sub_B[2], sub_B[0]};
    const double bg[2] = {Badj[0] * sub_g[0] + Badj[1] * sub_g[1], Badj[2] * sub_g[0] + Badj[3] * sub_g[1]};
    double poly[5];
    poly[0] = r2; poly[1] = 2.0 * r2 * trB;
    poly[2] = r2 * (trB * trB + 2.0 * detB) - (sub_g[0] * sub_g[0] + sub_g[1] * sub_g[1]);
    poly[3] = -2.0 * ((sub_g[0] * bg[0] + sub_g[1] * bg[1]) - r2 * detB * trB);
    poly[4] = r2 * detB * detB - (bg[0] * bg[0] + bg[1] * bg[1]);
    std::vector<double> roots;
    double minimum[2] = {0, 0}; bool found = false;
    if (detail::real_roots_deg4(poly, &roots)) {
      double best = std::numeric_limits<double>::max();
      for (double yr : roots) {
        // x = -(B + y I)^-1 g  (2x2 solve with partial pivoting)
        double a = sub_B[0] + yr, b = sub_B[1], c2 = sub_B[2], d2 = sub_B[3] + yr, r0 = sub_g[0], r1 = sub_g[1];
        if (std::fabs(c2) > std::fabs(a)) { std::swap(a, c2); std::swap(b, d2); std::swap(r0, r1); }
        if (a == 0) continue;
        const double f = c2 / a; const double d3 = d2 - f * b, r3 = r1 - f * r0;
        if (d3 == 0) continue;
        const double x1 = r3 / d3, x0 = (r0 - b * x1) / a;
        const double xi[2] = {-x0, -x1};
        const double xn = std::sqrt(xi[0] * xi[0] + xi[1] * xi[1]);
        if (xn > 0 && std::isfinite(xn)) {
          const double v[2] = {radius / xn * xi[0], radius / xn * xi[1]};
          const double fi = sub_eval(v);
          found = true;
          if (fi < best) { best = fi; minimum[0] = xi[0]; minimum[1] = xi[1]; }
        }
      }
    }
    if (!found) { traditional(); return; }
    const double gm[2] = {sub_B[0] * minimum[0] + sub_B[1] * minimum[1] + sub_g[0], sub_B[2] * minimum[0] + sub_B[3] * minimum[1] + sub_g[1]};
    const double mn = std::sqrt(minimum[0] * minimum[0] + minimum[1] * minimum[1]), gmn = std::sqrt(gm[0] * gm[0] + gm[1] * gm[1]);
    const double cosang = -(minimum[0] * gm[0] + minimum[1] * gm[1]) / (mn * gmn);
    if (cosang < 0.99) { traditional(); return; }
    for (int i = 0; i < n; ++i) step[i] = basis0[i] * minimum[0] + basis1[i] * minimum[1];
    dogleg_step_norm = radius;
    for (int i = 0; i < n; ++i) step[i] /= diag[i];
  };
  auto subspace_model = [&]() -> bool {
    // orthonormal basis of span{grad_d, gn} (column-pivoted: larger column first)
    const double n0 = norm(grad_d), n1 = norm(gn);
    const std::vector<double>& first = (n0 >= n1) ? grad_d : gn;
    const std::vector<double>& second = (n0 >= n1) ? gn : grad_d;
    const double nf = std::max(n0, n1);
    if (!(nf > 0)) return false;  // rank 0
    for (int i = 0; i < n; ++i) basis0[i] = first[i] / nf;
    const double pr = dot(basis0, second);
    for (int i = 0; i < n; ++i) basis1[i] = second[i] - pr * basis0[i];
    const double pr2 = dot(basis0, basis1);  // re-orthogonalise once
    for (int i = 0; i < n; ++i) basis1[i] -= pr2 * basis0[i];
    const double ns = norm(basis1);
    if (ns <= nf * 2.0 * std::numeric_limits<double>::epsilon() * 2.0) { sub_1d = true; return true; }
    sub_1d = false;
    for (int i = 0; i < n; ++i) basis1[i] /= ns;
    sub_g[0] = dot(basis0, grad_d); sub_g[1] = dot(basis1, grad_d);
    for (int i = 0; i < n; ++i) { tmp[i] = basis0[i] / diag[i]; tmp2[i] = basis1[i] / diag[i]; }
    std::vector<double> h0(n), h1(n);
    ops.symv(tmp.data(), h0.data()); ops.symv(tmp2.data(), h1.data());
    sub_B[0] = dot(tmp, h0); sub_B[1] = dot(tmp, h1); sub_B[2] = sub_B[1]; sub_B[3] = dot(tmp2, h1);
    return true;
  };
  // ---- Levenberg-Marquardt (levenberg_marquardt_strategy.cc:69-160).  `diag` holds the CLAMPED SQUARED column norms here
  // (Ceres' diagonal_), `reuse` is reuse_diagonal_; the linear solve is (Hs + diag/radius) y = gs, step = -y: the normal
  // equations of the regularised least-squares problem Ceres hands to its linear solver (DENSE_QR in the front end,
  // dense_qr_solver.cc:120-153 - same minimiser, different rounding).
  const bool lm = opt_.trust_region_strategy == 1;
  double lm_decrease = 2.0;
  auto lm_compute_step = [&]() -> int {
    if (!reuse) for (int i = 0; i < n; ++i) diag[i] = std::min(std::max(hs_diag[i], opt_.min_lm_diagonal), opt_.max_lm_diagonal);
    reuse = true;
    for (int i = 0; i < n; ++i) shift[i] = std::sqrt(diag[i] / radius);
    S.num_linear_solves++;
    const auto tl0 = clk::now();
    const bool ok = ops.shifted_solve(shift.data(), gs.data(), y.data());
    S.linear_solver_seconds += std::chrono::duration<double>(clk::now() - tl0).count();
    if (!ok) return 1;
    for (int i = 0; i < n; ++i) step[i] = -y[i];
    return 0;
  };
  // returns: 0 ok, 1 linear solver failure
  auto compute_step = [&]() -> int {
    if (lm) return lm_compute_step();
    if (reuse) { if (opt_.dogleg_type == 0) traditional(); else subspace(); return 0; }
    reuse = true;
    for (int i = 0; i < n; ++i) diag[i] = std::sqrt(std::min(std::max(hs_diag[i], opt_.min_lm_diagonal), opt_.max_lm_diagonal));
    for (int i = 0; i < n; ++i) grad_d[i] = gs[i] / diag[i];
    for (int i = 0; i < n; ++i) tmp[i] = grad_d[i] / diag[i];
    ops.symv(tmp.data(), tmp2.data());
    alpha = dot(grad_d, grad_d) / dot(tmp, tmp2);
    bool ok = false;
    while (mu < max_mu) {
      const double sm = std::sqrt(mu);
      for (int i = 0; i < n; ++i) shift[i] = diag[i] * sm;
      S.num_linear_solves++;
      const auto tl0 = clk::now();
      const bool chol_ok = ops.shifted_solve(shift.data(), gs.data(), y.data());
      S.linear_solver_seconds += std::chrono::duration<double>(clk::now() - tl0).count();
      if (chol_ok) { ok = true; break; }
      mu *= mu_inc;
    }
    if (!ok) return 1;
    for (int i = 0; i < n; ++i) gn[i] = -diag[i] * y[i];
    if (opt_.dogleg_type == 0) traditional();
    else { if (!subspace_model()) return 1; subspace(); }
    return 0;
  };

  // ---- iteration zero (trust_region_minimizer.cc:181-263) ----
  IterationRecord it{};
  it.iteration = 0;
  S.num_evaluations++; S.num_jacobian_evaluations++;
  if (!eval(x.data(), true, &x_cost, 0, g.data()) || !ops.shape_ok(n)) {
    S.termination = TERM_FAILURE; S.message = "Residual and Jacobian evaluation failed."; return;
  }
  S.initial_cost = x_cost; S.final_cost = x_cost;
  if (opt_.jacobi_scaling) { ops.diag(hdiag.data()); for (int i = 0; i < n; ++i) scale[i] = 1.0 / (1.0 + std::sqrt(hdiag[i])); }
  apply_scaling();
  it.cost = x_cost; gradient_norms(it);
  it.step_is_valid = 1; it.step_is_successful = 1;
  StepEvaluator ev(x_cost, opt_.use_nonmonotonic_steps ? opt_.max_consecutive_nonmonotonic_steps : 0);

  auto finalize_and_continue = [&]() -> bool {
    if (it.step_is_successful) {
      ++S.num_successful_steps;
      if (x_cost < minimum_cost) { minimum_cost = x_cost; std::memcpy(x_io, x.data(), sizeof(double) * na); S.final_cost = x_cost; }
    } else ++S.num_unsuccessful_steps;
    it.trust_region_radius = radius; it.mu = mu;
    S.iterations.push_back(it);
    // trust_region_minimizer.cc:327-333, :605-619 (MaxSolverTimeReached, checked before the iteration limit): wall clock since the start of the solve
    if (std::chrono::duration<double>(clk::now() - t_begin).count() >= opt_.max_solver_time_in_seconds) { S.termination = TERM_NO_CONVERGENCE; S.message = "Maximum solver time reached."; return false; }
    if (it.iteration >= opt_.max_num_iterations) { S.termination = TERM_NO_CONVERGENCE; S.message = "Maximum number of iterations reached."; return false; }
    if (it.step_is_successful && it.gradient_max_norm <= opt_.gradient_tolerance) { S.termination = TERM_CONVERGENCE; S.message = "Gradient tolerance reached."; return false; }
    if (radius <= opt_.min_trust_region_radius) { S.termination = TERM_CONVERGENCE; S.message = "Minimum trust region radius reached."; return false; }
    return true;
  };

  while (finalize_and_continue()) {
    const IterationRecord prev = it;
    it = IterationRecord{};
    it.iteration = prev.iteration + 1;
    // ComputeTrustRegionStep (:364-430)
    const int rc = compute_step();
    bool valid = false;
    if (rc == 0) {
      ops.symv(step.data(), tmp.data());
      model_cost_change = -(dot(step, gs) + 0.5 * dot(step, tmp));
      valid = model_cost_change > 0.0;
      if (valid) { for (int i = 0; i < n; ++i) delta[i] = step[i] * scale[i]; num_consecutive_invalid = 0; }
    }
    it.step_is_valid = valid ? 1 : 0;
    if (!valid) {   // HandleInvalidStep (:438-458)
      if (++num_consecutive_invalid >= opt_.max_num_consecutive_invalid_steps) {
        S.termination = TERM_FAILURE; S.message = "Number of consecutive invalid steps more than max_num_consecutive_invalid_steps"; return;
      }
      if (lm) { radius /= lm_decrease; lm_decrease *= 2.0; reuse = true; }   // LevenbergMarquardtStrategy::StepIsInvalid = StepRejected(0)
      else { mu *= mu_inc; reuse = false; }                                   // DoglegStrategy::StepIsInvalid
      it.cost = x_cost; it.cost_change = 0; it.gradient_max_norm = prev.gradient_max_norm; it.gradient_norm = prev.gradient_norm;
      it.step_norm = 0; it.relative_decrease = 0; it.step_is_successful = 0;
      continue;
    }
    S.steps.insert(S.steps.end(), delta.begin(), delta.end());
    // ComputeCandidatePointAndEvaluateCost (:727-743)
    plus(x.data(), delta.data(), cand.data());
    const bool fused = opt_.fuse_candidate_jacobian;
    S.num_evaluations++; if (fused) S.num_jacobian_evaluations++;
    if (!eval(cand.data(), fused, &cand_cost, 1, fused ? gc.data() : nullptr))
      cand_cost = std::numeric_limits<double>::max();
    // ParameterToleranceReached (:676-693)
    { double s2 = 0; for (int i = 0; i < na; ++i) { const double d = x[i] - cand[i]; s2 += d * d; } it.step_norm = std::sqrt(s2); }
    if (it.step_norm <= opt_.parameter_tolerance * (x_norm + opt_.parameter_tolerance)) {
      S.termination = TERM_CONVERGENCE; S.message = "Parameter tolerance reached."; return;
    }
    // FunctionToleranceReached (:695-713)
    it.cost_change = x_cost - cand_cost;
    if (std::fabs(it.cost_change) <= opt_.function_tolerance * x_cost) {
      S.termination = TERM_CONVERGENCE; S.message = "Function tolerance reached."; return;
    }
    // IsStepSuccessful (:745-755)
    it.relative_decrease = ev.quality(cand_cost, model_cost_change);
    if (it.relative_decrease > opt_.min_relative_decrease) {
      // HandleSuccessfulStep (:757-771)
      x = cand;
      { double s2 = 0; for (int i = 0; i < na; ++i) s2 += x[i] * x[i]; x_norm = std::sqrt(s2); }
      if (fused) { ops.swap(); g.swap(gc); x_cost = cand_cost; }
      else {
        S.num_evaluations++; S.num_jacobian_evaluations++;
        if (!eval(x.data(), true, &x_cost, 0, g.data())) { S.termination = TERM_FAILURE; S.message = "Residual and Jacobian evaluation failed."; return; }
      }
      apply_scaling();
      it.cost = x_cost; gradient_norms(it);
      it.step_is_successful = 1;
      if (lm) {
        // LevenbergMarquardtStrategy::StepAccepted (levenberg_marquardt_strategy.cc:143-150)
        radius = radius / std::max(1.0 / 3.0, 1.0 - std::pow(2.0 * it.relative_decrease - 1.0, 3));
        radius = std::min(opt_.max_trust_region_radius, radius);
        lm_decrease = 2.0;
      } else {
        // DoglegStrategy::StepAccepted (:616-632)
        if (it.relative_decrease < 0.25) radius *= 0.5;
        if (it.relative_decrease > 0.75) radius = std::max(radius, 3.0 * dogleg_step_norm);
        mu = std::max(min_mu, 2.0 * mu / mu_inc);
      }
      reuse = false;
      ev.accepted(cand_cost, model_cost_change);
    } else {
      // HandleUnsuccessfulStep (:773-778) + DoglegStrategy::StepRejected
      it.step_is_successful = 0;
      if (lm) { radius /= lm_decrease; lm_decrease *= 2.0; }   // LevenbergMarquardtStrategy::StepRejected (:152-156)
      else radius *= 0.5;
      reuse = true;
      it.cost = cand_cost; it.gradient_max_norm = prev.gradient_max_norm; it.gradient_norm = prev.gradient_norm;
    }
  }
}

}  // namespace glio
