// shim_driver.h — what the shim route drivers (shim_routes_test, shim_pose_routes_test, shim_dd_psr_routes_test) share: reading
// the problem file, the device context, kernel launch counts and the lines every solve prints.  Problem builders, mode flags and
// file formats stay in each driver.
#ifndef GLIO_TESTS_SHIM_DRIVER_H_
#define GLIO_TESTS_SHIM_DRIVER_H_

#include <cerrno>
#include <cstdio>
#include <cstdlib>
#include <initializer_list>
#include <vector>

#include "ceres/ceres.h"

template <class T> static void rd(FILE* f, T* p, size_t n) {
  if (fread(p, sizeof(T), n, f) != n) { fprintf(stderr, "%s: truncated problem file\n", program_invocation_short_name); exit(2); }
}

// a context on device 0; the profiler counts launches unless the solves are timed (--repeat), which leave it off
static glio_ctx* create_context(const glio_params& prm, bool count_launches) {
  glio_ctx* ctx = nullptr;
  if (glio_create(0, &prm, &ctx) != GLIO_OK) { fprintf(stderr, "glio_create: %s\n", glio_last_error(nullptr)); exit(3); }
  if (count_launches && glio_profile_enable(ctx, 1) != GLIO_OK) exit(3);
  return ctx;
}

// launches so far of the named kernels; 0 without a context
static int64_t launches(glio_ctx* ctx, std::initializer_list<const char*> names) {
  int64_t n = 0;
  if (ctx)
    for (const char* k : names) { int64_t c = 0; glio_profile_get(ctx, k, nullptr, &c); n += c; }
  return n;
}

// a solve's first lines; the driver's block and launch counts follow, then print_solve_tail
static void print_solve_head(const ceres::Solver::Summary& S) {
  printf("termination %d\n", (int)S.termination_type);
  printf("iters %d\n", (int)S.iterations.size());
}

// costs, iterations and each keyframe's pose (t, q) and, if given, speed-bias, at %.17g
static void print_solve_tail(const ceres::Solver::Summary& S, int K, const std::vector<double>& t, const std::vector<double>& q,
                             const std::vector<double>* sb) {
  printf("cost %.17g %.17g\n", S.initial_cost, S.final_cost);
  for (auto& it : S.iterations) printf("it %d %d %.17g %.17g\n", it.iteration, (int)it.step_is_successful, it.cost, it.trust_region_radius);
  for (int k = 0; k < K; ++k) {
    printf("pose %d %.17g %.17g %.17g %.17g %.17g %.17g %.17g\n", k, t[3 * k], t[3 * k + 1], t[3 * k + 2], q[4 * k], q[4 * k + 1], q[4 * k + 2], q[4 * k + 3]);
    if (sb) { printf("sb %d", k); for (int i = 0; i < 9; ++i) printf(" %.17g", (*sb)[9 * k + i]); printf("\n"); }
  }
}

#endif  // GLIO_TESTS_SHIM_DRIVER_H_
