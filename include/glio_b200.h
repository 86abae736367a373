/*
 * glio_b200.h — C ABI of the H100-native LiDAR hot path of GLIO.
 *
 * This is the drop-in boundary: plain pointers and sizes, no torch / Eigen / PCL / Ceres / ROS types.
 * Every entry point names the reference interface it replaces (paths relative to the GLIO repository
 * root, reference commit 332d19ff).  The Ceres-compatible C++ shim (glio_b200/shim/ceres/ headers) and the
 * Python mirror (glio_b200/api.py) are thin layers over exactly these functions.
 *
 * Conventions
 *   - points: float32 xyz with a caller-given stride in floats (3 = packed xyz, 8 = pcl::PointXYZI as
 *     stored in pcl::PointCloud<PointType>::points, GLIO/include/utils/common.h:87-89).
 *   - poses: double[7] = t(x,y,z), q(w,x,y,z) — the reference's tmpTrans[k] / tmpQuat[k] parameter
 *     blocks (GLIO/src/Estimator.cpp:345-347).
 *   - every function returns 0 on success or a negative glio_status; glio_last_error() gives the text.
 *     No exception crosses the boundary and nothing aborts.
 *   - mem: GLIO_HOST pointers are copied for the duration of the call only; GLIO_DEVICE pointers are
 *     device addresses on the context's GPU (used by bench "value" runs with inputs resident in HBM).
 *   - a glio_ctx is single-threaded; create one per concurrent caller (window solve / batch solve run on
 *     different threads in the reference, Estimator.cpp:5352-5368).  Each context owns one CUDA stream.
 *     Distinct contexts may run at the same time on any threads and on any GPUs of the process; one context
 *     is never called from two threads at once.
 *   - a call runs on its context's GPU and returns with the calling thread's current CUDA device as it found
 *     it, so contexts on several GPUs can be driven from one thread.
 *   - there is NO CPU fallback: without a CUDA device glio_create fails with GLIO_ERR_NO_DEVICE.
 */
#ifndef GLIO_B200_H
#define GLIO_B200_H
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct glio_ctx glio_ctx;

typedef enum {
  GLIO_OK = 0,
  GLIO_ERR_NO_DEVICE = -1,
  GLIO_ERR_CUDA = -2,
  GLIO_ERR_ARG = -3,
  GLIO_ERR_STATE = -4,
  GLIO_ERR_NCCL = -5,
  GLIO_ERR_NUMERIC = -6
} glio_status;

enum { GLIO_HOST = 0, GLIO_DEVICE = 1 };

/* per-query association status (mirrors the reference's three failure counters, Estimator.cpp:3641-3643) */
enum { GLIO_MATCH_VALID = 0, GLIO_MATCH_FAIL_RADIUS = 1, GLIO_MATCH_FAIL_PLANE = 2, GLIO_MATCH_FAIL_WEIGHT = 3 };
/* per-query edge association status (glio_window_associate_edges) */
enum { GLIO_EDGE_VALID = 0, GLIO_EDGE_FAIL_RADIUS = 1, GLIO_EDGE_FAIL_LINE = 2 };

/* All tunables of the path in one POD (SURVEY.md §5 "Config / flags"). */
typedef struct {
  double kd_max_radius;    /* Estimator/kd_max_radius 1.5 — compared with a SQUARED distance (Estimator.cpp:3651) */
  double surf_dist_thres;  /* Estimator/surf_dist_thres 0.18 (Estimator.cpp:3671) */
  double lidar_const;      /* Estimator/lidar_const 7.5 (Estimator.cpp:3690) */
  double weight_min;       /* 0.3 hard-coded (Estimator.cpp:3681) */
  double huber_delta;      /* lossKernel 1.0 (Estimator.cpp:70,2092); <= 0 disables the loss */
  double q_lb[4];          /* extrinsic, wxyz (Estimator.cpp:270-274,873-877) */
  double t_lb[3];
  double batch_max_radius; /* 1.5 hard-coded (Estimator.cpp:3751) */
  double batch_dist_thres; /* 0.18 hard-coded (Estimator.cpp:3778) */
  double batch_score;      /* 2.5 hard-coded (Estimator.cpp:3798) */
  float cell_size;         /* uniform-grid cell edge in metres; 0 = choose from point density */
  int32_t keep_debug;      /* 1: keep idx5/sqd5/plane/pm per query for glio_get_assoc_debug (parity tests) */
  int32_t unit_score;      /* 0: residual score = lidar_const*weight (LidarPlaneNormFactor, Estimator.cpp:3690);
                            * 1: score = lidar_const for every match - with lidar_const = 1, identity extrinsic, kd_max_radius 1.0,
                            *    surf_dist_thres 0.06, weight_min 0.4, huber_delta 0.1 this is the front end's scan matcher
                            *    (LidarOdometry.cpp:343-404, :499-521; LidarPlaneNormIncreFactor, LidarKeyframeFactor.h:222-257) */
} glio_params;

void glio_default_params(glio_params* p);

/* lifecycle */
int glio_create(int device, const glio_params* params, glio_ctx** out);
void glio_destroy(glio_ctx* ctx);
const char* glio_last_error(const glio_ctx* ctx);   /* ctx may be NULL: the last error of the calling thread */
int glio_synchronize(glio_ctx* ctx);
/* the context's CUDA stream (cudaStream_t as void*) so callers can time with events on it */
void* glio_stream(glio_ctx* ctx);
/* number of kernels this context has launched so far (bench.py "gpu_launches") */
int64_t glio_launch_count(const glio_ctx* ctx);

/* per-kernel device time: when enabled every launch is bracketed by CUDA events on the context's stream;
 * glio_profile_get sums the elapsed time of all launches of the named kernel since profiling was enabled
 * (names: K0 k_init_bounds, k_load_bounds, k_cell_hist, k_cell_scatter, k_scan_block, k_scan_add;
 * K1 k_transform_hist, k_order_scatter, k_knn_box, k_plane_fit, k_plane_fit_pair, k_flags, k_compact;
 * K2 k_eval_unary, k_eval_unary_cost, k_eval_binary, k_eval_binary_cost, k_bin_assemble; local map k_lm_transform, k_vox_*;
 * front end k_feat_curvature, k_feat_select, k_feat_voxel, k_feat_offsets, k_feat_gather; sweep preparation k_sp_bounds,
 * k_sp_consts, k_sp_classify, k_sp_ranges, k_sp_emit; odometry k_odom_publish; loop-closure registration k_lc_load, k_lc_qhist,
 * k_lc_qscatter, k_lc_init, k_lc_nn, k_lc_compact, k_lc_sum0, k_lc_sum1, k_lc_means, k_lc_solve, k_lc_transform, k_lc_final,
 * k_lc_fitness; band Cholesky k_band_chol_solve). */
int glio_profile_enable(glio_ctx* ctx, int on);
int glio_profile_get(glio_ctx* ctx, const char* kernel_name, double* ms_total, int64_t* launches);
/* statistics: number of queries a first kNN search pass handed to a second pass.  The box search has no second pass, so
 * this always reports 0 and `reset` is ignored; the entry point is kept for existing callers. */
int glio_get_stats(glio_ctx* ctx, int64_t* knn_fallback_queries, int reset);
/* vec_surf_res_cnt for slots 0..W-1 (all matches) and the number currently active (after glio_select) */
int glio_get_match_counts(glio_ctx* ctx, int W, int64_t* n_match, int64_t* n_active);

/* lidar->map pose of a keyframe:  Q2 = Q * q_lb^-1 ; T2 = T - Q2 * t_lb   (Estimator.cpp:2216-2217) */
void glio_lidar_pose(const glio_params* prm, const double pose_body[7], double t2[3], double q2[4]);

/* ---- K0: local-map upload + uniform-grid build.
 * Replaces kd_tree_surf_local_map->setInputCloud(surf_local_map_ds)  (Estimator.cpp:2056).
 * Coordinate domain of every grid kNN search (surf / corner association, pair mode, loop-closure ICP): any finite float
 * coordinates.  The searches stay exact (bit-identical to brute force) at any world offset and grid extent: their face
 * tests keep a margin of max(2 mm, 8 float spacings of the grid's largest coordinate), 2 mm while the grid stays within
 * 2^12 m of the origin.  Above that the margin grows with the coordinates (6 cm at 2^16 m, 1 m at 2^20 m), and with it the
 * cells a query scans; results do not change.  Tested to 2^18 m offsets and 200 km wide grids. */
int glio_set_map(glio_ctx* ctx, const float* xyz, int64_t M, int stride_floats, int mem);
/* start the upload of the NEXT map from (pinned) host memory on the copy stream and return; the following glio_set_map with the same
 * pointer / count / stride uses the staged copy.  The poses a map is built from are final when the solve returns, so a caller can
 * hand the rebuilt map over while the window is still being marginalised. */
int glio_map_prefetch(glio_ctx* ctx, const float* xyz, int64_t M, int stride_floats);

/* ---- Local map maintenance on the device (SURVEY 8 f-1).
 * Replaces Estimator::buildLocalMapWithLandMark (Estimator.cpp:3529-3610: the deque `recent_surf_keyframes` of
 * world-frame keyframe clouds and their concatenation `surf_local_map`) and the map half of downSampleCloud
 * (:3615-3618: ds_filter_surf_map, pcl::VoxelGrid leaf 0.4 m set at :854) followed by
 * kd_tree_surf_local_map->setInputCloud (:2056).  The keyframe clouds stay resident on the GPU; only a new keyframe's
 * cloud crosses PCIe.
 *   glio_localmap_push       recent_surf_keyframes.push_front / push_back(transformCloud(cloud, {t, q}))   (:3574, :3600)
 *                            with t = q_po*t_bl + t_po, q = q_po*q_bl formed by the caller as at :3563-3564
 *   glio_localmap_pop_front  recent_surf_keyframes.pop_front()                                               (:3580)
 *   glio_localmap_clear      recent_surf_keyframes.clear()                                                   (:3549)
 *   glio_localmap_build      concatenate (:3605-3608), VoxelGrid(leaf) (:3617-3618), make it the searchable map; leaf <= 0
 *                            skips the filter.  PCL sums the points of a voxel in the order std::sort leaves them; this
 *                            sums them in input order (the deterministic member of that family).
 *   glio_get_map             the points of the current map in their original order (filtered map: ascending voxel index). */
int glio_localmap_clear(glio_ctx* ctx);
int glio_localmap_push(glio_ctx* ctx, int at_front, const float* cloud_xyz, int64_t n, int stride_floats, int mem,
                       const double t[3], const double q[4]);
int glio_localmap_pop_front(glio_ctx* ctx);
int glio_localmap_size(glio_ctx* ctx, int* n_frames, int64_t* n_points);
int glio_localmap_build(glio_ctx* ctx, float leaf, int64_t* n_map);
int glio_get_map(glio_ctx* ctx, int64_t capacity, float* xyz, int64_t* n_map);

/* ---- pcl::VoxelGrid of any cloud (SURVEY 8 f-8): downSampleCloud's scan filter ds_filter_surf.filter (Estimator.cpp:3628-3630,
 * leaf surfDSRange set at :852), whose output surf_last_ds becomes the keyframe cloud surf_frames[k] (:4150-4153).
 * xyz[n] (0 <= n < 2^31): x,y,z at floats 0..2 of a stride in [3,64] (8 = pcl::PointXYZI), host or device memory (device: 4-byte
 * aligned memory of the context's GPU).  PCL's applyFilter: inv = 1/leaf, float min / max; when (int64)((max - min) inv) + 1
 * multiplied over the axes exceeds INT32_MAX the input x,y,z come back in input order with *filtered = 0; otherwise voxel index
 * ijk0 + ijk1 div0 + ijk2 div0 div1 (int arithmetic, wrapped to 32 bits, ordered unsigned), one point per occupied voxel in
 * ascending index, its float sums in input order divided by the float count (*filtered = 1).  PCL sums a voxel in the order
 * std::sort leaves it; input order is the deterministic member of that family, the one glio_localmap_build produces too.  Only
 * x,y,z are carried: PCL also averages intensity, which GLIO sets to scanID + 0.1 relTime (Preprocessing.cpp:509), not a
 * measurement.  Output: packed x,y,z in out_xyz (host or device memory per out_mem; device: 4-byte aligned memory of the context's
 * GPU).  *n_out always receives the true count; when it exceeds capacity the call fails with GLIO_ERR_ARG and writes nothing to
 * out_xyz.  n = 0 gives 0 points and launches nothing.  Non-finite coordinates, leaf <= 0 or non-finite, a stride out of range,
 * null or misaligned pointers are GLIO_ERR_ARG.  filtered may be NULL.  The cost follows n, not the bounding box (a stable radix
 * sort of the voxel keys); no box size is refused.  Uses its own work space: the context's parameters, map, local map, window
 * slots, batch frames, odometries and loop objects are untouched.  Returns when its work is complete. */
int glio_voxel_filter(glio_ctx* ctx, const float* xyz, int64_t n, int stride_floats, int in_mem, float leaf, int64_t capacity, float* out_xyz,
                      int out_mem, int64_t* n_out, int32_t* filtered);

/* ---- K1: scan-to-map surf association for ONE keyframe slot.
 * Replaces Estimator::findCorrespondingSurfFeatures(idx, q, t)  (Estimator.cpp:3633-3708):
 * q,t is the lidar->map pose (Q2,T2 of Estimator.cpp:2216-2217).  The scan stays resident in the slot.
 * *n_match receives vec_surf_res_cnt[idVec].  Matches are kept on the device in scan order (the order of the
 * reference's push_back), as (point, weight*normal, weight*d, weight). */
int glio_assoc_scan_to_map(glio_ctx* ctx, int slot, const float* scan_xyz, int64_t Q, int stride_floats, int mem,
                           const double t[3], const double q[4], int64_t* n_match);

/* One keyframe's scan into one slot (host buffers travel on the copy stream; the next association waits for them), and the
 * slide of the window by one keyframe (slideWindow in the reference: slot k+1 -> slot k, matches included; no copies).  A
 * sliding window hands over ONE new scan per keyframe: the other W-1 stay resident. */
int glio_window_set_scan(glio_ctx* ctx, int slot, const float* scan_xyz, int64_t Q, int stride_floats, int mem);
int glio_window_slide(glio_ctx* ctx, int W);

/* All W keyframes of the window in one launch (same results as W calls of glio_assoc_scan_to_map).
 * poses_body[W*7] are the keyframe (IMU-body) poses tmpTrans/tmpQuat; the lidar->map pose is formed on the
 * device-side host code exactly as Estimator.cpp:2216-2217 with params.q_lb/t_lb.
 * glio_window_set_scans with GLIO_HOST buffers is ASYNCHRONOUS: the copies run on the context's copy stream and the next
 * association waits for them, so the host buffers must stay valid until that association (or glio_synchronize) returns.
 * It does not touch the matches of the previous association: the scans of the NEXT window may be handed over while the
 * current window is still being solved (upload overlaps the solve). */
int glio_window_set_scans(glio_ctx* ctx, int W, const float* const* scans, const int64_t* Q, int stride_floats, int mem);
int glio_window_associate(glio_ctx* ctx, int W, const double* poses_body, int64_t* n_match /*W*/);

/* direct upload of a slot's match list when the association was done elsewhere (e.g. by an unmodified Estimator through
 * PCL): cp[3n], nsd[4n] = (weight*n, weight*d), weight[n]; score = lidar_const*weight.  Used by the Ceres shim. */
int glio_set_matches(glio_ctx* ctx, int slot, const float* cp, const float* nsd, const float* weight, int64_t n);
int glio_get_params(const glio_ctx* ctx, glio_params* out);

/* copy-out of one slot's matches (parity tests, and the Ceres shim's host view).  Any pointer may be NULL.
 *   cp[3n] float (scan-frame point), nsd[4n] float (weight*n, weight*d), weight[n] float, src[n] int32
 *   (index of the match's scan point).  score = lidar_const * (double)weight. */
int glio_get_matches(glio_ctx* ctx, int slot, int64_t capacity, float* cp, float* nsd, float* weight, int32_t* src,
                     int64_t* n_match);
/* per-query debug view (needs params.keep_debug): status[Q] u8, idx5[5Q], sqd5[5Q], pm[3Q], plane[4Q] double */
int glio_get_assoc_debug(glio_ctx* ctx, int slot, int64_t Q, uint8_t* status, int32_t* idx5, float* sqd5, float* pm,
                         double* plane);

/* ---- feature selection as an INPUT (Estimator.cpp:3894-3992 is an RNG sub-sampling; SURVEY fact 3).
 * keep[n] are indices into the slot's match list; n < 0 clears the selection (all matches active). */
int glio_select(glio_ctx* ctx, int slot, const int32_t* keep, int64_t n);

/* ---- feature selection on the device, with the reference's rules (Estimator.cpp:3894-4116) and a seeded sampler in place of its
 * std::random_device draws (DESIGN 2).  Every selection is an ordered uniform sample without replacement of F (window) or B
 * (batch) positions out of 0 .. n-2 of a list of n matches (the last match is never chosen, as in the reference).  Draw j:
 *   u_j = word j % 4 of Philox4x64-10 at counter (j/4 + 1, stream, nonce, 0) with key (seed, domain) -- the words of
 *         numpy.random.Philox(key=[seed, domain], counter=[0, stream, nonce, 0]).random_raw();
 *   r_j = mulhi64(u_j, n-1-j), no rejection: uniform on [0, n-1-j) up to a bias below 2^-33 for n < 2^31;
 *   index = the r_j-th (0-based) position of 0 .. n-2 not chosen yet, ascending.
 * domain: 0 window, 1 batch start/end, 2 batch incremental (3 to 5: the edge selections, glio_select_random_edges).  stream: the caller's id per window slot (the keyframe index, so a
 * keyframe's sample does not depend on its slot), (uint64)cur << 32 | oth per pair (so a sharded run selects what one context
 * selects).  nonce: per call, for the reference's fresh draws per solve or batch round (e.g. activation * 4 + iterCount).
 * One k_sel_sample launch per call covers every sampled slot or pair; its table goes up in one copy and the call does not
 * synchronise the stream (only a call whose predecessor's table upload has not run yet waits for that copy).  The host decides
 * each outcome from the match counts it already holds.  The selected records land where glio_select puts them. */
typedef struct {
  int32_t feature_res_num;        /* F = 100 (config_urban_hk.yaml:100), in [1, 4096] */
  int32_t rand_set_num;           /* R = 300 (:101), >= 1; decides only which sizes the reference leaves undefined */
  int32_t batch_feature_res_num;  /* B = 25 (:102), in [1, 4096] */
  int32_t batch_rand_set_num;     /* BR = 400 (:103), >= B */
  int32_t random_select;          /* 1 (:104) */
  int32_t reserved;
  uint64_t seed;                  /* 0 */
  uint64_t nonce;                 /* 0 */
} glio_select_options;
void glio_select_default_options(glio_select_options* o);   /* the shipped configuration above */
/* featureSelection for slots 0..W-1 after their association; stream_ids[W].  A slot of n matches keeps all of them when n < 1 or
 * n - 1 < F, keeps none when random_select is 0 (the reference's loop never runs), else the F sampled matches in draw order.
 * n_active[W] (may be NULL) receives the active counts. */
int glio_select_random(glio_ctx* ctx, int W, const int64_t* stream_ids, const glio_select_options* options, int64_t* n_active);
/* The active index list of a slot (glio_select's list or the sampled one): *n = -1 when all matches are active, else the count;
 * keep[capacity] receives it (NULL: only *n is written; a capacity below the count is GLIO_ERR_ARG). */
int glio_get_selection(glio_ctx* ctx, int slot, int64_t capacity, int32_t* keep, int64_t* n);

/* ---- K2: evaluate all active unary plane residuals at the given body poses.
 * Replaces ceres::ResidualBlock::Evaluate over LidarPlaneNormFactor (LidarKeyframeFactor.h:73-122) + HuberLoss +
 * QuaternionParameterization and the J^T J / J^T r accumulation for those blocks.
 *   jac_kind 0: Ceres tangent Jacobian (solve path); 1: ambient x,y,z quaternion columns
 *   (marginalisation path, MarginalizationFactor.cpp:9-17).
 *   H[W*36] row-major 6x6 per keyframe (t | rotation), g[W*6] = J^T r, cost[W] = sum 0.5*rho(r^2).
 *   H and g may be NULL (cost-only evaluation at a candidate point). */
int glio_eval_unary(glio_ctx* ctx, int W, const double* poses_body, int jac_kind, double* H, double* g, double* cost);

/* per-residual view for the Ceres-API path: r[n], J[6n] (corrected, tangent) for one slot */
int glio_eval_unary_residuals(glio_ctx* ctx, int slot, const double pose_body[7], int jac_kind, int64_t capacity,
                              double* r, double* J, int64_t* n);

/* ---- the minimizer iteration around K2 (replaces ceres::Solve for the window problem, Estimator.cpp:2424-2433):
 * Ceres 2.0.0 TrustRegionMinimizer + DoglegStrategy + Jacobi scaling + normal-equation Cholesky semantics
 * (ceres.tgz::internal/ceres/{trust_region_minimizer,dogleg_strategy,trust_region_step_evaluator}.cc).
 * LiDAR blocks come from the device, and so does the IMU chain when glio_window_use_imu_factors is on (the factors from the
 * caller's pre-integration, glio_window_set_imu_factors).  The other factors of the problem (the marginalisation prior, the
 * first window's speed-bias prior, the IMU chain when the switch is off) are added by the host_factors callback into the same
 * dense tangent-space normal equations. */
typedef struct {
  int32_t max_num_iterations;            /* 15 (Estimator.cpp:2427); batch: max_num_iter */
  int32_t dogleg_type;                   /* 0 TRADITIONAL_DOGLEG (window), 1 SUBSPACE_DOGLEG (batch, Estimator.cpp:3280) */
  int32_t use_nonmonotonic_steps;        /* 0 window (Estimator.cpp:2430) / 1 batch (:3281) */
  int32_t max_consecutive_nonmonotonic_steps; /* 5  (ceres solver.h:263) */
  double initial_trust_region_radius;    /* 1e4  (solver.h:276) */
  double max_trust_region_radius;        /* 1e16 */
  double min_trust_region_radius;        /* 1e-32 */
  double min_relative_decrease;          /* 1e-3 */
  double min_lm_diagonal;                /* 1e-6 */
  double max_lm_diagonal;                /* 1e32 */
  int32_t max_num_consecutive_invalid_steps; /* 5 */
  int32_t jacobi_scaling;                /* 1 */
  double function_tolerance;             /* 1e-6 */
  double gradient_tolerance;             /* 1e-10 */
  double parameter_tolerance;            /* 1e-8 */
  int32_t fuse_candidate_jacobian;       /* 1: evaluate J with the candidate cost and reuse it on acceptance (same numbers, one pass less) */
  int32_t trust_region_strategy;         /* 0 DOGLEG (Estimator.cpp:2427, :3278), 1 LEVENBERG_MARQUARDT (Ceres' default: the front end's scan
                                            matcher, LidarOdometry.cpp:521-530; ceres.tgz::internal/ceres/levenberg_marquardt_strategy.cc) */
} glio_solver_options;
void glio_default_solver_options(glio_solver_options* o);

typedef struct {
  int32_t iteration, step_is_valid, step_is_successful, reserved;
  double cost, cost_change, gradient_max_norm, gradient_norm, step_norm, relative_decrease, trust_region_radius, mu;
} glio_iteration;

typedef struct {
  int32_t termination;                   /* 0 CONVERGENCE, 1 NO_CONVERGENCE, 2 FAILURE */
  int32_t num_iterations;                /* records written to the iteration log (iteration 0 included) */
  int32_t num_successful_steps, num_unsuccessful_steps;
  int32_t num_evaluations, num_jacobian_evaluations, num_linear_solves, num_valid_steps;
  double initial_cost, final_cost;
  double eval_seconds;                   /* wall clock inside residual/Jacobian evaluation (device kernel + copies + host factors) */
  double linear_solver_seconds;          /* wall clock inside the band Cholesky solves */
  double total_seconds;
  char message[128];
} glio_solver_summary;

/* Adds the host-side factors at the given state.  n = W*(speed_bias ? 15 : 6), tangent order per keyframe
 * [t(3), rotation(3), speed_bias(9)].  H (n*n row-major, full symmetric) and g (n) are ACCUMULATED INTO when
 * want_jac != 0 (they already hold the LiDAR blocks); *cost is accumulated into.  Return 0 on success. */
typedef int (*glio_host_factors_fn)(void* user, int W, const double* poses, const double* speed_bias, int want_jac,
                                    double* H, double* g, double* cost);

/* poses[W*7] (and speed_bias[W*9], may be NULL) are in/out: on return the lowest-cost accepted state, like the
 * parameter blocks after ceres::Solve.  iter_log[iter_cap] and step_log[step_cap doubles: one n-vector per valid
 * step, the tangent update Delta_k of SURVEY B.4] may be NULL. */
int glio_window_solve(glio_ctx* ctx, int W, double* poses, double* speed_bias, glio_host_factors_fn host_factors, void* user,
                      const glio_solver_options* options, glio_solver_summary* summary, glio_iteration* iter_log, int iter_cap,
                      double* step_log, int64_t step_cap);

/* Same solve with the host factors accumulating straight into LOWER-BAND storage (entry (i,j), i-hb <= j <= i, at
 * Hband[i*(hb+1) + (j-i+hb)]): no dense n x n scratch.  half_bandwidth must cover every coupling the host factors create
 * (window: prior + IMU chain -> 2*nt-1 = 29 with speed-bias states); < 5 means dense.  With glio_window_use_imu_factors on, the
 * band covers the device IMU pairs' span whatever half_bandwidth says. */
typedef int (*glio_host_factors_band_fn)(void* user, int K, const double* poses, const double* speed_bias, int want_jac,
                                         double* Hband, int hb, double* g, double* cost);
int glio_window_solve_band(glio_ctx* ctx, int W, double* poses, double* speed_bias, glio_host_factors_band_fn host_factors,
                           int half_bandwidth, void* user, const glio_solver_options* options, glio_solver_summary* summary,
                           glio_iteration* iter_log, int iter_cap, double* step_log, int64_t step_cap);

/* ---- stand-in host factors (CPU C++, analytic) with the block structure of the reference's non-LiDAR factors:
 * prior 15x[t,q,sb] (marginalisation-prior-like), between 15x[t,q,sb|t,q,sb] (IMU-chain-like), range 1x[t,q]
 * (pseudorange-like).  glio_hf_evaluate has the glio_host_factors_fn signature (user = the set).  They exist so the
 * plumbing of host factors + device LiDAR blocks can be tested and benchmarked without ROS / GNSS data; the real
 * MarginalizationFactor / dd_psr_factor plug in through the same callback (or the Ceres shim); the real ImuFactor chain also
 * runs on the device (glio_window_use_imu_factors, glio_batch_use_imu_factors). */
typedef struct glio_host_factor_set glio_host_factor_set;
glio_host_factor_set* glio_hf_create(void);
void glio_hf_destroy(glio_host_factor_set* s);
void glio_hf_add_prior(glio_host_factor_set* s, int kf, const double t0[3], const double q0[4], const double* sb0 /*9 or NULL*/,
                       const double sqrt_w[15]);
void glio_hf_add_between(glio_host_factor_set* s, int i, int j, const double dp[3], const double dq[4], const double dv[3], double dt,
                         const double sqrt_w[15]);
void glio_hf_add_range(glio_host_factor_set* s, int kf, const double lever[3], const double sat[3], double rho, double w);
int glio_hf_evaluate(void* user, int W, const double* poses, const double* speed_bias, int want_jac, double* H, double* g, double* cost);

/* ---- front-end feature extraction (SURVEY 8 f-4): Preprocessing::cloudHandler, GLIO/src/Preprocessing.cpp:529-655.
 * cloud_xyzi = `laserCloud` of the reference: the scan lines concatenated ring after ring, x,y,z,intensity at stride_floats
 * (>= 4) with the intensity at float intensity_offset (packed x,y,z,i: stride 4, offset 3; pcl::PointXYZI: stride 8, offset 4),
 * scan_start / scan_end = scanStartInd / scanEndInd per ring (:529-534; every range inside
 * [5, n-6]).  The processed rings (scan_end - scan_start >= 6 and ring % ds_rate == 0) run concurrently, so ordered by
 * scan_start each must begin at least 5 points after the previous one's scan_end (the reference's layout leaves 11); a table
 * with processed rings closer than that, or overlapping, is refused with GLIO_ERR_ARG naming the two rings.
 * Outputs, any may be NULL: cloudCurvature[n], cloudLabel[n] (2 sharp, 1 less sharp, -1 flat, 0 other), and the four feature sets in the reference's push_back order as indices into the cloud (cornerPointsSharp, cornerPointsLessSharp,
 * surfPointsFlat, the less-flat points BEFORE the voxel filter) plus surfPointsLessFlat itself (x,y,z,intensity after the
 * per-ring pcl::VoxelGrid of leaf ds_v).  Equal curvatures are ordered by index (std::sort leaves it open). */
int glio_extract_features(glio_ctx* ctx, const float* cloud_xyzi, int64_t n, int stride_floats, int intensity_offset, int mem, int n_scans, const int32_t* scan_start,
                          const int32_t* scan_end, int ds_rate, double edge_thres, double surf_thres, float ds_v, float* curvature, int8_t* label,
                          int32_t* sharp, int64_t* n_sharp, int32_t* less_sharp, int64_t* n_less_sharp, int32_t* flat, int64_t* n_flat,
                          int32_t* less_flat, int64_t* n_less_flat, float* less_flat_ds, int64_t* n_less_flat_ds);

/* ---- front-end sweep preparation (SURVEY 8 f-5): Preprocessing::cloudHandler, GLIO/src/Preprocessing.cpp:387-526.
 * raw = the sweep as received, x,y,z at floats 0..2 of stride_floats (pcl::PointXYZI: stride 8; the input intensity is not used).
 * Points with a non-finite coordinate or closer than 3 m are dropped (:396-397), every other point gets its ring id from its
 * elevation for n_scans 16 / 32 / 64 (:438-483; out-of-range rings are skipped), its relative time from the azimuth state machine
 * (:489-507), intensity = ring + 0.1 relTime, and is de-skewed by Identity.slerp(relTime, q_imu) conjugated by q_lb
 * (undistortion, :176-200).  out_xyzi receives `laserCloud`: the kept points ring after ring in input order as packed float4
 * x,y,z,intensity (the stride 4, offset 3 layout of glio_extract_features), scan_start / scan_end[n_scans] =
 * scanStartInd / scanEndInd (:521-526; an empty ring has start = end + 11).  q_imu / q_lb are w,x,y,z; NULL means identity,
 * and a q_imu with a NaN component is replaced by identity (:415-417).  *n_out is always the true count; if it exceeds
 * out_capacity the call fails with GLIO_ERR_ARG and nothing is written past out_capacity.  out_mem = GLIO_DEVICE writes
 * straight into device memory, ready for glio_extract_features(..., 4, 3, GLIO_DEVICE, ...); that out_xyzi must be
 * 16-byte aligned (it is written as float4), raw must be 4-byte aligned, and GLIO_DEVICE pointers must belong to the
 * context's GPU (otherwise GLIO_ERR_ARG before anything runs).  The call returns when its work is complete.  A sweep in which no point
 * survives the NaN / 3 m filters fails with GLIO_ERR_ARG (the reference would read point 0 of an empty cloud).
 * atanf / atan2f are correctly rounded (DESIGN 2); glio_scanprep_stats counts the evaluations that needed the double-double
 * decision (reset != 0 zeroes the counter). */
int glio_prepare_scan(glio_ctx* ctx, const float* raw, int64_t n, int stride_floats, int mem, int n_scans, const double q_imu[4],
                      const double q_lb[4], float* out_xyzi, int out_mem, int64_t out_capacity, int64_t* n_out,
                      int32_t* scan_start, int32_t* scan_end);
int glio_scanprep_stats(glio_ctx* ctx, int64_t* guard_hits, int reset);

/* The sweep's IMU rotation qIMU: Preprocessing::processIMU + solveRotation (:202-207, :222-259, deltaQ of
 * GLIO/include/utils/math_tools.h:126-138), integrating the gyro samples of the buffer up to t_scan_next from identity.
 * stamps[n_buf] (seconds) and gyro_xyz[3*n_buf] (rad/s) are the whole IMU buffer received so far (imu_buf); the state carries
 * idx_imu / current_time_imu / gyr_0 from sweep to sweep.  Zero-initialise it: the first call with samples performs
 * imuHandler's first-sample initialisation (:281-293).  With no sample yet q = identity.  Host code, no context. */
typedef struct {
  int64_t idx_imu;
  double current_time_imu;
  double gyr_0[3];
  int32_t first_imu;
  int32_t reserved;
} glio_imu_state;
int glio_imu_sweep_rotation(glio_imu_state* st, const double* stamps, const double* gyro_xyz, int64_t n_buf, double t_scan_next,
                            double q_wxyz[4]);

/* ---- front-end LiDAR odometry (SURVEY 8 f-6): the LidarOdometry node, GLIO/src/LidarOdometry.cpp:661-695 (run) and what it calls.
 * One glio_odom_step per sweep takes that sweep's surf features (`/surf_features`, the less_flat_ds of glio_extract_features) and
 * optionally its full cloud (`/lidar_cloud_cutted`, the output of glio_prepare_scan), both packed float4 x,y,z,intensity, and runs
 *   sweep 1      savePoses of the identity pose and an EMPTY scan frame, clouds published unchanged, no odometry (checkInitialization);
 *   later sweeps poseInitialization (:406-433); the local map (:267-288): on sweep 2 the sweep's own surf cloud, afterwards the last
 *                20 sweeps' VoxelGrid(0.2)-filtered surf clouds moved to the world frame by their final poses, concatenated oldest
 *                first; VoxelGrid(0.2) of the map and of the surf cloud (:305-313; PCL's pass-through on voxel-index overflow
 *                included); fewer than 10 map points: stop here, the pose stays the prediction and the keyframe flag keeps its
 *                previous value (:477-480); otherwise scan_match_cnt rounds (8 on sweep 2) of association (findCorrespondingSurfFeatures,
 *                :343-404: squared radius 1.0, plane 0.06, weight 0.4) + a fresh Levenberg-Marquardt solve (HuberLoss(0.1),
 *                LidarPlaneNormIncreFactor; a round without matches leaves the pose as it is, like Ceres with no residual) +
 *                unifyQuaternion; the keyframe rule (:566-578); savePoses; computeRelative (:435-471); on a keyframe the
 *                clouds are published, translation de-skewed by the relative pose when deskew != 0 (publishCloudLast, :619-659).
 * The odometry runs on its context's device, stream, launch counter and profiler but owns all its state: it never reads or
 * changes the context's glio_params, map, local map, window slots or batch frames, so one context can run
 * prepare -> extract -> odometry and the window path side by side.  glio_destroy frees odometries still attached to the context. */
typedef struct {
  int32_t max_num_iter;       /* lidar_odometry/max_num_iter: 12 (GLIO/config/config_urban_hk.yaml:19; code default 15) */
  int32_t scan_match_cnt;     /* 1 (:20); the second sweep always runs 8 rounds (LidarOdometry.cpp:493-496); at most 8 */
  int32_t deskew;             /* if_to_deskew: 0 (:21; code default 1) */
  int32_t reserved;
  double max_solver_time_s;   /* max_solver_time_in_seconds 0.015 (LidarOdometry.cpp:524): wall clock, checked after every iteration */
} glio_odom_options;
void glio_odom_default_options(glio_odom_options* o);   /* the shipped configuration above */

enum { GLIO_ODOM_MAX_ROUNDS = 8 };
typedef struct {
  double pose[7];             /* /odom: t(x,y,z), q(w,x,y,z) - the reference's abs_pose is q(w,x,y,z), t(x,y,z) */
  double rel_pose[7];         /* /each_odom, the pose relative to the previous sweep, t then q (reference rel_pose: q then t) */
  int32_t initialised;        /* 1 on the first sweep after creation / reset: clouds passed through, no odometry */
  int32_t keyframe;           /* kf: the clouds were published (always 0 on the first sweep) */
  int32_t skipped;            /* the filtered map had fewer than 10 points: no round ran */
  int32_t n_rounds;
  int64_t n_map, n_scan;      /* points of the filtered map and of the filtered scan */
  int64_t round_n_match[GLIO_ODOM_MAX_ROUNDS];
  int32_t round_iterations[GLIO_ODOM_MAX_ROUNDS];    /* LM iteration records (iteration 0 included); 0 for a round without matches */
  int32_t round_successful[GLIO_ODOM_MAX_ROUNDS];    /* successful steps */
  int32_t round_termination[GLIO_ODOM_MAX_ROUNDS];   /* glio_solver_summary.termination */
  int32_t reserved;
  double round_pose[GLIO_ODOM_MAX_ROUNDS][7];        /* pose after each round (t, q), after unifyQuaternion */
  glio_solver_summary summary;                       /* the last round's solve */
} glio_odom_report;

typedef struct glio_odom glio_odom;
int glio_odom_create(glio_ctx* ctx, const glio_odom_options* options /* NULL: defaults */, glio_odom** out);
void glio_odom_destroy(glio_odom* od);
int glio_odom_reset(glio_odom* od);   /* back to the state before the first sweep (buffers are kept) */
/* surf_xyzi[n_surf] / full_xyzi[n_full] (full may be NULL with n_full = 0) are host or device memory as surf_mem / full_mem say;
 * surf_out / full_out (each as large as its input, either may be NULL) are written only when the node publishes: on the first
 * sweep and on keyframes.  Device pointers must be 16-byte aligned memory of the context's GPU (the clouds are read and written
 * as float4); a bad argument is GLIO_ERR_ARG before anything runs.  An empty surf cloud is allowed (nothing matches).
 * The call returns when its work is complete. */
int glio_odom_step(glio_odom* od, const float* surf_xyzi, int64_t n_surf, int surf_mem, const float* full_xyzi, int64_t n_full, int full_mem,
                   float* surf_out, float* full_out, int out_mem, glio_odom_report* rep);
/* debug copy-out of the last step's filtered map (surf_from_map_ds, x,y,z in the filter's output order) and filtered scan
 * (surf_last_ds); either pointer may be NULL; the counts are always written.  Fails with GLIO_ERR_ARG if a capacity is too small. */
int glio_odom_get_clouds(glio_odom* od, int64_t map_capacity, float* map_xyz, int64_t* n_map, int64_t scan_capacity, float* scan_xyz,
                         int64_t* n_scan);

/* ---- loop-closure registration (SURVEY 8 f-7): the registration half of the Estimator's loop closure, detectLoopClosure and
 * performLoopClosure (GLIO/src/Estimator.cpp:5101-5273) up to the GTSAM BetweenFactor, which stays with the caller.
 *
 * glio_icp_align = pcl::IterativeClosestPoint<PointXYZI, PointXYZI>::align with an identity guess (:5204-5214), restated from PCL 1.8
 * (registration/impl/icp.hpp, transformation_estimation_svd.hpp = pcl::umeyama without scaling, correspondence_estimation.hpp,
 * default_convergence_criteria.hpp) and getFitnessScore (registration.hpp).  Per iteration: exact 1-NN of every source point in the
 * target (FLANN L2_Simple<float> distances, ties by index), kept when the float squared distance is <= max_correspondence_distance^2,
 * in source order; fewer than 3: NO_CORRESPONDENCES, not converged; else umeyama in float (Eigen 3.3 JacobiSVD<Matrix3f>), the
 * source transformed IN PLACE by that transformation in float ((t0 x + t1 y) + t2 z) + t3, final = transformation * final, and
 * DefaultConvergenceCriteria (max iterations: converged; cos = 0.5 (float trace - 1) >= 1 - eps and float |t|^2 <= eps; absolute
 * MSE change < 1e-12; relative MSE change < euclidean_fitness_epsilon).  The aligned cloud is the input transformed by final; the
 * fitness is the double mean of the 1-NN squared distances of that cloud over every point (DBL_MAX when no point counts).  Sums run
 * in the fixed order documented in glio_b200/csrc/loop.cu (DESIGN 2).  Kernel names for glio_profile_get: k_lc_load, k_lc_qhist,
 * k_lc_qscatter, k_lc_init, k_lc_nn, k_lc_compact, k_lc_sum0, k_lc_sum1, k_lc_means, k_lc_solve, k_lc_transform, k_lc_final,
 * k_lc_fitness (and the K0 grid kernels). */
enum { GLIO_ICP_NOT_CONVERGED = 0, GLIO_ICP_ITERATIONS = 1, GLIO_ICP_TRANSFORM = 2, GLIO_ICP_ABS_MSE = 3, GLIO_ICP_REL_MSE = 4,
       GLIO_ICP_NO_CORRESPONDENCES = 5 };   /* pcl::registration::DefaultConvergenceCriteria::ConvergenceState */
typedef struct {
  int32_t max_iterations;              /* setMaximumIterations(100)              (Estimator.cpp:5198) */
  int32_t reserved;
  double max_correspondence_distance;  /* setMaxCorrespondenceDistance(30)       (:5197) */
  double transformation_epsilon;       /* setTransformationEpsilon(1e-6)         (:5199) */
  double euclidean_fitness_epsilon;    /* setEuclideanFitnessEpsilon(1e-6)       (:5200); setRANSACIterations(5) has no effect on plain ICP */
} glio_icp_options;
void glio_icp_default_options(glio_icp_options* o);   /* the settings above */

typedef struct {
  float transformation[16];            /* this iteration's transformation_, row-major 4x4 */
  int64_t n_corr;                      /* correspondences it was estimated from */
  double mse;                          /* double mean of their squared distances (calculateMSE) */
} glio_icp_iteration;

typedef struct {
  int32_t converged;                   /* hasConverged() */
  int32_t state;                       /* GLIO_ICP_* */
  int32_t iterations;                  /* nr_iterations_ */
  int32_t host_syncs;                  /* host synchronisations the registration cost */
  int64_t n_source, n_target;
  int64_t n_corr;                      /* correspondences of the last correspondence estimation */
  int64_t launches;                    /* kernels launched */
  float final_transformation[16];      /* getFinalTransformation(), row-major 4x4 */
  double fitness;                      /* getFitnessScore() */
} glio_icp_result;

/* src[n_src] / tgt[n_tgt]: x,y,z at floats 0..2 of stride_floats (3..64), host or device memory as src_mem / tgt_mem say (device
 * pointers: 4-byte aligned memory of the context's GPU).  options NULL = glio_icp_default_options.  aligned_xyz[3 n_src] (host, may
 * be NULL): the aligned cloud.  iter_log[iter_cap] (may be NULL): the first iter_cap iterations.  corr_query / corr_match / corr_dist
 * (host, each may be NULL, room for corr_cap entries): the last correspondence estimation, (source index, target index, float squared
 * distance) in source order; res->n_corr is its true length.  Does not touch the context's map, local map, window slots or batch
 * frames.  Returns when its work is complete. */
int glio_icp_align(glio_ctx* ctx, const float* src, int64_t n_src, int src_stride, int src_mem, const float* tgt, int64_t n_tgt,
                   int tgt_stride, int tgt_mem, const glio_icp_options* options, float* aligned_xyz, glio_icp_result* res,
                   glio_icp_iteration* iter_log, int iter_cap, int32_t* corr_query, int32_t* corr_match, float* corr_dist, int64_t corr_cap);

/* The loop object: the Estimator's keyframe store for the loop closure and its detection / registration step.
 *   keyframe k: surf_frames[k] (its surf_last_ds, lidar frame, :4150-4153), pose_info_keyframe[k] (body pose t, q and time,
 *   :4253-4264) and pose_keyframe[k] (the same position as float x,y,z, the cloud of the radius search).  Keyframe clouds stay
 *   resident on the device: each crosses PCIe once, in glio_loop_add_keyframe.  glio_loop_set_poses overwrites poses after
 *   insertion (updatePose, :3435-3450; correctPoses); the times stay.
 *   glio_loop_step(select_xyz, time_new_odom) = performLoopClosure (:5183-5273) without the GTSAM half:
 *     detection (:5101-5181): radius search of pose_keyframe around select_xyz (float squared distance < float(r^2), sorted by
 *       distance, ties by index), closest_his_idx = the first result with |time - time_new_odom| > lc_time_thres; no candidate when
 *       none passes or |time_last_loop - time_new_odom| < 0.2; latest_frame_idx_loop = size - slide_window_width;
 *     the latest cloud: keyframes latest - j, j = 0..5, newest first, negative indices skipped; the history cloud: closest + j,
 *       j = -lc_map_width..lc_map_width, oldest first, outside [0, latest] skipped; each moved by q_po*q_bl, q_po*t_bl + t_po
 *       (transformCloud, :1517-1545; q_bl = q_lb^-1, t_bl = -(q_bl t_lb), :873-877), concatenated, VoxelGrid(leaf) (:855);
 *     glio_icp_align(latest_ds onto his_ds) with the options' ICP settings; accepted when converged and fitness <= lc_icp_thres;
 *     then pose_from = (qIncre * q_latest, qIncre * t_latest + t) with qIncre Eigen's quaternion of final's rotation, pose_to = the
 *       history keyframe's pose, noise score = fitness, time_last_loop = time[latest] (the caller adds
 *       BetweenFactor(poseFrom.between(poseTo)) to its own pose graph).
 *   With no candidate the step launches nothing.  The loop object runs on its context's device, stream, launch counter and profiler
 *   but owns its state: it never reads or changes the context's glio_params, map, local map, window slots, batch frames or
 *   odometries.  glio_destroy frees loop objects still attached to the context. */
typedef struct {
  double lc_search_radius;             /* 25 (GLIO/config/config_urban_hk.yaml:80; code default 7.0, Estimator.cpp:667-670) */
  double lc_time_thres;                /* 30 (:83; code default 30, Estimator.cpp:637-640) */
  int32_t lc_map_width;                /* 25 (:81; code default 25) */
  float lc_icp_thres;                  /* 0.2 (:82; code default 0.3); a float in the reference (Estimator.cpp:230) */
  int32_t slide_window_width;          /* 5 (:66) */
  float leaf;                          /* ds_filter_his_frames.setLeafSize(0.4) (Estimator.cpp:855) */
  double q_lb[4];                      /* extrinsic, w,x,y,z (config_urban_hk.yaml:90-93) */
  double t_lb[3];                      /* (:94-97) */
  glio_icp_options icp;
} glio_loop_options;
void glio_loop_default_options(glio_loop_options* o);   /* the shipped configuration above */

typedef struct {
  int32_t detected;                    /* detectLoopClosure() returned true: the registration ran */
  int32_t closest_his_idx;             /* -1: no keyframe passed the radius and time tests */
  int32_t latest_frame_idx;            /* latest_frame_idx_loop (valid when detected) */
  int32_t accepted;                    /* converged and fitness <= lc_icp_thres */
  int64_t n_latest, n_latest_ds, n_his, n_his_ds;   /* cloud sizes before / after the voxel filter */
  int64_t n_candidates;                /* keyframes inside the search radius */
  glio_icp_result icp;
  double pose_from[7], pose_to[7];     /* t then q (the reference builds gtsam poses from q and t) */
  double noise_score;                  /* the fitness, the variance of the loop factor's diagonal noise model */
  double time_last_loop;               /* after this step */
} glio_loop_report;

typedef struct glio_loop glio_loop;
int glio_loop_create(glio_ctx* ctx, const glio_loop_options* options /* NULL: defaults */, glio_loop** out);
void glio_loop_destroy(glio_loop* lp);
int glio_loop_reset(glio_loop* lp);    /* no keyframe, time_last_loop = 0 (device buffers are kept) */
/* cloud[n] (n >= 0) with stride_floats in [3,64], host or device memory (device: 4-byte aligned memory of the context's GPU);
 * pose[7] = body pose t, q; returns the keyframe's index in *index (may be NULL). */
int glio_loop_add_keyframe(glio_loop* lp, const float* cloud, int64_t n, int stride_floats, int mem, const double pose[7], double time,
                           int32_t* index);
int glio_loop_set_poses(glio_loop* lp, int first, int count, const double* poses /* count x 7 */);
int glio_loop_size(glio_loop* lp, int* n_keyframes);
int glio_loop_step(glio_loop* lp, const float select_xyz[3], double time_new_odom, glio_loop_report* rep);
/* debug copy-out of the last registration's filtered clouds (latest_key_frames_ds, his_key_frames_ds; x,y,z in the filter's output
 * order); either pointer may be NULL, the counts are always written; GLIO_ERR_ARG if a capacity is too small. */
int glio_loop_get_clouds(glio_loop* lp, int64_t latest_capacity, float* latest_xyz, int64_t* n_latest, int64_t his_capacity, float* his_xyz,
                         int64_t* n_his);
/* save_pcd's global map from the keyframe store (Estimator.cpp:5324-5349; mapping_interval 3 in config_urban_hk.yaml:87,
 * ds_filter_global_map leaf 0.2 at :856): keyframes 0, interval, 2 interval, ... < size, in that order, each point moved by
 * transformCloud(transformCloud(surf_frames[i], &Tbl), &pose_info_keyframe[i]) (:5340) with Tbl = (q_bl, t_bl) and the keyframe's
 * current pose (glio_loop_set_poses), each transform Eigen's double rotation rounded to float (two roundings, not the one combined
 * pose of the loop clouds); the concatenation (*n_raw points, n_raw may be NULL) filtered as glio_voxel_filter(leaf) does, PCL's
 * pass-through included.  Only x,y,z (the store holds no intensity).  Output conventions as glio_voxel_filter.  interval < 1 or
 * leaf <= 0 is GLIO_ERR_ARG; an empty store gives 0 points.  Writing the PCD file stays with the caller.  Neither the loop object's
 * state nor the context's changes. */
int glio_loop_global_map(glio_loop* lp, int interval, float leaf, int64_t capacity, float* xyz, int out_mem, int64_t* n_map, int64_t* n_raw,
                         int32_t* filtered);

/* ---- K3: marginalisation of the oldest keyframe (MarginalizationInfo, GLIO/src/MarginalizationFactor.cpp:82-202; call site
 * Estimator.cpp:2462-2608).  The reference re-evaluates EVERY LiDAR factor of the window (:2538-2576, one virtual Evaluate per
 * residual) plus the IMU factor KF0->KF1 and the previous prior, accumulates the dense A = J^T J, b = J^T r with the ambient
 * x,y,z quaternion columns (:9-17), removes KF0's 15 states by a Schur complement and factors the rest by an
 * eigen-decomposition (:176-201).  glio_window_marginalize does the LiDAR part on the device (K2 with jac_kind = 1: one 6x6
 * block + 6-vector per keyframe), asks the host callback for the other factors, and does the small dense algebra on the host.
 * Orderings (see glio_b200/csrc/marg.h): marginalisation ordering N = 6W+18 = [KF0: t,q,sb | KF1: t,q,sb | KF k>=2: t,q];
 * the prior keeps n = 6W+3 states, numbered as the NEXT window numbers them (addr_shift, Estimator.cpp:2583-2597).
 * host_marg(user, W, poses, speed_bias, A[N*N], b[N]) ACCUMULATES the non-LiDAR factors (may be NULL); with
 * glio_window_use_imu_factors on, the window's IMU factor KF0 -> KF1 comes from the device instead (see there). */
typedef int (*glio_host_marg_fn)(void* user, int W, const double* poses, const double* speed_bias, double* A, double* b);
typedef struct glio_marg_prior glio_marg_prior;
int glio_window_marginalize(glio_ctx* ctx, int W, const double* poses, const double* speed_bias, glio_host_marg_fn host_marg, void* user,
                            double eps /* 1e-8 in the reference */, glio_marg_prior** prior_out);
/* The same pass with its host half (A/b assembly, Schur complement, decomposition, prior) on a worker thread of the
 * context: the call returns when the device half is queued and host_marg has run, so the caller can hand the NEXT window's map and
 * association to the GPU meanwhile (the reference does these strictly one after the other, Estimator.cpp:2462-2608 then the next
 * processImage).  One job at a time per context.  glio_marg_job_wait joins the job, frees it and returns the prior (identical to
 * glio_window_marginalize's); call it before the next solve needs the prior.  glio_destroy joins AND frees an abandoned job: a job
 * handle must not be used after its context is gone (the same holds for a glio_odom, which glio_destroy also frees).  A context is otherwise single-threaded: calls on one context must not
 * overlap, the worker is the library's own. */
typedef struct glio_marg_job glio_marg_job;
int glio_window_marginalize_async(glio_ctx* ctx, int W, const double* poses, const double* speed_bias, glio_host_marg_fn host_marg,
                                  void* user, double eps, glio_marg_job** job_out);
int glio_marg_job_wait(glio_marg_job* job, glio_marg_prior** prior_out);
glio_marg_prior* glio_marg_prior_create(int W, const double* lin_jac, const double* lin_res, const double* x0_poses, const double* x0_sb);
void glio_marg_prior_destroy(glio_marg_prior* p);
int glio_marg_prior_size(const glio_marg_prior* p, int* n, int* W);
/* linearized_jacobians[n*n] row-major, linearized_residuals[n], keep_block_data (x0_poses[(W-1)*7], x0_sb[9]), and the
 * information form A_info = J^T J [n*n], b_info = J^T r [n]; any pointer may be NULL */
int glio_marg_prior_get(const glio_marg_prior* p, double* lin_jac, double* lin_res, double* x0_poses, double* x0_sb, double* A_info, double* b_info);
/* stand-in host factors: attach the prior to the next window's factor set (it then takes part in glio_hf_evaluate[_band] as a
 * MarginalizationFactor, MarginalizationFactor.cpp:232-330) and glio_hf_marg_evaluate = the glio_host_marg_fn of the set
 * (previous prior + priors on KF0 + the between factor KF0->KF1). */
int glio_hf_set_marg_prior(glio_host_factor_set* s, const glio_marg_prior* p /* copied; NULL removes */);
int glio_hf_marg_evaluate(void* user, int W, const double* poses, const double* speed_bias, double* A, double* b);
int glio_hf_marg_half_bandwidth(const glio_host_factor_set* s);

/* ---- K1b: scan-to-multiscan (batch) association.
 * Replaces findGlobalCorrespondingSurfFeatures_Batch / ...Add_Batch (Estimator.cpp:3710-3892) and their driver
 * batchFeatureAssociation (:3413-3432).  Frames (one keyframe's surf scan, stored as received + its pose from
 * pose_info_keyframe, quirks Q7/Q8) are registered once; a pair (cur, oth) associates every point of frame `cur`
 * against the world cloud of frame `oth`.  The uniform grid of a frame is built once and reused by every pair
 * that searches it (the reference rebuilds a kd-tree per pair, Estimator.cpp:3729-3731: same neighbours). */
int glio_batch_set_frame(glio_ctx* ctx, int frame, const float* scan_xyz, int64_t Q, int stride_floats, int mem,
                         const double pose[7]);
int glio_batch_set_pose(glio_ctx* ctx, int frame, const double pose[7]);
/* associate `cur` against each of oth[n_oth]; n_match[n_oth] receives gl_vec_surf_res_cnt[cur][oth]. */
int glio_batch_associate(glio_ctx* ctx, int cur, const int32_t* oth, int n_oth, int64_t* n_match);
/* many pairs at once (grouped by searched frame internally): pairs_cur[n], pairs_oth[n] */
int glio_batch_associate_pairs(glio_ctx* ctx, const int32_t* pairs_cur, const int32_t* pairs_oth, int64_t n_pairs,
                               int64_t* n_match);
/* matches of one pair: cp[3n] float (point of cur, local), weight[n] float (score = batch_score*weight),
 * normal_cent[6n] double (unit normal and centroid of the 5 neighbours in oth's LOCAL frame), src[n] */
int glio_batch_get_matches(glio_ctx* ctx, int cur, int oth, int64_t capacity, float* cp, float* weight,
                           double* normal_cent, int32_t* src, int64_t* n_match);
/* globalFeatureSelection_Batch (Estimator.cpp:3994-4116) as an input index list; n < 0 clears */
int glio_batch_select(glio_ctx* ctx, int cur, int oth, const int32_t* keep, int64_t n);
/* globalFeatureSelection_Batch (mode 0) / globalFeatureSelectionAdd_Batch (mode 1) over cur[n_pairs], oth[n_pairs], grouped by cur
 * and visited in list order (the reference visits ascending oth).  Mode 0: the first pair of a run with n - 1 < B or n < 50 and
 * every later pair of that run keep all their matches (the reference returns); mode 1: a pair with n <= B keeps all its matches
 * (continue).  Any other pair keeps its B sampled matches.  n_active[n_pairs] may be NULL.  GLIO_ERR_ARG, with nothing changed,
 * when a list is not grouped by cur, lists a pair twice, has cur == oth or a pair that was never associated, mode is not 0 / 1, or
 * an option is out of range. */
int glio_batch_select_random(glio_ctx* ctx, const int32_t* cur, const int32_t* oth, int64_t n_pairs, int mode,
                             const glio_select_options* options, int64_t* n_active);
int glio_batch_get_selection(glio_ctx* ctx, int cur, int oth, int64_t capacity, int32_t* keep, int64_t* n);
int glio_batch_pair_list(glio_ctx* ctx, int64_t capacity, int32_t* cur, int32_t* oth, int64_t* n_pairs);
int glio_batch_clear(glio_ctx* ctx);   /* also empties the pose-factor, DD-pseudorange and IMU lists (glio_batch_set_pose_factors,
                                          glio_batch_set_dd_psr_factors, glio_batch_set_imu_factors) */

/* Creates (empty) pair entries in the given order without associating them: on a keyframe-sharded multi-GPU run
 * every rank declares the SAME global pair list and then associates only the pairs it owns, so the block
 * buffers have one layout everywhere.  Every pair needs cur >= 0, oth >= 0 and cur != oth (the rule of
 * glio_batch_set_pair_matches), and n_pairs > 0 needs both arrays; otherwise the call returns GLIO_ERR_ARG and
 * leaves the pair list unchanged.  Pairs already declared are kept in place. */
int glio_batch_declare_pairs(glio_ctx* ctx, const int32_t* pairs_cur, const int32_t* pairs_oth, int64_t n_pairs);

/* Upload the matches of pair (cur, oth) instead of associating them (creates the pair when it does not exist yet) - the
 * path the Ceres-API shim takes for BinaryLidarPlaneNormFactor residual blocks, which carry their own data
 * (LidarKeyframeFactor.h:161-163: curr_point, planet_norm_cent, score = batch_score*weight). */
int glio_batch_set_pair_matches(glio_ctx* ctx, int cur, int oth, const float* cp, const double* normal_cent, const float* weight, int64_t n);

/* ---- K2b: evaluate all active binary plane residuals at poses[K*7].
 * Replaces ResidualBlock::Evaluate over BinaryLidarPlaneNormFactor (LidarKeyframeFactor.h:124-164; no loss function,
 * Estimator.cpp:2768) and the J^T J / J^T r accumulation.  Block-sparse output: Hdiag[K*36], Hoff[n_pairs*36]
 * (block (cur,oth): row = cur tangent, col = oth tangent, pairs in glio_batch_pair_list order), g[K*6], cost. */
int glio_eval_binary(glio_ctx* ctx, int K, const double* poses, double* Hdiag, double* Hoff, double* g, double* cost);

/* ---- K3: the marginalisation Schur step of MarginalizationInfo::Marginalize (GLIO/src/MarginalizationFactor.cpp:176-201),
 * host C++ (123 x 15 x 123 at W = 20: too small for the GPU to matter).  A[n_total x n_total] row-major and b[n_total]
 * are the dense normal equations with the m states to drop first (LiDAR part: glio_eval_unary with jac_kind = 1);
 * outputs linearized_jacobians[(n_total-m)^2] row-major and linearized_residuals[n_total-m].  eps = 1e-8 in the reference. */
int glio_marginalize(const double* A, const double* b, int n_total, int m, double eps, double* lin_jac, double* lin_res);

/* ---- K2e: point-to-edge residuals (LidarEdgeFactor, LidarKeyframeFactor.h:12-70).  The reference defines this factor
 * but never instantiates it and has no edge association (SURVEY fact 1), so the correspondences are an input:
 * cp[3n] scan point, pa/pb[3n] two points of the map line, s[n] weight.  Huber(huber_delta) as for the plane factors.
 * glio_eval_edge returns the same per-keyframe 6x6 / 6 / cost blocks as glio_eval_unary (add them to the plane blocks). */
int glio_set_edges(glio_ctx* ctx, int slot, const float* cp, const float* pa, const float* pb, const double* s, int64_t n);
int glio_eval_edge(glio_ctx* ctx, int W, const double* poses_body, double* H, double* g, double* cost);
/* The same blocks with jac_kind 0 (Ceres tangent rotation columns: identical to glio_eval_edge) or 1 (the ambient x,y,z quaternion
 * columns of MarginalizationFactor.cpp:9-17 with ResidualBlockInfo::Evaluate's Huber corrector: what the marginalisation uses). */
int glio_eval_edge_kind(glio_ctx* ctx, int W, const double* poses_body, int jac_kind, double* H, double* g, double* cost);
/* on != 0: every evaluation inside glio_window_solve, glio_window_solve_band, glio_window_marginalize and
 * glio_window_marginalize_async (Jacobian and cost-only alike) adds the edge blocks of slots 0..W-1 (glio_set_edges or
 * glio_window_associate_edges) to their plane blocks: tangent columns in the solve, ambient columns in the marginalisation.
 * Default off: those calls then ignore edges entirely.  The K2e work-item plan is rebuilt only when an edge list, the window or
 * this switch changes.  K2e is launched on the context's stream before K2, and its result is copied to pinned host memory
 * before K2 starts, so the host reads it after K2's completion flag and never earlier; the asynchronous marginalisation adds
 * it in the same place, so its prior stays bit-identical to the synchronous pass. */
int glio_window_use_edges(glio_ctx* ctx, int on);

/* ---- K1e: scan-to-map EDGE association on the device, producing K2e's inputs.  The reference defines LidarEdgeFactor but has
 * no association for it, so this library defines one (the LOAM-family line form); nothing in the reference pins it.  For each
 * corner point p of slot k, with the lidar->map pose (Q2, T2) of Estimator.cpp:2216-2217 formed from poses_body[k]:
 *   1. p_m = float(Q2 double(p) + T2), the transform and rounding of K1;
 *   2. the exact 5 nearest neighbours a_0..a_4 of p_m in the CORNER map (squared float distances ascending, ties by index: the
 *      K0 grid and K1's box search);
 *   3. status GLIO_EDGE_FAIL_RADIUS unless (double)sqd[4] < max_sqdist;
 *   4. centroid c = (a_0 + a_1 + a_2 + a_3 + a_4) / 5.0 in double, summed nearest first;
 *   5. scatter matrix C = sum_j (a_j - c)(a_j - c)^T in double, same order, not divided;
 *   6. eigen-decomposition of C by cyclic Jacobi: rotations (0,1), (0,2), (1,2) per sweep; rotation theta = (c_qq - c_pp) /
 *      (2 c_pq), t = sgn(theta) / (|theta| + sqrt(theta^2 + 1)) with sgn(0) = +1, c = 1 / sqrt(t^2 + 1), s = t c; an element with
 *      |c_ii| + 100 |c_pq| == |c_ii| for both i = p, q is zeroed without rotating; sweeps stop when all three off-diagonal elements
 *      are zero, at most 32 sweeps.  Eigenvalues lambda_0 <= lambda_1 <= lambda_2 (stable: ties by index); v = the eigenvector of
 *      lambda_2 with its largest-magnitude component (lowest index on ties) positive.  Only + - * / sqrt, round-to-nearest, no FMA;
 *   7. status GLIO_EDGE_FAIL_LINE unless lambda_2 > min_ratio * lambda_1 (five identical points fail, exactly collinear ones pass);
 *   8. otherwise GLIO_EDGE_VALID and, in scan order, cp = p (scan frame), pa = float(c + h v), pb = float(c - h v),
 *      s = (float)score, src = the index of p in the scan, h = half_length.
 * Eigen's SelfAdjointEigenSolver would give eigenvalues a few ulps away, so a ratio within a few ulps of min_ratio may decide the
 * other way there. */
typedef struct {
  double max_sqdist;    /* 1.0: gate on the squared 5th distance (m^2), > 0 */
  double min_ratio;     /* 3.0: line gate lambda_2 > min_ratio lambda_1, >= 0 */
  double half_length;   /* 0.1: pa, pb lie half_length (m) either side of the centroid, > 0 */
  double score;         /* 1.0: s of every edge residual */
} glio_edge_options;
void glio_edge_default_options(glio_edge_options* o);
/* The corner map: its own K0 grid, M >= 5 points (stride in [3,64], host or device memory as glio_set_map).  The surf map and its
 * grid are untouched. */
int glio_set_edge_map(glio_ctx* ctx, const float* xyz, int64_t M, int stride_floats, int mem);
/* The corner local map: a second local map of the context (the corner counterpart of glio_localmap_*, same semantics);
 * glio_edge_localmap_build makes it the corner map. */
int glio_edge_localmap_clear(glio_ctx* ctx);
int glio_edge_localmap_push(glio_ctx* ctx, int at_front, const float* cloud_xyz, int64_t n, int stride_floats, int mem,
                            const double t[3], const double q[4]);
int glio_edge_localmap_pop_front(glio_ctx* ctx);
int glio_edge_localmap_build(glio_ctx* ctx, float leaf, int64_t* n_map);
/* One keyframe's corner scan (e.g. glio_extract_features' less-sharp points) into one slot: host buffers travel on the copy
 * stream as with glio_window_set_scan.  glio_window_slide moves the corner scans and edges with their slots and leaves the
 * recycled last slot with neither. */
int glio_window_set_edge_scan(glio_ctx* ctx, int slot, const float* xyz, int64_t Q, int stride_floats, int mem);
/* Edge association of slots 0..W-1 against the corner map in one pass (launch count independent of W); each slot's edge list
 * (what glio_set_edges would upload, src included) is replaced, n_edge[W] (may be NULL) receives the counts.  options NULL = the
 * defaults.  One host synchronisation, for the counts.  Bad options are GLIO_ERR_ARG; no corner map, or a slot without a corner
 * scan, is GLIO_ERR_STATE; both change nothing. */
int glio_window_associate_edges(glio_ctx* ctx, int W, const double* poses_body, const glio_edge_options* options, int64_t* n_edge);
/* copy-out of a slot's edge list (any pointer may be NULL): cp/pa/pb[3n] float, s[n] double, src[n] int32 (-1 for edges uploaded
 * with glio_set_edges).  *n receives the count; all arrays NULL only counts, otherwise a capacity below the count is GLIO_ERR_ARG. */
int glio_get_edges(glio_ctx* ctx, int slot, int64_t capacity, float* cp, float* pa, float* pb, double* s, int32_t* src, int64_t* n);
/* per-query view of the slot's last edge association (needs params.keep_debug): status[Q] u8 (GLIO_EDGE_*), idx5[5Q] (-1: none),
 * sqd5[5Q], pm[3Q], eig[3Q] double (lambda ascending; 0 for GLIO_EDGE_FAIL_RADIUS). */
int glio_get_edge_debug(glio_ctx* ctx, int slot, int64_t Q, uint8_t* status, int32_t* idx5, float* sqd5, float* pm, double* eig);

/* ---- K1be / K2be: scan-to-multiscan EDGE association and binary point-to-edge factors in the batch solve.  The reference has
 * neither; this is the batch counterpart of K1e / K2e, written the way K1b / K2b extend K1 / K2.
 *
 * The corner scan of a batch frame already registered with glio_batch_set_frame (unknown frame: GLIO_ERR_STATE, nothing changes):
 * Q >= 0 points (0 to 4 are accepted: no pair that searches the frame gets an edge), stride in [3,64], host or device memory as
 * glio_batch_set_frame; stored as received, in the body frame (quirk Q7).  The frame's pose is the one of glio_batch_set_frame /
 * glio_batch_set_pose; both drop the corner grid as they drop the surf grid, and glio_batch_clear releases it. */
int glio_batch_set_edge_frame(glio_ctx* ctx, int frame, const float* xyz, int64_t Q, int stride_floats, int mem);
/* K1be: edge association of the pairs (cur[i], oth[i]).  For every corner point p of frame cur, with (t_c, q_c) cur's pose:
 *   1. p_w = float(R(q_c) double(p) + t_c): K1b's transform, the body pose applied directly;
 *   2. the exact 5 nearest neighbours of p_w in oth's corner cloud moved by oth's pose (the same transform), on its own K0 grid,
 *      built once and reused by every pair that searches oth until oth's pose or corner scan changes;
 *   3.-7. steps 3-7 of K1e on those five world points: the gate (double)sqd[4] < max_sqdist, the centroid, the scatter matrix, the
 *      cyclic Jacobi and the line gate lambda_2 > min_ratio lambda_1 (status GLIO_EDGE_FAIL_RADIUS / GLIO_EDGE_FAIL_LINE);
 *   8. for a valid query, steps 4-6 again on the same five indices in oth's LOCAL coordinates as stored (no gate on that fit; the
 *      pair plane fit refits its plane the same way, Estimator.cpp:3752-3772), giving c_l and v_l; then, in scan order,
 *      cp = p, pa = float(c_l + h v_l), pb = float(c_l - h v_l) (oth's frame), s = (float)score, src = the index of p in cur's scan.
 * The arithmetic rules of K1e hold (only + - * / sqrt, round-to-nearest, no FMA).  Each pair's edge list is replaced; a pair not on
 * the pair list yet is appended, with no plane matches (as glio_batch_set_pair_matches appends one).  Pairs are grouped by oth: one
 * search launch and one host synchronisation (for the counts) per group, besides the grid build's own when oth's grid is built.
 * n_edge[n_pairs] (may be NULL) receives the counts.  options NULL = the defaults.  An unknown frame, cur == oth or bad options is
 * GLIO_ERR_ARG, a cur or oth without a corner scan is GLIO_ERR_STATE; both change nothing.  The plane selection calls
 * (glio_batch_select*) leave edge lists alone; glio_batch_select_random_edges selects edges.  Without an edge selection all edges of
 * a pair are evaluated. */
int glio_batch_associate_edges_pairs(glio_ctx* ctx, const int32_t* cur, const int32_t* oth, int64_t n_pairs, const glio_edge_options* options,
                                     int64_t* n_edge);
/* copy-out of the edge list of pair (cur, oth), the conventions of glio_get_edges (pa / pb in oth's frame); a pair not on the pair
 * list is GLIO_ERR_ARG */
int glio_batch_get_edges(glio_ctx* ctx, int cur, int oth, int64_t capacity, float* cp, float* pa, float* pb, double* s, int32_t* src,
                         int64_t* n);
/* upload of the edge list of pair (cur, oth) (appended to the pair list if needed), as glio_set_edges: cp[3n] in cur's frame,
 * pa/pb[3n] in oth's frame, s[n] (stored as float); src reads back as -1 */
int glio_batch_set_pair_edges(glio_ctx* ctx, int cur, int oth, const float* cp, const float* pa, const float* pb, const double* s, int64_t n);
/* K2be, the binary point-to-edge factor, with the conventions of BinaryLidarPlaneNormFactor (no extrinsic, the line moves with oth,
 * no loss, Estimator.cpp:2768):
 *   p_w = R(q_c) cp + t_c,  A = R(q_o) pa + t_o,  B = R(q_o) pb + t_o,  e = (p_w - A) x (p_w - B),  r = s |e| / |A - B|;
 *   g = s / |A - B| ((A - B) x e / |e|),  J_c = [g | 2 (R(q_c) cp x g)],  J_o = [-g | 2 (g x (p_w - t_o))]  (tangent columns).
 * A point exactly on its line (|e| = 0) is treated as by K2e: r = 0 and non-finite Jacobian entries.
 * glio_eval_binary_edge returns the edge blocks alone in glio_eval_binary's layout and pair order (with the all-reduce hook, if set,
 * as glio_eval_binary). */
int glio_eval_binary_edge(glio_ctx* ctx, int K, const double* poses, double* Hdiag, double* Hoff, double* g, double* cost);
/* on != 0: every evaluation inside glio_batch_solve (Jacobian and cost-only alike) adds the pairs' edge blocks: each pair's sums are
 * S_plane + S_edge, each summed in item order, before the one block assembly, so a sharded run makes the same all-reduce calls as
 * without edges.  Default off: glio_batch_solve then launches what it launches without edges; so it does when no pair has an edge.
 * glio_eval_binary never includes edges.  The edge work-item plan is rebuilt only when an edge list, K, the pair count or this
 * switch changes. */
int glio_batch_use_edges(glio_ctx* ctx, int on);

/* ---- K2p: the batch refinement's pose factors (optimizeBatchWithLandMark, Estimator.cpp:2831-2954), evaluated on the device.
 *   GLIO_POSE_RELATIVE (LidarPoseFactorBatchRelativeAutoDiff, blocks t_i, q_i, t_j, q_j, 6 rows, no loss):
 *     r[0..2] = 10 (2 vec(dq^-1 q_i^-1 q_j)),  r[3..5] = 20 (q_i^-1 (t_j - t_i) - dp)
 *   GLIO_POSE_DELTA_Q (delta_q_factor_auto, blocks q_i, q_j, 3 rows, no loss):  r = 10000 vec(dq^-1 q_i^-1 q_j)
 * with Eigen's semantics at any quaternion: q^-1 = conj(q) / |q|^2 (0 for q = 0), q v = v + 2w (u x v) + 2 u x (u x v).  dq is
 * (w, x, y, z); dp is read by the relative kind only.  The Jacobian columns are the tangent columns of Ceres'
 * QuaternionParameterization (ambient Jacobian times its 4 x 3 local Jacobian at the current q) and the translation columns.
 * The weights are the reference's, fixed per kind.  active = 0: the factor is not evaluated by this context, but it still makes
 * its pair entry, so keyframe-sharded ranks that pass one list with their own active masks share one pair layout. */
enum { GLIO_POSE_RELATIVE = 0, GLIO_POSE_DELTA_Q = 1 };
/* keyframe indices of a pose factor are < GLIO_POSE_MAX_KF (the host plan holds one incidence start per keyframe up to the largest) */
enum { GLIO_POSE_MAX_KF = 1 << 22 };
typedef struct { int32_t i, j, kind, active; double dq[4]; /* w,x,y,z */ double dp[3]; } glio_pose_factor;
/* Replaces the pose-factor list (n = 0 empties it; glio_batch_clear empties it too).  The whole list is checked first (i != j, both
 * in [0, GLIO_POSE_MAX_KF), a known kind; f may be NULL only when n = 0); a refused call (GLIO_ERR_ARG) leaves the previous list in place.  The
 * distinct unordered pairs (a, b), a = min(i, j) < b, form the pose-pair table in order of first appearance.  Device buffers are
 * allocated and filled here, and the context takes the new list only once they are complete: a call that fails for any reason
 * leaves the previous list in place.  Evaluations allocate nothing for the list. */
int glio_batch_set_pose_factors(glio_ctx* ctx, const glio_pose_factor* f, int64_t n);
/* the pose-pair table (a[k] < b[k]), glio_batch_pair_list's conventions: NULL arrays only count */
int glio_batch_pose_pair_list(glio_ctx* ctx, int64_t capacity, int32_t* a, int32_t* b, int64_t* n_pairs);
/* The pose blocks alone, for the active factors: Hdiag[K*36] (per keyframe 6 x 6 over (t, delta)), Hoff[n_pose_pairs*36]
 * (block k = d2 cost / d x_a d x_b of pose pair k, rows for a), g[K*6], cost (attributed to a); NULL outputs are skipped and
 * without Hdiag, Hoff and g only the cost is formed.  Per pair the factors are summed in list order, per keyframe the pairs in
 * table order.  With the all-reduce hook set, the K x 28 and n_pose_pairs x 36 buffers are summed over the ranks, as in
 * glio_eval_binary.  A list that references a keyframe >= K is GLIO_ERR_ARG. */
int glio_eval_pose_factors(glio_ctx* ctx, int K, const double* poses, double* Hdiag, double* Hoff, double* g, double* cost);
/* on != 0: every evaluation inside glio_batch_solve adds the pose blocks of the active factors to the LiDAR pair blocks, before the
 * all-reduce: a sharded run then sums K x 28 and (P + P_pose) x 36 doubles, one call per buffer.  The band's half bandwidth covers
 * the pose pairs' span, and the solve works with no LiDAR pair at all (the reference's sms_fusion_level 0 problem).  Default off;
 * with the switch off or an empty list glio_batch_solve launches what it launches without pose factors.  A list that references
 * a keyframe >= K makes glio_batch_solve return GLIO_ERR_ARG.  glio_eval_binary and glio_eval_binary_edge never add pose blocks. */
int glio_batch_use_pose_factors(glio_ctx* ctx, int on);

/* ---- K2g: the batch refinement's double-differenced pseudorange factors (dd_psr_factor_20, added per epoch and constellation by
 * optimizeBatchWithLandMark through addDDPsrResFactor_gl, Estimator.cpp:3086-3272 and :1902-1913), evaluated on the device.
 * Per list: R = R_ecef_local (row-major 3 x 3) = ecef2rotation(anchor) * R_enu_local(yaw), and anchor = anchor_ecef; the caller
 * forms R once, since the yaw and anchor blocks are constant in the batch.  Per factor: keyframes i != j, ratio, threshold,
 * station (the factor's Station_pos), n_sat satellites (2 <= n_sat <= GLIO_DD_PSR_MAX_SAT: the reference's fixed buffer holds 19
 * rows) at sats[sat_offset .. sat_offset + n_sat), the master 0 <= master < n_sat, and a dense row-major (n_sat-1) x (n_sat-1)
 * weight W at W[w_offset ..], or w_offset = -1 for identity (the batch passes identity).  Rows k = 0 .. n_sat-2 belong to the
 * satellites s != master in index order:
 *   local = ratio t_i + (1 - ratio) t_j,  P = R local + anchor
 *   e_k = (|sat_user_s - P| - |sat_ref_s - station|) - (|sat_user_m - P| - |sat_ref_m - station|)
 *         - ((psr_user_s - psr_ref_s) - (psr_user_m - psr_ref_m))
 *   w_k = 0.05 if |e_k| > threshold else 1 (strict, on the raw residual, before W),  r_k = w_k e_k
 *   J_i row k = (-u_s^T R w_k ratio) - (-u_m^T R w_k ratio),  J_j row k the same with (1 - ratio),  u = normalized(sat_user - P)
 *   r = W r_raw,  J = W J_raw,  cost = 0.5 |r|^2 (no loss function)
 * normalized() is Eigen 3.3's: v / |v| when |v|^2 > 0, else v itself (the zero vector for a zero-length line of sight).  Only the
 * t columns of the (t, delta) keyframe layout are non-zero.  The threshold is the factor's own: the reference sets it per outer
 * pass from {1e9, 10, 8, 6}.  active = 0: as for the pose factors, the factor makes its pair entry but is not evaluated here. */
enum { GLIO_DD_PSR_MAX_SAT = 20, GLIO_DD_PSR_MAX_KF = 1 << 22 };
typedef struct {
  int32_t i, j, n_sat, master, active, reserved;   /* reserved: 0 */
  int64_t sat_offset, w_offset;                    /* w_offset = -1: identity */
  double ratio, threshold, station[3];
} glio_dd_psr_factor;
typedef struct { double sat_user[3], sat_ref[3], psr_user, psr_ref; } glio_dd_psr_sat;
/* Replaces the DD-pseudorange list (n = 0 empties it; glio_batch_clear empties it too).  The whole list is checked first: i != j,
 * both in [0, GLIO_DD_PSR_MAX_KF), 2 <= n_sat <= GLIO_DD_PSR_MAX_SAT, 0 <= master < n_sat, the satellites inside [0, n_sats), the
 * weight inside [0, n_w) or w_offset = -1, and R_ecef_local and anchor_ecef given when n > 0; a refused call (GLIO_ERR_ARG) leaves
 * the previous list in place.  The distinct unordered pairs (a, b), a = min(i, j) < b, form the DD pair table in order of first
 * appearance.  The list, the satellites and the weights are copied to device buffers allocated here; the context takes them only
 * once complete, so a call that fails for any reason leaves the previous list in place.  Evaluations allocate nothing for it. */
int glio_batch_set_dd_psr_factors(glio_ctx* ctx, const glio_dd_psr_factor* f, int64_t n, const glio_dd_psr_sat* sats, int64_t n_sats,
                                  const double* W, int64_t n_w, const double* R_ecef_local, const double* anchor_ecef);
/* the DD pair table (a[k] < b[k]), glio_batch_pair_list's conventions: NULL arrays only count */
int glio_batch_dd_psr_pair_list(glio_ctx* ctx, int64_t capacity, int32_t* a, int32_t* b, int64_t* n_pairs);
/* The DD blocks alone, for the active factors, in glio_eval_pose_factors' layout: Hdiag[K*36], Hoff[n_dd_pairs*36] (rows for a),
 * g[K*6], cost (attributed to a); NULL outputs are skipped and without Hdiag, Hoff and g only the cost is formed.  Per pair the
 * factors are summed in list order, per keyframe the pairs in table order.  With the all-reduce hook set, the K x 28 and
 * n_dd_pairs x 36 buffers are summed over the ranks.  A list that references a keyframe >= K is GLIO_ERR_ARG. */
int glio_eval_dd_psr_factors(glio_ctx* ctx, int K, const double* poses, double* Hdiag, double* Hoff, double* g, double* cost);
/* on != 0: every evaluation inside glio_batch_solve adds the DD blocks of the active factors before the all-reduce.  The
 * off-diagonal buffer holds the LiDAR pairs, then the pose pairs (glio_batch_use_pose_factors on), then the DD pairs: a sharded run
 * sums K x 28 and (P + P_pose + P_dd) x 36 doubles, one call per buffer.  The band's half bandwidth covers the DD pairs' span, and
 * the solve works with no LiDAR pair.  Default off; with the switch off or an empty list glio_batch_solve launches what it launches
 * without DD factors.  A list that references a keyframe >= K makes glio_batch_solve return GLIO_ERR_ARG.  glio_eval_binary,
 * glio_eval_binary_edge and glio_eval_pose_factors never add DD blocks. */
int glio_batch_use_dd_psr_factors(glio_ctx* ctx, int on);

/* ---- K2i: the batch refinement's IMU factors (ImuFactor between consecutive keyframes at sms_fusion_level 1,
 * Estimator.cpp:2993-3001), evaluated on the device from the caller's pre-integration: the library integrates no IMU samples
 * and inverts no covariance.  Per factor, with T = sum_dt, g = g_vec, Q_i and Q_j normalised (Eigen's normalize()), q^-1 =
 * conj(q) / |q|^2, q v Eigen's rotation, deltaQ(theta) = (1, theta / 2) (not normalised), and the speed-bias state
 * SB = [V(3), Ba(3), Bg(3)]:
 *   dba = Ba_i - linearized_ba,  dbg = Bg_i - linearized_bg,  cdq = delta_q deltaQ(dq_dbg dbg)
 *   cdp = delta_p + dp_dba dba + dp_dbg dbg,  cdv = delta_v + dv_dba dba + dv_dbg dbg
 *   r_P = Q_i^-1 (-g T^2 / 2 + P_j - P_i - V_i T) - cdp,  r_R = 2 vec(normalized(cdq^-1 (Q_i^-1 Q_j)))
 *   r_V = Q_i^-1 (-g T + V_j - V_i) - cdv,  r_BA = Ba_j - Ba_i,  r_BG = Bg_j - Bg_i
 *   r = sqrt_info r_raw,  cost = |r|^2 / 2 (no loss function)
 * The Jacobian is ImuFactor's analytic one, which is not the exact derivative of r (its rotation rows, its bias columns and the
 * missing normalisation term are kept as written), each column multiplied by sqrt_info.  The quaternion columns are its ambient
 * 15 x 4 blocks times Ceres' QuaternionParameterization local Jacobian at the unnormalised parameter q.  Tangent order per
 * keyframe: [t(3), delta(3), v(3), ba(3), bg(3)], glio_batch_solve's 15 columns with speed-bias.  active = 0: as for the pose
 * factors, the factor makes its pair entry but is not evaluated here.  sqrt_info is what ImuFactor forms from the covariance,
 * LLT(covariance.inverse()).matrixL().transpose(); the jacobian_ blocks and sqrt_info are row-major. */
enum { GLIO_IMU_MAX_KF = 1 << 22 };
typedef struct {
  int32_t i, j, active, reserved;                 /* reserved: 0 */
  double sum_dt, g_vec[3];
  double delta_p[3], delta_q[4] /* w,x,y,z */, delta_v[3];
  double linearized_ba[3], linearized_bg[3];
  double dp_dba[9], dp_dbg[9], dq_dbg[9], dv_dba[9], dv_dbg[9];
  double sqrt_info[225];
} glio_imu_factor;
/* Replaces the IMU list (n = 0 empties it; glio_batch_clear empties it too).  The whole list is checked first: i != j, both in
 * [0, GLIO_IMU_MAX_KF), every double finite, f given when n > 0; a refused call (GLIO_ERR_ARG) leaves the previous list in place.
 * The distinct unordered pairs (a, b), a = min(i, j) < b, form the IMU pair table in order of first appearance.  The list is
 * copied to device buffers allocated here; the context takes them only once complete, so a call that fails for any reason leaves
 * the previous list in place.  Evaluations allocate nothing for it. */
int glio_batch_set_imu_factors(glio_ctx* ctx, const glio_imu_factor* f, int64_t n);
/* the IMU pair table (a[k] < b[k]), glio_batch_pair_list's conventions: NULL arrays only count */
int glio_batch_imu_pair_list(glio_ctx* ctx, int64_t capacity, int32_t* a, int32_t* b, int64_t* n_pairs);
/* The IMU blocks alone, for the active factors, at poses[K*7] and speed_bias[K*9] (both required): Hdiag[K*225] (per keyframe
 * 15 x 15, row-major), Hoff[n_imu_pairs*225] (block k = d2 cost / d x_a d x_b of IMU pair k, rows for a), g[K*15], cost
 * (attributed to a); NULL outputs are skipped and without Hdiag, Hoff and g only the cost is formed.  Per pair the factors are
 * summed in list order, per keyframe the pairs in table order.  With the all-reduce hook set, the K x 241 (Hdiag, g, cost) and
 * n_imu_pairs x 225 buffers are summed over the ranks.  A list that references a keyframe >= K is GLIO_ERR_ARG. */
int glio_eval_imu_factors(glio_ctx* ctx, int K, const double* poses, const double* speed_bias, double* Hdiag, double* Hoff, double* g,
                          double* cost);
/* on != 0: every evaluation inside glio_batch_solve adds the IMU blocks of the active factors into the 15-column band, after the
 * LiDAR, pose and DD blocks.  The speed-bias states are uploaded with the poses at every evaluation; a sharded run sums the IMU
 * buffers (K x 241, then n_imu_pairs x 225) after the others, one call per buffer.  The band's half bandwidth covers the IMU pairs'
 * span, and the solve works with no LiDAR pair.  Default off; with the switch off or an empty list glio_batch_solve launches what it
 * launches without IMU factors.  With the switch on and a non-empty list, speed_bias == NULL or a list that references a keyframe
 * >= K makes glio_batch_solve return GLIO_ERR_ARG.  The other glio_eval_* calls never add IMU blocks. */
int glio_batch_use_imu_factors(glio_ctx* ctx, int on);

/* ---- K2i in the sliding window: the window problem's IMU chain (Estimator.cpp:2179-2193: ImuFactor(pre_integrations[idx+1])
 * between window slots), with the factor, the record and the Jacobian described above.  The window keeps its own list, separate
 * from the batch one: glio_batch_clear and glio_batch_set_imu_factors leave it alone, and this list's calls leave the batch list
 * alone.  i and j are window slots.  glio_window_slide leaves the list as it is: the reference builds a new problem per window, so
 * a caller sets a new list for each window. */
/* Replaces the window IMU list (n = 0 empties it).  The whole list is checked first: i != j, both in [0, 4096) (the window's
 * size cap), every double finite; a refused or failed call leaves the previous list in place. */
int glio_window_set_imu_factors(glio_ctx* ctx, const glio_imu_factor* f, int64_t n);
/* the window IMU pair table (a[k] < b[k]), glio_batch_pair_list's conventions */
int glio_window_imu_pair_list(glio_ctx* ctx, int64_t capacity, int32_t* a, int32_t* b, int64_t* n_pairs);
/* The window IMU blocks alone at poses[W*7] and speed_bias[W*9], in glio_eval_imu_factors' layout.  jac_kind 0: the tangent
 * columns; 1: the quaternion columns are the ambient x, y, z columns of the 15 x 4 blocks (ImuFactor.h:77-100 and :139-150,
 * rightCols(3), times sqrt_info), what the marginalisation reads.  No all-reduce.  A list that references a slot >= W is
 * GLIO_ERR_ARG. */
int glio_eval_window_imu_factors(glio_ctx* ctx, int W, const double* poses, const double* speed_bias, int jac_kind, double* Hdiag,
                                 double* Hoff, double* g, double* cost);
/* on != 0 with a non-empty list:
 * - glio_window_solve and glio_window_solve_band: every evaluation uploads the speed-bias states and queues K2i (tangent columns)
 *   and the copy of its blocks on the main stream ahead of K2; the host adds the 15 x 15 diagonal and pair blocks into the band at
 *   15 columns per keyframe, after the LiDAR blocks and the callback's factors.  The band covers the IMU pairs' span (29 for a
 *   chain) in both forms of the solve.  speed_bias == NULL or a list slot >= W is GLIO_ERR_ARG.  A window with no LiDAR match
 *   still solves.
 * - glio_window_marginalize and glio_window_marginalize_async: the device half also queues K2i with the ambient columns over
 *   the active factors of pair {0, 1} (KF0 -> KF1, Estimator.cpp:2520-2534) ahead of K2; the host half adds that pair's 30 x 30
 *   block and 30-vector into A and b at the marginalisation ordering (KF0 [0, 15), KF1 [15, 30)), after host_marg's factors.
 *   Factors that do not touch slot 0 take no part; an active factor between slot 0 and a slot other than 1 is GLIO_ERR_ARG.
 *   The synchronous and asynchronous priors are the same bit for bit.
 * Default off; with the switch off or an empty list the solve and the marginalisation launch what they launch without it. */
int glio_window_use_imu_factors(glio_ctx* ctx, int on);

/* ---- seeded device selection of EDGE correspondences.  The reference selects plane matches only; this library applies the same
 * rules and the same sampler (glio_select_random / glio_batch_select_random, k_sel_sample) to edge lists, with the sizes of a
 * glio_select_options passed to these calls, so edge sizes are set independently of plane sizes:
 *   window (glio_select_random_edges): featureSelection's rule on the slot's edge count n: keep all edges when n < 1 or n - 1 < F,
 *     none when random_select is 0, else the F sampled edges in draw order;
 *   batch mode 0 (start/end): the run rule of glio_batch_select_random on edge counts (n - 1 < B or n < 50 ends the run of its cur,
 *     whose later pairs keep all their edges); mode 1 (incremental): keep all edges when n <= B, else sample B.
 * Draws as for plane matches, from positions 0 .. n-2: the last edge of a list is never chosen.  That quirk of the reference's plane
 * selection is carried over on purpose, so that one kernel and one reference serve both.  Philox domains: 3 window edges, 4 batch
 * start/end edges, 5 batch incremental edges; the streams are those of the plane calls (the keyframe id per slot, cur << 32 | oth
 * per pair), so an edge sample is independent of the plane sample with the same seed, stream and nonce, and a sharded run selects
 * what one context selects.  One k_sel_sample launch per call, no stream synchronisation (as the plane calls).
 * Every consumer of an edge list evaluates its active edges: the selected subset in draw order if there is one, else all edges --
 * glio_eval_edge / glio_eval_edge_kind, the edge blocks of glio_window_solve, glio_window_solve_band, glio_window_marginalize and
 * glio_window_marginalize_async, glio_eval_binary_edge and the edge blocks of glio_batch_solve.  glio_get_edges / glio_batch_get_edges
 * return the full list.  Replacing a list (glio_set_edges, glio_window_associate_edges, glio_batch_associate_edges_pairs,
 * glio_batch_set_pair_edges, glio_batch_clear) drops its selection; glio_window_slide moves a selection with its slot and leaves the
 * recycled last slot with none.  Plane selection calls leave edge selections alone, and these calls leave plane matches, plane
 * selections and the plane evaluations alone.  n_active (may be NULL) receives the active edge counts.  The batch call returns
 * GLIO_ERR_ARG, with nothing changed, on the cases glio_batch_select_random refuses; the window call on bad W, stream_ids or
 * options. */
int glio_select_random_edges(glio_ctx* ctx, int W, const int64_t* stream_ids, const glio_select_options* options, int64_t* n_active);
int glio_batch_select_random_edges(glio_ctx* ctx, const int32_t* cur, const int32_t* oth, int64_t n_pairs, int mode,
                                   const glio_select_options* options, int64_t* n_active);
/* The selected edge indices of a slot / pair in draw order, with glio_get_selection's conventions: *n = -1 when all edges are
 * active; a pair not on the pair list is GLIO_ERR_ARG. */
int glio_get_edge_selection(glio_ctx* ctx, int slot, int64_t capacity, int32_t* keep, int64_t* n);
int glio_batch_get_edge_selection(glio_ctx* ctx, int cur, int oth, int64_t capacity, int32_t* keep, int64_t* n);

/* ---- batch minimizer (replaces ceres::Solve of optimizeBatchWithLandMark, Estimator.cpp:3275-3284: SUBSPACE_DOGLEG,
 * nonmonotonic steps, max_num_iter iterations; options == NULL selects exactly those).  The normal equations are
 * block-banded (half bandwidth (max|cur-oth|+1)*nt - 1) and stored/factored in band form.  Host factors (IMU chain, prior;
 * the pose factors run on the device through glio_batch_use_pose_factors, the DD pseudorange factors through
 * glio_batch_use_dd_psr_factors, the IMU factors through glio_batch_use_imu_factors) accumulate into the same LOWER-BAND storage:
 * entry (i,j), i-hb <= j <= i, lives at Hband[i*(hb+1) + (j-i+hb)]. */
int glio_hf_evaluate_band(void* user, int K, const double* poses, const double* speed_bias, int want_jac, double* Hband, int hb,
                          double* g, double* cost);
int glio_batch_solve(glio_ctx* ctx, int K, double* poses, double* speed_bias, glio_host_factors_band_fn host_factors, void* user,
                     const glio_solver_options* options, glio_solver_summary* summary, glio_iteration* iter_log, int iter_cap,
                     double* step_log, int64_t step_cap);

/* on != 0: every glio_batch_solve on this context runs the minimizer's band algebra on the device.  Each Jacobian evaluation
 * uploads the host callback's band (a zeroed band with the usual contract; none when host_factors is NULL) and gathers the device
 * blocks onto it (k_band_assemble, each entry in the host path's order, so the band is the host path's bit for bit); the Jacobi
 * scaling, the shifted factor-and-solve (K4, below) and the band products run on the device, and only n-vectors cross PCIe.
 * The back-substitution and the band product sum in another order than the host's, so results differ from the host path by
 * rounding.  Needs a half bandwidth <= GLIO_BAND_MAX_HB (GLIO_ERR_ARG otherwise).  Default off: glio_batch_solve then runs exactly
 * the host path.  Kernel names for glio_profile_get: k_band_assemble, k_band_assemble_g, k_band_scale, k_band_shift, k_band_symv. */
int glio_batch_use_device_solver(glio_ctx* ctx, int on);
/* The batch normal equations at one state: the band (n x (hb+1), n = K * (speed_bias ? 15 : 6), capacity >= n * (hb+1) doubles),
 * *hb, g (n) and the cost, assembled by the host path (on_device = 0) or by k_band_assemble (on_device != 0), with the switches and
 * lists glio_batch_solve would use.  A failing callback or a non-finite cost is GLIO_ERR_NUMERIC. */
int glio_batch_normal_equations(glio_ctx* ctx, int K, const double* poses, const double* speed_bias, glio_host_factors_band_fn host_factors,
                                void* user, int on_device, int64_t capacity, double* Hband, int* hb, double* g, double* cost);

/* ---- K4: the band Cholesky factor-and-solve on the device, one system at a time.  band[n*(hb+1)] holds the lower band of a
 * symmetric A in glio_batch_solve's layout (entry (i,j), i-hb <= j <= i, at band[i*(hb+1) + (j-i+hb)]); on return it holds L,
 * A = L L^T, in the same layout, and x[n] solves A x = b.  Slots of the layout with j < 0 are left as they are.  The factor and
 * the forward half follow the scalar host band Cholesky's operation order (right-looking, updates in ascending column order, one
 * 1.0 / l per column), so L is bit-identical to it; the backward substitution is in axpy form over descending rows, so x differs
 * from the host's by rounding.  *ok = 1 on success; *ok = 0 when a pivot is not positive and finite or x is not finite (the
 * host's LINEAR_SOLVER_FAILURE), and then band and x hold partial results.  Bad arguments, and 0 > hb or hb > GLIO_BAND_MAX_HB
 * (the shared-memory window of one thread block), are GLIO_ERR_ARG.  Host buffers in and out; the call returns when x and *ok
 * have arrived.  Kernel name for glio_profile_get: k_band_chol_solve. */
enum { GLIO_BAND_MAX_HB = 160 };
int glio_band_solve(glio_ctx* ctx, int n, int hb, double* band, const double* b, double* x, int* ok);
/* The device minimizer's three small band passes on host buffers, in the order a solve uses them: Hs = S H S (entry (i,j) is
 * (H_ij * s_i) * s_j) and hs_diag = diag(Hs); A = Hs + diag(v * v); y = Hs x, per row the columns max(0, i-hb) .. i from row i and
 * then i+1 .. min(n-1, i+hb) from the rows below, each term one rounded product and one rounded sum, starting from 0.0.  H, Hs
 * and A are n x (hb+1) in glio_band_solve's layout; s, v, x, hs_diag and y have n entries.  H's slots with j < 0 are never read,
 * and those of Hs and A are left unspecified.  Same argument checks as glio_band_solve.  Kernel names for glio_profile_get:
 * k_band_scale, k_band_shift, k_band_symv. */
int glio_band_ops(glio_ctx* ctx, int n, int hb, const double* H, const double* s, const double* v, const double* x, double* Hs,
                  double* hs_diag, double* A, double* y);

/* ---- multi-GPU (batch path only; the window path is "replicas only", SURVEY 8e).
 * Keyframe-sharded ranks sum their pose-block buffers once per evaluation.  The library does not link NCCL: the
 * caller installs the reduction (in-place sum over ranks of count doubles at device pointer d_buf, enqueued on
 * `cuda_stream`).  glio_b200/libglio_nccl.so provides glio_nccl_allreduce for an ncclComm_t; Python callers may
 * install a torch.distributed-based hook instead. */
typedef int (*glio_allreduce_fn)(void* user, double* d_buf, int64_t count, void* cuda_stream);
int glio_set_allreduce(glio_ctx* ctx, glio_allreduce_fn fn, void* user);

#ifdef __cplusplus
}
#endif
#endif
