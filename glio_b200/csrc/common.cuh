// common.cuh — shared device/host declarations of the glio_b200 CUDA library (sm_90a).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include <algorithm>
#include <cmath>
#include <cstring>
#include <deque>
#include <memory>
#include <string>
#include <vector>

#include "../../include/glio_b200.h"

namespace glio {

// SMs of an H100 SXM: the grid size of the grid-stride kernels is a multiple of it (a tuning choice, not a correctness one)
constexpr int kNumSMs = 132;

// ----------------------------------------------------------------------------------------------
// error plumbing: every CUDA call is checked; failures become a status + message, never abort.
// ----------------------------------------------------------------------------------------------
struct Error {
  int code;
  std::string msg;
};

#define GLIO_CUDA_TRY(expr)                                                                   \
  do {                                                                                        \
    cudaError_t _e = (expr);                                                                  \
    if (_e != cudaSuccess) {                                                                  \
      char _b[512];                                                                           \
      snprintf(_b, sizeof(_b), "%s:%d: %s -> %s", __FILE__, __LINE__, #expr, cudaGetErrorString(_e)); \
      throw ::glio::Error{GLIO_ERR_CUDA, _b};                                                 \
    }                                                                                         \
  } while (0)

#define GLIO_REQUIRE(cond, code, text)                      \
  do {                                                      \
    if (!(cond)) throw ::glio::Error{(code), (text)};       \
  } while (0)

// grow-only device buffer that owns its memory: freed on destruction, moved but never copied (a copy would free it twice)
template <class T>
struct DevBuf {
  T* p = nullptr;
  size_t cap = 0;
  DevBuf() = default;
  DevBuf(const DevBuf&) = delete;
  DevBuf& operator=(const DevBuf&) = delete;
  DevBuf(DevBuf&& o) noexcept : p(o.p), cap(o.cap) { o.p = nullptr; o.cap = 0; }
  DevBuf& operator=(DevBuf&& o) noexcept {
    if (this != &o) { release(); p = o.p; cap = o.cap; o.p = nullptr; o.cap = 0; }
    return *this;
  }
  ~DevBuf() { release(); }
  void reserve(size_t n) {
    if (n <= cap) return;
    if (p) GLIO_CUDA_TRY(cudaFree(p));
    p = nullptr; cap = 0;
    size_t want = n + n / 8 + 64;
    GLIO_CUDA_TRY(cudaMalloc((void**)&p, want * sizeof(T)));
    cap = want;
  }
  void release() { if (p) cudaFree(p); p = nullptr; cap = 0; }   // result ignored: runs in the destructor, which must not throw
};

// the same for page-locked host memory
template <class T>
struct PinnedBuf {
  T* p = nullptr;
  size_t cap = 0;
  PinnedBuf() = default;
  PinnedBuf(const PinnedBuf&) = delete;
  PinnedBuf& operator=(const PinnedBuf&) = delete;
  PinnedBuf(PinnedBuf&& o) noexcept : p(o.p), cap(o.cap) { o.p = nullptr; o.cap = 0; }
  PinnedBuf& operator=(PinnedBuf&& o) noexcept {
    if (this != &o) { release(); p = o.p; cap = o.cap; o.p = nullptr; o.cap = 0; }
    return *this;
  }
  ~PinnedBuf() { release(); }
  void reserve(size_t n) {
    if (n <= cap) return;
    if (p) GLIO_CUDA_TRY(cudaFreeHost(p));
    p = nullptr; cap = 0;
    size_t want = n + n / 8 + 64;
    GLIO_CUDA_TRY(cudaMallocHost((void**)&p, want * sizeof(T)));
    cap = want;
  }
  void release() { if (p) cudaFreeHost(p); p = nullptr; cap = 0; }   // result ignored, as above
};

// ----------------------------------------------------------------------------------------------
// Uniform grid over a point cloud (K0 output).  Points are counting-sorted by cell with x the
// fastest-varying cell coordinate, so the three x-adjacent cells of a (y,z) row are ONE contiguous range.
// pts[k] = (x, y, z, bitcast(original index)).
// ----------------------------------------------------------------------------------------------
struct GridDesc {
  float ox, oy, oz;     // origin (min corner of cell (0,0,0))
  float cell, inv_cell;
  // margin (metres) the kNN face tests take off a float face distance before they call a face closed: a point that
  // cell_coord puts beyond a face can lie up to a few float spacings of the grid's coordinates nearer than the face
  // as computed (grid_build)
  float slack;
  int nx, ny, nz;
  int64_t npts;
  const int* cell_start;   // [nx*ny*nz + 1]
  const float4* pts;       // [npts] sorted by cell
};

// One association segment = one scan transformed by one pose, queried against the launch's grid.
struct SegDesc {
  const float* src;     // scan points, stride floats apart
  int stride;
  int64_t count;
  int64_t offset;       // first global query index of the segment
  double t[3];
  double q[4];
};

struct AssocGates {
  double max_radius;    // compared with the squared 5th distance (quirk Q1)
  double dist_thres;
  double weight_min;
};

// workspace views handed to the association kernels (global query index g in [0, Qt))
struct AssocWork {
  int64_t Qt;
  float4* pm;           // transformed query (x,y,z, _)
  float4* pmq;          // the same, cell-sorted order, .w = bitcast scan index (written by k_order_scatter)
  uint16_t* seg;        // segment id of the query
  int32_t* knn_idx;     // [5][Qt] neighbour indices, sorted order (K1a -> K1b)
  float* knn_sqd;       // [5][Qt] squared distances, sorted order
  uint8_t* status;
  float4* nsd;          // weight*n, weight*d   (scan-to-map)
  float* weight;
  double* normal_cent;  // 6 per query (pair mode) or nullptr
  // debug (nullable)
  int32_t* idx5;
  float* sqd5;
  double* plane;
};

// destination of one segment's compacted matches
struct CompactDst {
  float4* cpw;
  float4* nsd;
  double* nc;
  int32_t* src;
};

// per-block work item of the evaluation kernels: a contiguous run of residuals of one keyframe
struct EvalItem {
  const float4* cpw;    // (cp.xyz, weight)
  const float4* nsd;    // (n_s.xyz, d_s)
  int32_t count;
  int32_t kf;
};

// Launch bookkeeping: counts every kernel launch (bench "gpu_launches") and, when profiling is enabled, brackets
// each launch with CUDA events on the launching stream so per-kernel device time can be read back
// (bench.py roofline: measured live inside the timed region).
struct LaunchCounter {
  int64_t n = 0;
  bool prof = false;
  struct Rec { const char* name; cudaEvent_t a, b; };
  std::vector<Rec> recs;
  std::vector<cudaEvent_t> pool;
  cudaEvent_t get_event() {
    if (!pool.empty()) { cudaEvent_t e = pool.back(); pool.pop_back(); return e; }
    cudaEvent_t e; cudaEventCreate(&e); return e;
  }
  void begin(const char* name, cudaStream_t st) {
    ++n;
    if (prof) { Rec r{name, get_event(), get_event()}; cudaEventRecord(r.a, st); recs.push_back(r); }
  }
  void end(cudaStream_t st) { if (prof && !recs.empty()) cudaEventRecord(recs.back().b, st); }
};

// ---- K0 (grid.cu)
struct GridBuild {
  DevBuf<int> cell_start;
  DevBuf<float4> pts;
  DevBuf<float4> tmp4;     // unsorted (transformed) points, original order: (x,y,z,idx)
  DevBuf<int> sorted_pos;  // original index -> position in pts (cell-sorted)
  DevBuf<int> fill;        // scatter cursors
  DevBuf<int> scan_tmp;
  DevBuf<int> bounds;      // 6 order-preserving ints on device
  GridDesc desc{};
};
void grid_build(GridBuild& gb, const float* d_xyz, int stride, int64_t n, const double* t, const double* q,
                float cell_size_hint, float pts_per_cell, cudaStream_t st, LaunchCounter& lc);
void exclusive_scan_i32(const int* in, int* out, int64_t n, DevBuf<int>& tmp, cudaStream_t st, LaunchCounter& lc);

// ---- local map maintenance (grid.cu): world-frame keyframe clouds -> pcl::VoxelGrid-style down-sampling
struct VoxelWork {
  DevBuf<float4> tmp4;
  DevBuf<int> bounds, count, start, opos, order, sorted, scan_tmp, out_vox;
  DevBuf<float> out_xyz;      // filtered points, 3 floats each, ascending voxel index
};
void localmap_transform(const float* d_xyz, int stride, int64_t n, const double* t, const double* q, float4* d_out, cudaStream_t st, LaunchCounter& lc);
// returns the number of filtered points (in w.out_xyz / w.out_vox), or -1 when PCL would pass the input through unchanged
int64_t voxel_filter_run(VoxelWork& w, const float4* d_in, int64_t n, float leaf, cudaStream_t st, LaunchCounter& lc);

// ---- sort-based pcl::VoxelGrid (grid.cu): same output as voxel_filter_run, cost in the number of points, any bounding box
struct VoxelSortWork {
  DevBuf<float4> tmp4;                  // the input as (x, y, z, index)
  DevBuf<unsigned> key0, key1;          // radix sort ping-pong: voxel keys
  DevBuf<int> val0, val1;               //                       point indices
  DevBuf<int> bounds, bad, hist, flags, pos, scan_tmp;
  DevBuf<float> out_xyz;                // result, 3 floats per point
};
// n (> 0, < 2^31) points stride floats apart on the device -> w.out_xyz; returns its size.  *filtered = false: PCL's leaf-size check
// passed the input through (w.out_xyz holds the input x,y,z).  Non-finite coordinates are GLIO_ERR_ARG.
int64_t voxel_sort_run(VoxelSortWork& w, const float* d_xyz, int stride, int64_t n, float leaf, bool* filtered, cudaStream_t st, LaunchCounter& lc);

// A deque of world-frame clouds, their concatenation and its voxel filter: the context's local map (glio_localmap_*,
// Estimator.cpp:3529-3618) and the odometry's (LidarOdometry.cpp:267-288, :305-313) are both one of these.
struct LocalMap {
  struct Frame { DevBuf<float4> pts; int64_t n = 0; };
  std::deque<std::unique_ptr<Frame>> frames;
  std::vector<std::unique_ptr<Frame>> spare;   // buffers of popped frames, reused by the next push (no cudaFree / cudaMalloc per frame)
  DevBuf<float4> cat;
  VoxelWork vox;
  // transformCloud(cloud, {t, q}) = float(q*double(p)+t) on the device, then push_front / push_back
  void push(bool at_front, const float* d_xyz, int stride, int64_t n, const double* t, const double* q, cudaStream_t st, LaunchCounter& lc);
  void pop_front();            // the stream is ordered: anything still reading the popped buffer was enqueued before whatever reuses it
  void clear();                // drops every frame and frees its buffer
  int64_t n_points() const;
  // concatenate (oldest first) and VoxelGrid(leaf) when leaf > 0; *pts / *stride receive the device cloud.  Returns its size and
  // sets *filtered = false when leaf <= 0 or PCL's overflow rule passed the concatenation through unchanged.
  int64_t build(float leaf, const float** pts, int* stride, bool* filtered, cudaStream_t st, LaunchCounter& lc);
};

// ---- K1 / K1b (assoc.cu)
void assoc_run(const GridBuild& gb, const SegDesc* d_segs, int nseg, const AssocWork& w, const AssocGates& gates,
               const float* oth_local, int oth_stride, DevBuf<int>& cell_count, DevBuf<int>& cell_pos,
               DevBuf<int>& scan_tmp, cudaStream_t st, LaunchCounter& lc);
void compact_count(const AssocWork& w, const SegDesc* d_segs, int nseg, int* d_flags, int* d_pos, DevBuf<int>& scan_tmp,
                   int* d_counts, cudaStream_t st, LaunchCounter& lc);
void compact_scatter(const AssocWork& w, const SegDesc* d_segs, int nseg, const int* d_pos, const void* d_dst, cudaStream_t st,
                     LaunchCounter& lc);
void compact_run(const AssocWork& w, const SegDesc* d_segs, int nseg, int* d_flags, int* d_pos, DevBuf<int>& scan_tmp,
                 const void* d_dst /*CompactDst[nseg]*/, int* d_counts, cudaStream_t st, LaunchCounter& lc);
void gather_selection(const int32_t* d_keep, int64_t n, int64_t n_match, const float4* cpw, const float4* nsd, const double* nc,
                      float4* o_cpw, float4* o_nsd, double* o_nc, int* d_bad, cudaStream_t st, LaunchCounter& lc);

// ---- K1e (assoc.cu): scan-to-map edge association (glio_window_associate_edges)
struct EdgeFitParams {
  double max_sqdist, min_ratio, half_length;
};
// destination of one segment's compacted edge records (the slot's K2e inputs)
struct EdgeDst {
  float4* cps;    // (cp.xyz, s)
  float4* pa;
  float4* pb;
  int32_t* src;
};
// search + line fit: w.status (GLIO_EDGE_*), pa / pb per query in scan order; w.idx5 / w.sqd5 / eig (3 per query) when w.idx5 is set.
// oth_local != nullptr: pair mode (K1be), the line of a valid query refitted in the searched frame's stored coordinates (oth_stride
// floats apart, original order); no debug views.
void edge_assoc_run(const GridBuild& gb, const SegDesc* d_segs, int nseg, const AssocWork& w, const EdgeFitParams& ep, float4* pa, float4* pb,
                    double* eig, const float* oth_local, int oth_stride, DevBuf<int>& cell_count, DevBuf<int>& cell_pos,
                    DevBuf<int>& scan_tmp, cudaStream_t st, LaunchCounter& lc);
// after compact_count on w.status: the valid records of every segment into dst[segment]
void compact_edge_scatter(const AssocWork& w, const SegDesc* d_segs, const int* d_pos, const float4* pa, const float4* pb, float score,
                          const EdgeDst* d_dst, cudaStream_t st, LaunchCounter& lc);

// ---- feature selection (select.cu): one segment = one slot's or one pair's seeded sample of k of its n plane matches or edges
struct SelSeg {
  const float4* cpw;    // the segment's records: plane matches (cp.xyz, weight) or edges (cp.xyz, s)
  const float4* nsd;    // (n_s.xyz, d_s), window plane matches; nullptr otherwise
  const double* nc;     // 6 per match, pair plane matches; nullptr otherwise
  const float4* pa;     // edges: the line points pa and pb; nullptr for plane matches
  const float4* pb;
  float4* o_cpw; float4* o_nsd; double* o_nc;   // the selection buffers (same layout as gather_selection writes)
  float4* o_pa; float4* o_pb;
  int32_t* keep;        // [k] the selected record indices in draw order
  int64_t n;            // records; the draws come from 0 .. n-2
  uint64_t stream;
  int32_t k, pad;
};
constexpr int GLIO_SEL_MAX = 4096;   // largest k (F or B) a segment may draw
void select_sample_run(const SelSeg* d_segs, int nseg, int k_max, uint64_t seed, uint64_t domain, uint64_t nonce, cudaStream_t st,
                       LaunchCounter& lc);

// ---- K2 / K2b / K2e (eval.cu)
struct EvalParams {
  double q_lb[4], t_lb[3];
  double lidar_const;
  double huber_delta;
  int unit_score;       // 1: score = lidar_const for every match (front-end factor), 0: lidar_const * weight
};
constexpr int GLIO_NACC = 28;        // 21 upper-triangular H + 6 g + 1 cost
constexpr int EV_MAXW = 64;          // poses are passed in the kernel parameters up to this many keyframes
constexpr int GLIO_ITEM_MAX = 2048;  // residuals per evaluation work item
void eval_unary_run(const EvalItem* d_items, int nitems, int W, const double* d_poses, const EvalParams& ep, int jac_kind,
                    bool want_jac, double* d_partials, double* d_out, const int* d_kf_item_start, unsigned int* d_ticket,
                    cudaStream_t st, LaunchCounter& lc, unsigned int* done_flag = nullptr, unsigned int epoch = 0,
                    const double* h_poses = nullptr);   // h_poses: host copy of the poses, passed by value when W <= EV_MAXW
void eval_unary_residuals_run(const float4* cpw, const float4* nsd, int64_t n, const double* d_pose, const EvalParams& ep,
                              int jac_kind, double* d_r, double* d_J, cudaStream_t st, LaunchCounter& lc);


// ---- K2e (eval.cu): edge factors
struct EdgeItem {
  const float4* cps;   // (cp.xyz, s)
  const float4* pa;    // line point a
  const float4* pb;    // line point b
  int32_t count;
  int32_t kf;
};
// jac_kind 0: tangent rotation columns; 1: ambient x,y,z quaternion columns (marginalisation)
void eval_edge_run(const EdgeItem* d_items, int nitems, int W, const double* d_poses, const EvalParams& ep, int jac_kind, bool want_jac,
                   double* d_partials, double* d_out, const int* d_kf_item_start, unsigned int* d_ticket, cudaStream_t st, LaunchCounter& lc);

// ---- K2b (eval.cu): binary plane factors
struct BinItem {
  const float4* cpw;          // (cp.xyz, weight)
  const double* nc;           // 6 per residual: local-frame unit normal, local-frame centroid
  int32_t count;
  int32_t kf_c, kf_o;
};
// Per-pair sums of the binary factors, whose Jacobians are J_c = [u | v], J_o = [-u | z] (u, v, z: 3-vectors): J^T J needs only
// the distinct products uu(6) uv(9) vv(6) uz(9) vz(9) zz(6) (uu, vv, zz upper-triangular, uv / uz / vz row-major), then J^T r as
// r*u(3) r*v(3) r*z(3), then the cost.  eval.cu's pair_accumulate writes it, k_bin_assemble reads it.
constexpr int GLIO_NACC_BIN = 55;
// incidence list of a keyframe for the deterministic block assembly: (pair index, role 0 = cur / 1 = oth)
struct BinIncidence { int32_t pair; int32_t role; };
// d_pair_sums_edge (nullable): per-pair K2be sums added to the plane sums (S = S_plane + S_edge) before the block assembly
void eval_binary_run(const BinItem* d_items, int nitems, const int* d_pair_item_start, int n_pairs, int K, const double* d_poses,
                     double score_scale, double huber_delta, bool want_jac, double* d_partials, double* d_pair_sums,
                     const int* d_kf_inc_start, const BinIncidence* d_inc, double* d_diag /*K*28*/, double* d_off /*n_pairs*36*/,
                     cudaStream_t st, LaunchCounter& lc, const double* d_pair_sums_edge = nullptr);
// k_bin_assemble alone: per-pair sums S -> d_diag (K x 28) and, with want_jac, d_off (n_pairs x 36)
void bin_assemble_run(const double* d_pair_sums, int K, int n_pairs, const int* d_kf_inc_start, const BinIncidence* d_inc, bool want_jac,
                      double* d_diag, double* d_off, cudaStream_t st, LaunchCounter& lc);

// ---- K2be (eval.cu): binary point-to-edge factors, the edge counterpart of BinaryLidarPlaneNormFactor
struct BinEdgeItem {
  const float4* cps;          // (cp.xyz in cur's body frame, s)
  const float4* pa;           // line point a in oth's body frame
  const float4* pb;           // line point b in oth's body frame
  int32_t count;
  int32_t kf_c, kf_o;
};
// per-item partials (GLIO_NACC_BIN layout of K2b) and their per-pair sums in item order -> d_pair_sums (n_pairs x 55)
void eval_binary_edge_run(const BinEdgeItem* d_items, int nitems, const int* d_pair_item_start, int n_pairs, const double* d_poses,
                          bool want_jac, double* d_partials, double* d_pair_sums, cudaStream_t st, LaunchCounter& lc);

// ---- K2p (eval.cu): the batch refinement's pose factors, LidarPoseFactorBatchRelativeAutoDiff (kind 0, 6 rows) and
// delta_q_factor_auto (kind 1, 3 rows); the layout of the public glio_pose_factor
struct PoseFactor { int32_t i, j, kind, active; double dq[4]; double dp[3]; };
// Per distinct keyframe pair (a, b), a < b, the sums of its factors' 12 x 12 J^T J, J^T r and cost over the tangent columns
// (t_a, d_a, t_b, d_b): aa upper-triangular (21), bb upper-triangular (21), ab row-major (36), g (12), cost.
constexpr int GLIO_NACC_POSE = 91;
// k_pose_pair_sums: the factors of pair p are f[fstart[p] .. fstart[p+1]) in list order -> d_sums (n_pairs x 91);
// k_pose_assemble: per keyframe k < n_inc_kf the pairs of its incidence list (role 0 = a, 1 = b), in order, summed into d_diag
// (K x 28, added to its contents when add, else written; the cost goes to a) and, with want_jac, the ab blocks -> d_off (n_pairs x 36).
// Two launches whatever K; with n_pairs = 0 only the assembly runs.
void eval_pose_run(const PoseFactor* d_f, const int* d_fstart, int n_pairs, int K, int n_inc_kf, const int* d_kf_inc_start,
                   const BinIncidence* d_inc, const double* d_poses, bool want_jac, bool add, double* d_sums, double* d_diag, double* d_off,
                   cudaStream_t st, LaunchCounter& lc);

// ---- K2g (eval.cu): the batch refinement's double-differenced pseudorange factors (dd_psr_factor_20); the layouts of the public
// glio_dd_psr_factor and glio_dd_psr_sat
struct DdPsrFactor { int32_t i, j, n_sat, master, active, reserved; int64_t sat_offset, w_offset; double ratio, threshold, station[3]; };
struct DdPsrSat { double sat_user[3], sat_ref[3], psr_user, psr_ref; };
// the per-list constants: R_ecef_local (row-major) and the anchor, passed by value
struct DdPsrFrame { double R[9]; double anchor[3]; };
// Per distinct keyframe pair (a, b), a < b, the sums of its factors' 6 x 6 J^T J, J^T r and cost over (t_a, t_b): aa and bb
// upper-triangular (6 + 6), ab row-major (9), g (3 + 3), cost.
constexpr int GLIO_NACC_DD = 28;
// k_psr_pair_sums: the factors of pair p are f[fstart[p] .. fstart[p+1]) in list order, their satellites and weights read at the
// records' offsets in d_sats / d_w -> d_sums (n_pairs x 28); k_psr_assemble: as k_pose_assemble, the t columns only.
// Two launches whatever K; with n_pairs = 0 only the assembly runs.
void eval_dd_psr_run(const DdPsrFactor* d_f, const int* d_fstart, const DdPsrSat* d_sats, const double* d_w, const DdPsrFrame& frame,
                     int n_pairs, int K, int n_inc_kf, const int* d_kf_inc_start, const BinIncidence* d_inc, const double* d_poses,
                     bool want_jac, bool add, double* d_sums, double* d_diag, double* d_off, cudaStream_t st, LaunchCounter& lc);

// ---- K2i (eval.cu): the batch refinement's IMU factors (ImuFactor) from the caller's pre-integration; the layout of the public
// glio_imu_factor.  The 3 x 3 jacobian_ blocks and sqrt_info are row-major.
struct ImuFactor {
  int32_t i, j, active, reserved;
  double sum_dt, g_vec[3];
  double delta_p[3], delta_q[4], delta_v[3];
  double linearized_ba[3], linearized_bg[3];
  double dp_dba[9], dp_dbg[9], dq_dbg[9], dv_dba[9], dv_dbg[9];
  double sqrt_info[225];
};
// Per distinct keyframe pair (a, b), a < b, the sums of its factors' 30 x 30 J^T J, J^T r and cost over the tangent columns
// (x_a, x_b), x = [t, delta, v, ba, bg]: aa (225), bb (225), ab (225), all row-major, g (15 + 15), cost.
constexpr int GLIO_NACC_IMU = 706;
// Per keyframe: its 15 x 15 diagonal block (row-major), g (15) and cost.
constexpr int GLIO_NACC_IMU_KF = 241;
// k_imu_pair_sums: the factors of pair p are f[fstart[p] .. fstart[p+1]) in list order, at poses (K x 7) and speed_bias (K x 9)
// -> d_sums (n_pairs x 706); k_imu_assemble: per keyframe k < n_inc_kf the pairs of its incidence list, in order, written into
// d_diag (K x 241; the cost goes to a) and, with want_jac, the ab blocks -> d_off (n_pairs x 225).  Two launches whatever K; with
// n_pairs = 0 only the assembly runs.  jac_kind 0: the delta columns are the tangent ones; 1: the ambient x, y, z quaternion columns
// (k_imu_pair_sums_ambient; the cost-only launch is the same for both).
void eval_imu_run(const ImuFactor* d_f, const int* d_fstart, int n_pairs, int K, int n_inc_kf, const int* d_kf_inc_start,
                  const BinIncidence* d_inc, const double* d_poses, const double* d_sb, int jac_kind, bool want_jac, double* d_sums,
                  double* d_diag, double* d_off, cudaStream_t st, LaunchCounter& lc);
// k_imu_pair_sums alone over n_pairs pairs starting at d_fstart (a sub-range of a list's plan) -> d_sums (n_pairs x 706)
void eval_imu_pair_sums_run(const ImuFactor* d_f, const int* d_fstart, int n_pairs, const double* d_poses, const double* d_sb, int jac_kind,
                            bool want_jac, double* d_sums, cudaStream_t st, LaunchCounter& lc);

// ---- front-end feature extraction (features.cu; Preprocessing.cpp:529-655)
constexpr int FEAT_MAX_SHARP = 12, FEAT_MAX_LESS_SHARP = 60, FEAT_MAX_FLAT = 24;   // per ring: 6 sectors x (2, 10, 4)
struct FeatArgs {
  const float* cloud; int stride; int ioff; int64_t n;     // ioff: float offset of the intensity (3 packed, 4 in pcl::PointXYZI)
  int n_scans; const int32_t* scan_start; const int32_t* scan_end; int ds_rate;
  double edge_thres, surf_thres; float ds_v;
  float* curv; int8_t* label; int8_t* picked;
  int32_t* ring_sharp; int32_t* ring_less_sharp; int32_t* ring_flat;   // [n_scans][MAX] slots
  int32_t* ring_less_flat;                                             // [n] ring r's list starts at scan_start[r]
  float4* ring_ds;                                                     // [n] ring r's down-sampled points start at scan_start[r]
  int32_t* counts;                                                     // [5][n_scans]: sharp, less_sharp, flat, less_flat, ds
  int32_t* offsets;                                                    // [5][n_scans + 1]
  int32_t* err;                                                        // != 0: a sector / ring exceeded the shared-memory capacity
  int32_t* out_sharp; int32_t* out_less_sharp; int32_t* out_flat; int32_t* out_less_flat; float4* out_ds;
};

void features_run(FeatArgs& a, cudaStream_t st, LaunchCounter& lc);

// ---- front-end sweep preparation (scanprep.cu; Preprocessing.cpp:387-526)
struct SweepConsts {
  int ok;                              // 0: no point survives the NaN / 3 m filters
  float start_ori, end_ori;            // :401-410
  double c_first_lo, c_first_hi;       // startOri - M_PI/2, startOri + M_PI*3/2   (:491-494)
  double c_second_lo, c_second_hi;     // endOri - M_PI*3/2, endOri + M_PI/2       (:501-504)
};
struct ScanPrepArgs {
  const float* raw; int stride; int64_t n; int n_scans; int nb;    // nb: blocks of 256 raw points
  // per-sweep rotation constants, computed once on the host
  double q_imu[4], q_lb[4], q_lb_inv[4];                           // w, x, y, z
  double dot, theta, sin_theta; int slerp_linear;                  // Eigen slerp: d, acos|d|, sin(theta), |d| >= 1 - eps
  SweepConsts* consts;
  int32_t* small;                      // [0] first kept-by-filter index, [1] last, [2] halfPassed index, [3] ok, [4] count, [5..] ranges
  int8_t* ring; float* ori;            // [n] ring id (-1 skipped), raw azimuth -atan2f(y, x)
  int32_t* hist; int32_t* hscan;       // [n_scans][nb] per-block ring counts and their ring-major exclusive scan
  DevBuf<int>* scan_tmp;
  unsigned long long* guard_hits;      // correctly rounded atanf / atan2f: evaluations decided in double-double
  float4* out; int64_t out_capacity;
};
void scanprep_run(ScanPrepArgs& a, cudaStream_t st, LaunchCounter& lc);
void imu_sweep_rotation(glio_imu_state* st, const double* stamps, const double* gyro, int64_t n, double t_cur, double q[4]);

// ---- front-end odometry (odometry.cu; LidarOdometry.cpp).  Poses here are the reference's abs_pose / rel_pose layout:
// q(w,x,y,z) then t(x,y,z).  Host arithmetic is scalar double in Eigen's operation order, built without FMA contraction.
void odom_predict(double abs_pose[7], const double rel_pose[7]);                                   // poseInitialization, :406-433
void odom_relative(const double prev[7], const double cur[7], double rel_pose[7]);                 // computeRelative, :435-471
// the keyframe test of updateTransformationWithCeres (:566-578); size = pose count before this sweep's savePoses
bool odom_keyframe_rule(const double t_cur[3], const double q_cur[4], const double t_last_kf[3], const double q_last_kf[4],
                        int64_t size, int64_t kf_num);
void odom_quat_inverse(const double q[4], double o[4]);                                              // Eigen inverse(): conj / squaredNorm
// publishCloudLast's undistortion (:176-200, :619-632) of surf and full in one launch: trans = rel_pose translation;
// deskew = 0 copies the clouds (checkInitialization, or if_to_deskew = false)
void odom_publish_run(const float4* surf, int64_t n_surf, const float4* full, int64_t n_full, float4* surf_out, float4* full_out,
                      const double trans[3], int deskew, cudaStream_t st, LaunchCounter& lc);

// ---- loop-closure registration (loop.cu; pcl::IterativeClosestPoint as Estimator.cpp:5183-5273 configures it)
// The registration state, resident on the device and read back once per iteration batch.  Matrices are row-major 4x4 floats.
struct IcpState {
  int32_t done;            // set by the one-thread kernels: every later kernel of the registration returns at once
  int32_t converged, state, nr_iter;
  int32_t n_corr;          // correspondences of the last correspondence estimation
  int32_t nr_fit, pad0, pad1;
  float transformation[16], final_T[16];
  float smean[3], tmean[3];
  double prev_mse, mse, fitness;
};
struct IcpConvergence {    // DefaultConvergenceCriteria as IterativeClosestPoint::computeTransformation sets it
  int32_t max_iterations, log_cap;
  double translation_threshold, rotation_threshold, mse_threshold_relative, mse_threshold_absolute;
};
struct IcpWork {
  GridBuild grid;                                     // the target (fixed over the iterations)
  DevBuf<float4> src0, cur, fit;                      // input, input_transformed (updated in place), input * final
  DevBuf<int> qcount, qstart, perm, scan_tmp;         // cell order of the source
  DevBuf<int> nn_idx, flags, pos, cq, cm;
  DevBuf<float> nn_d, cd;
  DevBuf<float> pf0, pf1; DevBuf<double> pd0, pd1;    // partial sums, levels 0 and 1
  DevBuf<glio_icp_iteration> log;
  DevBuf<IcpState> state;
  IcpState last{};
  int64_t n_src = 0, n_tgt = 0;
};
// one registration of d_src (n_src points, src_stride floats apart) onto d_tgt; *out receives the final state (fitness included).
// w.fit holds the aligned cloud (float4), w.cq / w.cm / w.cd the last correspondence list, w.log the first min(log_cap, iterations)
// iteration records.
void icp_run(IcpWork& w, const float* d_src, int src_stride, int64_t n_src, const float* d_tgt, int tgt_stride, int64_t n_tgt,
             const glio_icp_options& o, int log_cap, float pts_per_cell, cudaStream_t st, LaunchCounter& lc, IcpState* out, int* host_syncs);
// host pose arithmetic of performLoopClosure / detectLoopClosure (poses t, q; scalar double in Eigen's order)
void loop_quat_from_R(const double R[9], double q[4]);
void loop_extrinsic_bl(const double q_lb[4], const double t_lb[3], double q_bl[4], double t_bl[3]);
void loop_world_of_cloud(const double pose[7], const double q_bl[4], const double t_bl[3], double t[3], double q[4]);
void loop_pose_from(const float final_T[16], const double latest[7], double out[7]);
// save_pcd's concatenation (Estimator.cpp:5338-5341): segment s (n points, packed x,y,z) moved by first, then by its own pose, each
// transformCloud rounding to float; written to out + off as float4
struct GlobalMapSeg { const float* xyz; int64_t n, off; double t[3], q[4]; };
void loop_global_map_cloud(const GlobalMapSeg* d_segs, int nseg, int64_t n_max, const double t_first[3], const double q_first[4], float4* out,
                           cudaStream_t st, LaunchCounter& lc);

// ---- K4 (band.cu): band Cholesky factor-and-solve in one thread block (glio_band_solve).  d_band[n*(hb+1)] in A, out L;
// d_x[n] out; d_flag[0] = 1 on success, 0 on a pivot that is not positive and finite or a non-finite x.  Needs
// band_chol_smem_bytes(hb) of shared memory; hb <= GLIO_BAND_MAX_HB fits.
size_t band_chol_smem_bytes(int hb);
void band_chol_solve_run(double* d_band, const double* d_b, double* d_x, int n, int hb, int* d_flag, cudaStream_t st, LaunchCounter& lc);
// The device minimizer's band passes (glio_batch_use_device_solver).  The assembly plan: per nt x nt band block (ka, kb), ka >= kb,
// its contributions [c0, c1) in the host path's order; BAND_*_T blocks are read transposed.
enum BandContribKind { BAND_DIAG6 = 0, BAND_OFF6 = 1, BAND_OFF6_T = 2, BAND_IMU_DIAG = 3, BAND_IMU_OFF_T = 4 };
struct BandContrib { int32_t kind, idx; };
struct BandBlock { int32_t ka, kb, c0, c1; };
// d_H / d_g already hold the host callback's band and g (or zeros)
void band_assemble_run(double* d_H, int hb, int nt, const BandBlock* d_blocks, int n_blocks, const BandContrib* d_contrib,
                       const double* d_diag6, const double* d_off6, const double* d_imu_diag, const double* d_imu_off, double* d_g, int n,
                       cudaStream_t st, LaunchCounter& lc);
void band_scale_run(const double* d_H, double* d_Hs, const double* d_s, int n, int hb, double* d_hs_diag, cudaStream_t st, LaunchCounter& lc);
void band_shift_run(const double* d_Hs, double* d_A, const double* d_v, int n, int hb, cudaStream_t st, LaunchCounter& lc);
void band_symv_run(const double* d_Hs, const double* d_x, double* d_y, int n, int hb, cudaStream_t st, LaunchCounter& lc);

// ---- the band solve by block cyclic reduction (bcr.cu; glio_band_solve_bcr, GLIO_FACTOR_BCR).  Blocks of bcr_block_size(hb) rows;
// the workspace keeps L, U^T, V^T and w of every level for the back-substitution, grown to the largest shape solved.
int bcr_block_size(int hb);
struct BcrWork {
  DevBuf<double> D, E, U, R, X;   // m blocks each: b x b (D, E, U), b (R, X)
  DevBuf<int> flag;               // 1 after a pivot that is not positive and finite, or a non-finite x
  void reserve(int n, int hb);
};
// solves A x = b for the band d_band (n x (hb+1), glio_band_solve's layout; the band is only read), with d_v != nullptr the shifted
// A = band + diag(v * v); d_x[n] out, w.flag[0] = 0 on success.  hb <= GLIO_BAND_BCR_MAX_HB.
void bcr_solve_run(BcrWork& w, const double* d_band, const double* d_v, const double* d_b, double* d_x, int n, int hb, cudaStream_t st,
                   LaunchCounter& lc);

}  // namespace glio
