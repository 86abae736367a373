// capi.cu — the extern "C" boundary (include/glio_b200.h) and the context that owns device state.
// No CPU fallback: without a CUDA device glio_create fails.
#include <array>
#include <cfloat>
#include <atomic>
#include <condition_variable>
#include <mutex>
#include <thread>
#if defined(__linux__)
#include <pthread.h>
#include <sched.h>
#endif
#include <chrono>
#include <deque>
#include <map>
#include <set>
#include <memory>

#include "common.cuh"
#include "hostmath.h"
#include "solver.h"
#include "marg.h"

using namespace glio;

namespace {

// n points, stride floats apart, on the device: uploaded into `own`, or a caller-owned device pointer (GLIO_DEVICE input)
struct PointSet {
  int64_t n = 0;
  int stride = 3;
  DevBuf<float> own;
  const float* ptr = nullptr;    // == own.p, or the caller's pointer
  void clear() { n = 0; ptr = nullptr; }
};

// the per-query views of one association (keep_debug): fit holds 4 doubles per query (the plane) or 3 (the line's eigenvalues)
struct AssocDebug {
  DevBuf<uint8_t> status;
  DevBuf<int32_t> idx5;
  DevBuf<float> sqd5;
  DevBuf<float4> pm;
  DevBuf<double> fit;
  int64_t Q = 0;
};

// the records an evaluation or a selection reads: n records, a column the list's kind does not use is nullptr
struct CorrView {
  const float4* cpw; const float4* nsd; const double* nc; const float4* pa; const float4* pb;
  int64_t n;
};

// the three kinds of correspondence list and their columns
enum CorrKind {
  CORR_WINDOW_PLANES,   // a slot's plane matches: cpw = (cp.xyz, weight), nsd = (n_s.xyz, d_s)
  CORR_PAIR_PLANES,     // a pair's plane matches: cpw, nc = 6 doubles per record (local-frame unit normal, local-frame centroid)
  CORR_EDGES            // a slot's or a pair's edges: cpw = (cp.xyz, s), line points pa / pb
};

// the record columns of one list; only the columns of its kind are ever reserved
struct CorrCols {
  DevBuf<float4> cpw, nsd, pa, pb;
  DevBuf<double> nc;
  void reserve(CorrKind kind, int64_t q) {
    cpw.reserve((size_t)q);
    if (kind == CORR_WINDOW_PLANES) nsd.reserve((size_t)q);
    if (kind == CORR_PAIR_PLANES) nc.reserve(6 * (size_t)q);
    if (kind == CORR_EDGES) { pa.reserve((size_t)q); pb.reserve((size_t)q); }
  }
  CorrView view(int64_t n) const { return CorrView{cpw.p, nsd.p, nc.p, pa.p, pb.p, n}; }
};

// One correspondence list: n records (rec), src = the scan index of each record (has_src: for edges, whether an association wrote
// it), and the selected subset: n_sel records in keep order (a keep list or the sampler's draws), -1 when there is none and every
// record is active.  Every change of the list marks `plan`, the owner's work-item plan that reads it, stale (nullptr: the owner
// cuts its plan afresh for every evaluation).
struct CorrList {
  const CorrKind kind;
  bool* const plan;
  CorrCols rec; DevBuf<int32_t> src; int64_t n = 0; bool has_src = false;
  CorrCols sel; DevBuf<int32_t> keep; int64_t n_sel = -1;
  CorrList(CorrKind k, bool* p) : kind(k), plan(p) {}
  void set_selection(int64_t m) { n_sel = m; if (plan) *plan = true; }
  // replacing the list drops its selection
  void clear() { n = 0; has_src = false; set_selection(-1); }
  int64_t n_active() const { return n_sel >= 0 ? n_sel : n; }
  // what every consumer reads: the selected subset if there is one, otherwise the whole list
  CorrView active() const { return n_sel >= 0 ? sel.view(n_sel) : rec.view(n); }
  // room for q records and their src, which drops the selection; a reserve may drop the old contents, so the caller clears the
  // list first or sets n before the records are written
  void reserve(int64_t q) { set_selection(-1); rec.reserve(kind, q); src.reserve((size_t)q); }
  // the destination of an association's compacted records
  CompactDst plane_dst(int64_t q) { reserve(q); return CompactDst{rec.cpw.p, rec.nsd.p, rec.nc.p, src.p}; }
  EdgeDst edge_dst(int64_t q) { reserve(q); return EdgeDst{rec.cpw.p, rec.pa.p, rec.pb.p, src.p}; }
  // the k_sel_sample segment that draws k of the records into the selection columns
  SelSeg sample_seg(int k, uint64_t stream) {
    sel.reserve(kind, k); keep.reserve((size_t)k);
    SelSeg g{};
    g.cpw = rec.cpw.p; g.nsd = rec.nsd.p; g.nc = rec.nc.p; g.pa = rec.pa.p; g.pb = rec.pb.p;
    g.o_cpw = sel.cpw.p; g.o_nsd = sel.nsd.p; g.o_nc = sel.nc.p; g.o_pa = sel.pa.p; g.o_pb = sel.pb.p;
    g.keep = keep.p; g.n = n; g.stream = stream; g.k = k;
    return g;
  }
};

// A device pair-factor list of the batch solve (pose factors, DD pseudorange factors): its switch, its pair table, the largest
// keyframe referenced, and the plan built when the list is set: per-pair starts into the active records (grouped by pair in list
// order; the records sit beside the list in the context), per-keyframe incidence lists and the pair sums
struct PairFactorList {
  bool use = false;                                  // glio_batch_use_*: glio_batch_solve adds the list's blocks
  std::vector<std::pair<int, int>> pairs; int max_kf = -1;
  DevBuf<int> d_fstart, d_inc_start; DevBuf<BinIncidence> d_inc; DevBuf<double> d_sums;
  void clear() { pairs.clear(); max_kf = -1; }
  // a new list's table and buffers; the switch stays as it was
  void take(PairFactorList&& o) { const bool u = use; *this = std::move(o); use = u; }
};

// An IMU factor list (K2i): the pair-factor list, its active records, and the buffers of one evaluation: the speed-bias states and
// the IMU blocks (K x 241 and n_pairs x 225), on the device and in pinned memory.  The batch solve and the window keep one each.
struct ImuFactorList : PairFactorList {
  DevBuf<ImuFactor> d_f;
  DevBuf<double> d_sb, d_diag, d_off; PinnedBuf<double> h_sb, h_diag, h_off;
};

struct Slot {
  PointSet scan;                 // surf scan
  CorrList planes;               // glio_window_associate (scan order) or glio_set_matches
  CorrList edges;                // glio_set_edges or glio_window_associate_edges
  PointSet corners;              // corner scan (glio_window_set_edge_scan)
  AssocDebug dbg, edge_dbg;      // keep_debug: the last plane and the last edge association
  explicit Slot(bool* plane_plan = nullptr, bool* edge_plan = nullptr) : planes(CORR_WINDOW_PLANES, plane_plan), edges(CORR_EDGES, edge_plan) {}
};

// a map the window associates against (surf or corner points): its grid, and the local map that can build it
struct FeatureMap {
  GridBuild grid;
  bool valid = false;
  int64_t n = 0;
  DevBuf<float> stage;           // host-input staging
  LocalMap lm;
  DevBuf<float> lm_stage;
};

}  // namespace

// One marginalisation whose host half (A/b assembly, Schur, eigen-decomposition, prior) runs on the context's worker thread while
// the caller goes on (typically: hands the next window's association to the GPU).  The device half was queued by the caller.
struct glio_marg_job {
  glio_ctx* ctx = nullptr;
  int W = 0;
  double eps = 1e-8;
  unsigned int epoch = 0;
  int submit_cpu = -1;                 // CPU the submitting thread ran on (the worker keeps off it)
  std::vector<double> A, b;            // host-side accumulations (IMU / previous prior), marginalisation ordering
  std::vector<double> x0_pose, x0_sb;  // linearisation point of the kept states
  std::vector<double> out;             // snapshot of the device result (W x 28)
  std::atomic<int> copied{0};          // the worker no longer needs the context's result buffer
  std::atomic<int> done{0};
  int rc = 0;
  std::string err;
  glio_marg_prior* prior = nullptr;
  bool with_imu = false;               // the device half queued the window IMU factor KF0 -> KF1
  std::vector<double> imu;             // snapshot of its pair sums (706)
};

struct glio_ctx {
  int device = 0;
  // worker thread of glio_window_marginalize_async (started lazily, joined by glio_destroy)
  std::thread marg_thread;
  std::mutex marg_mu;
  std::condition_variable marg_cv;
  glio_marg_job* marg_queued = nullptr;      // handed to the worker (guarded by marg_mu)
  bool marg_quit = false;
  glio_marg_job* marg_pending = nullptr;     // the job in flight, caller-thread view (one at a time)
  cudaStream_t st = nullptr;
  glio_params prm{};
  std::string err;
  LaunchCounter lc;

  int eval_slots = 296;        // resident evaluation blocks: 2 per SM (set from the device at creation)
  float pts_per_cell = 8.0f;   // target points per occupied grid cell (tuning hook: env GLIO_PTS_PER_CELL)
  FeatureMap map, edge_map;    // surf and corner
  // map prefetch (glio_map_prefetch): the next window's local map travels on the copy stream while the current window is marginalised
  DevBuf<float> map_stage2; const float* pf_ptr = nullptr; int64_t pf_M = 0; int pf_stride = 0; cudaEvent_t ev_map = nullptr;

  std::vector<std::unique_ptr<Slot>> slots;

  // ---- batch (scan-to-multiscan) state
  // a frame's cloud and the grid of its world copy, built when a pair first searches it and dropped with the pose
  struct FrameCloud { PointSet pts; GridBuild grid; bool grid_valid = false; };
  struct Frame {
    double pose[7] = {0, 0, 0, 1, 0, 0, 0};
    FrameCloud surf;
    FrameCloud corners;          // glio_batch_set_edge_frame, 0 points allowed
    bool has_edge = false;
    void set_pose(const double p[7]) {
      for (int i = 0; i < 7; ++i) pose[i] = p[i];
      surf.grid_valid = false; corners.grid_valid = false;
    }
  };
  struct Pair {
    int cur = 0, oth = 0;
    CorrList planes;             // glio_batch_associate_pairs or glio_batch_set_pair_matches
    CorrList edges;              // glio_batch_associate_edges_pairs or glio_batch_set_pair_edges: cp in cur's frame, pa / pb in oth's
    Pair(int c, int o, bool* plane_plan, bool* edge_plan) : cur(c), oth(o), planes(CORR_PAIR_PLANES, plane_plan), edges(CORR_EDGES, edge_plan) {}
  };
  std::map<int, std::unique_ptr<Frame>> frames;
  std::vector<std::unique_ptr<Pair>> pairs;
  std::map<std::pair<int, int>, int> pair_index;
  bool bin_dirty = true; int bin_K = -1; int n_bin_items = 0;
  glio_allreduce_fn allreduce = nullptr; void* allreduce_user = nullptr;
  DevBuf<BinItem> d_bin_items; DevBuf<int> d_pair_item_start, d_kf_inc_start; DevBuf<BinIncidence> d_inc;
  DevBuf<double> d_bin_partials, d_pair_sums, d_bin_diag, d_bin_off, d_bin_poses;
  PinnedBuf<double> h_bin_diag, h_bin_off, h_bin_poses;
  // binary edge blocks (glio_batch_use_edges, glio_eval_binary_edge): the K2be work-item plan, rebuilt only when an edge list, K,
  // the pair count or the switch changes; its per-pair sums are added to the plane sums before the one block assembly
  bool batch_use_edges = false, bedge_dirty = true; int bedge_K = -1, bedge_P = -1, n_bedge_items = 0;
  DevBuf<BinEdgeItem> d_bedge_items; DevBuf<int> d_bedge_pstart; DevBuf<double> d_bedge_partials, d_bedge_sums;
  // pose factors (glio_batch_set_pose_factors, K2p): the list and its active records
  PairFactorList pose; DevBuf<PoseFactor> d_pose_f;
  // DD pseudorange factors (glio_batch_set_dd_psr_factors, K2g): the list, its active records, and the list's satellites, weights
  // and frame constants
  PairFactorList dd; DevBuf<DdPsrFactor> d_dd_f; DevBuf<DdPsrSat> d_dd_sats; DevBuf<double> d_dd_w; DdPsrFrame dd_frame{};
  // IMU factors (glio_batch_set_imu_factors, K2i), kept apart from the 6-column buffers above
  ImuFactorList imu;

  // association workspace
  DevBuf<float4> w_pm, w_pmq, w_nsd;
  DevBuf<uint16_t> w_seg;
  DevBuf<uint8_t> w_status;
  DevBuf<float> w_weight;
  DevBuf<double> w_nc, w_plane;
  DevBuf<int32_t> w_idx5;
  DevBuf<float> w_sqd5;
  DevBuf<int32_t> w_knn_idx;
  DevBuf<float> w_knn_sqd;
  DevBuf<int> w_flags, w_pos, cell_count, cell_pos, scan_tmp;
  DevBuf<SegDesc> d_segs;
  DevBuf<CompactDst> d_dst;
  DevBuf<int> d_counts;
  PinnedBuf<int> h_counts;
  DevBuf<int> d_bad;
  // seeded feature selection: the segment table of one k_sel_sample launch, staged in pinned memory; ev_sel marks its upload
  DevBuf<SelSeg> d_sel_segs; PinnedBuf<SelSeg> h_sel_segs; cudaEvent_t ev_sel = nullptr;
  // front-end feature extraction work space
  DevBuf<float> f_cloud, f_curv; DevBuf<int8_t> f_label, f_picked; DevBuf<int32_t> f_scan, f_ring, f_lf, f_counts, f_out; DevBuf<float4> f_ds, f_outds;
  // front-end sweep preparation work space
  DevBuf<float> sp_raw, sp_ori; DevBuf<int8_t> sp_ring; DevBuf<int32_t> sp_hist, sp_hscan, sp_small; DevBuf<int> sp_scan_tmp;
  DevBuf<SweepConsts> sp_consts; DevBuf<float4> sp_out; DevBuf<unsigned long long> sp_hits;
  // K2e scratch (kept in the context: no cudaMalloc / cudaFree per call, nothing to leak when a call throws)
  DevBuf<EdgeItem> e_items; DevBuf<int> e_start; DevBuf<double> e_part, e_out, e_poses;

  // evaluation
  DevBuf<EvalItem> d_items;
  DevBuf<int> d_kf_item_start;
  DevBuf<double> d_partials, d_out, d_poses, d_r, d_J;
  PinnedBuf<double> h_out, h_poses;
  // edge association (K1e): the per-query line-fit outputs (scan order)
  DevBuf<float4> w_pa, w_pb; DevBuf<double> w_eig; DevBuf<EdgeDst> d_edst;
  // edge blocks inside the window solve and marginalisation (glio_window_use_edges): the K2e work-item plan of slots 0..W-1, rebuilt
  // only when an edge list or W changes; K2e runs on the main stream before K2 and its W x 28 result is copied into pinned h_eout
  // there, so K2's completion flag covers it.  edge_epoch: the evaluation epoch whose result must add h_eout.
  bool use_edges = false, edge_items_dirty = true; int edge_items_W = -1, n_edge_items = 0;
  DevBuf<EdgeItem> se_items; DevBuf<int> se_start; DevBuf<double> se_part, se_out, se_poses; PinnedBuf<double> h_eout;
  unsigned int edge_epoch = 0; int edge_W = 0;
  // front-end odometries created on this context (glio_odom_create); glio_destroy frees those still attached
  std::vector<glio_odom*> odoms;
  // loop-closure registration: glio_icp_align's work space and staging, and the loop objects created on this context
  IcpWork icp; DevBuf<float> icp_src, icp_tgt;
  std::vector<glio_loop*> loops;
  // sort-based VoxelGrid of glio_voxel_filter and glio_loop_global_map: its own work space, host-input staging, the global map's
  // concatenation and segment table
  VoxelSortWork vsort; DevBuf<float> vs_stage; DevBuf<float4> gm_cat; DevBuf<GlobalMapSeg> gm_segs;
  cudaStream_t st_copy = nullptr;      // window scans travel on their own stream so the upload of the next window can overlap a running solve
  cudaEvent_t ev_scans = nullptr, ev_main = nullptr;
  bool scans_pending = false;
  PinnedBuf<unsigned int> h_flag;      // completion epoch written by the last block of k_eval_unary
  unsigned int eval_epoch = 0;
  DevBuf<unsigned int> d_ticket;
  bool items_dirty = true;
  int items_W = -1;
  int n_items = 0;

  // the window's IMU chain (glio_window_set_imu_factors, glio_window_use_imu_factors), separate from the batch list: its poses
  // travel from pinned memory; a marginalisation copies pair {0, 1}'s ambient-column sums into h_wimu_marg, which an asynchronous
  // marginalisation owns until its worker has copied it (wait_marg_copied).  Kept after the members above, whose layout stays as
  // it was without the window chain.
  ImuFactorList window_imu;
  DevBuf<double> wimu_poses; PinnedBuf<double> h_wimu_poses, h_wimu_marg;
  // what the marginalisation needs of the list's slot 0: the index of pair {0, 1} when an active factor joins slots 0 and 1 (-1
  // otherwise), and whether an active factor joins slot 0 to another slot
  int wimu_pair01 = -1; bool wimu_slot0_elsewhere = false;
  // glio_band_solve (K4): the band, right-hand side, solution and success flag, grown to the largest system solved
  DevBuf<double> band_a, band_b, band_x; DevBuf<int> band_flag;
  // glio_batch_use_device_solver: the device minimizer's bands (H, Hc, Hs, A), vectors and assembly plan, reserved per shape
  bool batch_device_solver = false;
  DevBuf<double> dm_H[2], dm_g, dm_Hs, dm_A, dm_v1, dm_v2, dm_v3; DevBuf<int> dm_flag;
  DevBuf<BandBlock> dm_blocks; DevBuf<BandContrib> dm_contrib; PinnedBuf<double> dm_h1, dm_h2;
  // glio_batch_device_factorization's kind, and the block cyclic reduction's workspace (glio_band_solve_bcr and the minimizer)
  int batch_factorization = GLIO_FACTOR_SEQUENTIAL;
  BcrWork bcr;

  Slot& slot(int k) {
    GLIO_REQUIRE(k >= 0 && k < 4096, GLIO_ERR_ARG, "slot index out of range");
    if ((size_t)k >= slots.size()) slots.resize((size_t)k + 1);
    if (!slots[k]) slots[k].reset(new Slot(&items_dirty, &edge_items_dirty));
    return *slots[k];
  }
};

namespace {

// GLIO_TRACE=1: wall-clock marks of the association call (each mark synchronises the stream first)
struct Trace {
  bool on; cudaStream_t st; std::chrono::steady_clock::time_point t0; const char* what;
  Trace(cudaStream_t s, const char* w) : on(getenv("GLIO_TRACE") != nullptr), st(s), t0(std::chrono::steady_clock::now()), what(w) {}
  void mark(const char* label) { if (!on) return; cudaStreamSynchronize(st); fprintf(stderr, "[glio trace] %s %-18s %8.1f us\n", what, label, std::chrono::duration<double, std::micro>(std::chrono::steady_clock::now() - t0).count()); }
};

// the last error of the calling thread: glio_last_error(NULL)
thread_local std::string tl_err;

// An entry point runs on its context's GPU and hands the calling thread back on the device it came with, so a caller that
// drives contexts on several GPUs (or allocates with torch's current device) keeps its own choice of device.
struct DeviceGuard {
  int prev = -1;
  DeviceGuard() { if (cudaGetDevice(&prev) != cudaSuccess) { cudaGetLastError(); prev = -1; } }
  cudaError_t use(int device) const { return device == prev ? cudaSuccess : cudaSetDevice(device); }
  ~DeviceGuard() {
    int now = -1;
    if (prev >= 0 && cudaGetDevice(&now) == cudaSuccess && now != prev) cudaSetDevice(prev);
  }
};

template <class F>
int guarded(glio_ctx* ctx, F&& f) {
  DeviceGuard dev;
  try {
    if (ctx) GLIO_CUDA_TRY(dev.use(ctx->device));
    f();
    return GLIO_OK;
  } catch (const Error& e) {
    if (ctx) ctx->err = e.msg;
    tl_err = e.msg;
    return e.code;
  } catch (const std::exception& e) {
    if (ctx) ctx->err = e.what();
    tl_err = e.what();
    return GLIO_ERR_STATE;
  }
}

// true when p is memory of the context's GPU that its kernels can address
bool on_ctx_device(const glio_ctx* c, const void* p) {
  cudaPointerAttributes at{};
  if (cudaPointerGetAttributes(&at, p) != cudaSuccess) { cudaGetLastError(); return false; }
  return (at.type == cudaMemoryTypeDevice || at.type == cudaMemoryTypeManaged) && at.device == c->device;
}

// bring `n` points (stride floats each) to the device; returns the device pointer to read from
const float* stage_points(glio_ctx* c, DevBuf<float>& buf, const float* xyz, int64_t n, int stride, int mem) {
  GLIO_REQUIRE(xyz != nullptr && n > 0, GLIO_ERR_ARG, "null or empty point array");
  GLIO_REQUIRE(stride >= 3 && stride <= 64, GLIO_ERR_ARG, "stride_floats must be in [3,64]");
  if (mem == GLIO_DEVICE) return xyz;
  buf.reserve((size_t)n * stride);
  GLIO_CUDA_TRY(cudaMemcpyAsync(buf.p, xyz, (size_t)n * stride * sizeof(float), cudaMemcpyHostToDevice, c->st));
  return buf.p;
}

// the same into a point set (main stream)
void stage_points(glio_ctx* c, PointSet& ps, const float* xyz, int64_t n, int stride, int mem) {
  ps.ptr = stage_points(c, ps.own, xyz, n, stride, mem);
  ps.n = n; ps.stride = stride;
}

// Host clouds travel on the copy stream, so the next window's upload can overlap a running solve; device clouds are borrowed.
// Per call the copy stream waits once for the main stream (nothing queued there may still read the buffers) and one event,
// which the next association waits for, marks the end of all the uploads.
void upload_points_async(glio_ctx* c, const std::vector<PointSet*>& sets, const float* const* xyz, const int64_t* n, int stride, int mem) {
  if (mem != GLIO_DEVICE) {
    GLIO_CUDA_TRY(cudaEventRecord(c->ev_main, c->st));
    GLIO_CUDA_TRY(cudaStreamWaitEvent(c->st_copy, c->ev_main, 0));
  }
  for (size_t i = 0; i < sets.size(); ++i) {
    PointSet& ps = *sets[i];
    if (mem == GLIO_DEVICE) ps.ptr = xyz[i];
    else {
      ps.own.reserve((size_t)n[i] * stride);
      GLIO_CUDA_TRY(cudaMemcpyAsync(ps.own.p, xyz[i], (size_t)n[i] * stride * sizeof(float), cudaMemcpyHostToDevice, c->st_copy));
      ps.ptr = ps.own.p;
    }
    ps.n = n[i]; ps.stride = stride;
  }
  if (mem != GLIO_DEVICE) { GLIO_CUDA_TRY(cudaEventRecord(c->ev_scans, c->st_copy)); c->scans_pending = true; }
}

// one association segment: the points of ps from global query index off on, moved by pose = (t, q)
SegDesc make_seg(const PointSet& ps, int64_t off, const double* pose) {
  SegDesc sd;
  sd.src = ps.ptr; sd.stride = ps.stride; sd.count = ps.n; sd.offset = off;
  for (int k = 0; k < 3; ++k) sd.t[k] = pose[k];
  for (int k = 0; k < 4; ++k) sd.q[k] = pose[3 + k];
  return sd;
}

// the x, y, z of n float4 into xyz (3 floats each) and, when w is set, their w
void unpack_float4(const float4* h, int64_t n, float* xyz, float* w = nullptr) {
  for (int64_t i = 0; i < n; ++i) {
    if (xyz) { xyz[3 * i] = h[i].x; xyz[3 * i + 1] = h[i].y; xyz[3 * i + 2] = h[i].z; }
    if (w) w[i] = h[i].w;
  }
}

// copy-out of a plane match list (glio_get_matches: nsd; glio_batch_get_matches: nc), every array nullable
void copy_matches_out(glio_ctx* c, const CorrList& l, int64_t capacity, float* cp, float* weight, float* nsd, double* nc, int32_t* src,
                      int64_t* n_out) {
  const int64_t n = l.n;
  if (n_out) *n_out = n;
  GLIO_REQUIRE(capacity >= n, GLIO_ERR_ARG, "capacity smaller than the match count");
  if (n == 0) return;
  std::vector<float4> h(cp || weight ? n : 0);
  if (!h.empty()) GLIO_CUDA_TRY(cudaMemcpyAsync(h.data(), l.rec.cpw.p, n * sizeof(float4), cudaMemcpyDeviceToHost, c->st));
  if (nsd) GLIO_CUDA_TRY(cudaMemcpyAsync(nsd, l.rec.nsd.p, n * sizeof(float4), cudaMemcpyDeviceToHost, c->st));
  if (nc) GLIO_CUDA_TRY(cudaMemcpyAsync(nc, l.rec.nc.p, 6 * n * sizeof(double), cudaMemcpyDeviceToHost, c->st));
  if (src) GLIO_CUDA_TRY(cudaMemcpyAsync(src, l.src.p, n * sizeof(int32_t), cudaMemcpyDeviceToHost, c->st));
  GLIO_CUDA_TRY(cudaStreamSynchronize(c->st));
  unpack_float4(h.data(), (int64_t)h.size(), cp, weight);
}

// upload of n > 0 plane matches into a cleared list: cp and weight, with nsd (4 floats per match) into a slot's list, where src is
// 0 (glio_set_matches), or nc (6 doubles per match) into a pair's, where src is the match index (glio_batch_set_pair_matches)
void upload_matches(glio_ctx* c, CorrList& l, int64_t n, const float* cp, const float* weight, const float* nsd, const double* nc) {
  const bool window = l.kind == CORR_WINDOW_PLANES;
  std::vector<float4> h0(n), h1(window ? n : 0);
  std::vector<int32_t> hs(window ? 0 : n);
  for (int64_t i = 0; i < n; ++i) {
    h0[i] = make_float4(cp[3 * i], cp[3 * i + 1], cp[3 * i + 2], weight[i]);
    if (window) h1[i] = make_float4(nsd[4 * i], nsd[4 * i + 1], nsd[4 * i + 2], nsd[4 * i + 3]);
    else hs[i] = (int32_t)i;
  }
  l.reserve(n);
  GLIO_CUDA_TRY(cudaMemcpyAsync(l.rec.cpw.p, h0.data(), n * sizeof(float4), cudaMemcpyHostToDevice, c->st));
  if (window) {
    GLIO_CUDA_TRY(cudaMemcpyAsync(l.rec.nsd.p, h1.data(), n * sizeof(float4), cudaMemcpyHostToDevice, c->st));
    GLIO_CUDA_TRY(cudaMemsetAsync(l.src.p, 0, n * sizeof(int32_t), c->st));
  } else {
    GLIO_CUDA_TRY(cudaMemcpyAsync(l.rec.nc.p, nc, 6 * n * sizeof(double), cudaMemcpyHostToDevice, c->st));
    GLIO_CUDA_TRY(cudaMemcpyAsync(l.src.p, hs.data(), n * sizeof(int32_t), cudaMemcpyHostToDevice, c->st));
  }
  GLIO_CUDA_TRY(cudaStreamSynchronize(c->st));
  l.n = n;
}

// glio_select / glio_batch_select: the plane matches keep[0..n) become the list's selection (n < 0: no selection)
void select_keep(glio_ctx* c, CorrList& l, const int32_t* keep, int64_t n) {
  if (n < 0) { l.set_selection(-1); return; }
  GLIO_REQUIRE(n == 0 || keep, GLIO_ERR_ARG, "null selection list");
  l.set_selection(n);
  if (n == 0) return;
  l.keep.reserve(n); c->d_bad.reserve(1); l.sel.reserve(l.kind, n);
  GLIO_CUDA_TRY(cudaMemcpyAsync(l.keep.p, keep, n * sizeof(int32_t), cudaMemcpyHostToDevice, c->st));
  GLIO_CUDA_TRY(cudaMemsetAsync(c->d_bad.p, 0, sizeof(int), c->st));
  gather_selection(l.keep.p, n, l.n, l.rec.cpw.p, l.rec.nsd.p, l.rec.nc.p, l.sel.cpw.p, l.sel.nsd.p, l.sel.nc.p, c->d_bad.p, c->st, c->lc);
  int bad = 0;
  GLIO_CUDA_TRY(cudaMemcpyAsync(&bad, c->d_bad.p, sizeof(int), cudaMemcpyDeviceToHost, c->st));
  GLIO_CUDA_TRY(cudaStreamSynchronize(c->st));
  if (bad) { l.set_selection(-1); throw Error{GLIO_ERR_ARG, "selection index out of range"}; }
}

// the *_get_selection calls: the selection's record indices (a count query when out is NULL)
void copy_selection(glio_ctx* c, const CorrList& l, int64_t cap, int32_t* out, int64_t* n) {
  if (n) *n = l.n_sel;
  if (l.n_sel <= 0 || !out) return;
  GLIO_REQUIRE(cap >= l.n_sel, GLIO_ERR_ARG, "capacity smaller than the selection");
  GLIO_CUDA_TRY(cudaMemcpyAsync(out, l.keep.p, l.n_sel * sizeof(int32_t), cudaMemcpyDeviceToHost, c->st));
  GLIO_CUDA_TRY(cudaStreamSynchronize(c->st));
}

// queues the copy of the association's per-query views [off, off + q) from the work space into d (fit: nfit doubles per query)
void capture_debug(glio_ctx* c, AssocDebug& d, const AssocWork& w, const double* fit, int nfit, int64_t off, int64_t q) {
  d.status.reserve(q); d.idx5.reserve(5 * q); d.sqd5.reserve(5 * q); d.pm.reserve(q); d.fit.reserve(nfit * q);
  GLIO_CUDA_TRY(cudaMemcpyAsync(d.status.p, w.status + off, q, cudaMemcpyDeviceToDevice, c->st));
  GLIO_CUDA_TRY(cudaMemcpyAsync(d.idx5.p, w.idx5 + 5 * off, 5 * q * sizeof(int32_t), cudaMemcpyDeviceToDevice, c->st));
  GLIO_CUDA_TRY(cudaMemcpyAsync(d.sqd5.p, w.sqd5 + 5 * off, 5 * q * sizeof(float), cudaMemcpyDeviceToDevice, c->st));
  GLIO_CUDA_TRY(cudaMemcpyAsync(d.pm.p, w.pm + off, q * sizeof(float4), cudaMemcpyDeviceToDevice, c->st));
  GLIO_CUDA_TRY(cudaMemcpyAsync(d.fit.p, fit + nfit * off, nfit * q * sizeof(double), cudaMemcpyDeviceToDevice, c->st));
  d.Q = q;
}

void ensure_work(glio_ctx* c, int64_t Qt, bool pair, bool keep_debug) {
  c->w_pm.reserve((size_t)Qt); c->w_pmq.reserve((size_t)Qt); c->w_seg.reserve((size_t)Qt);
  c->w_status.reserve((size_t)Qt); c->w_weight.reserve((size_t)Qt);
  c->w_flags.reserve((size_t)Qt + 1); c->w_pos.reserve((size_t)Qt + 1);
  c->w_knn_idx.reserve((size_t)Qt * 5); c->w_knn_sqd.reserve((size_t)Qt * 5);
  if (pair) c->w_nc.reserve((size_t)Qt * 6); else c->w_nsd.reserve((size_t)Qt);
  if (keep_debug) { c->w_idx5.reserve((size_t)Qt * 5); c->w_sqd5.reserve((size_t)Qt * 5); c->w_plane.reserve((size_t)Qt * 4); }
}

AssocWork make_work(glio_ctx* c, int64_t Qt, bool pair, bool keep_debug) {
  AssocWork w{};
  w.Qt = Qt; w.pm = c->w_pm.p; w.pmq = c->w_pmq.p; w.seg = c->w_seg.p; w.status = c->w_status.p;
  w.knn_idx = c->w_knn_idx.p; w.knn_sqd = c->w_knn_sqd.p;
  w.nsd = pair ? nullptr : c->w_nsd.p; w.weight = c->w_weight.p; w.normal_cent = pair ? c->w_nc.p : nullptr;
  if (keep_debug) { w.idx5 = c->w_idx5.p; w.sqd5 = c->w_sqd5.p; w.plane = c->w_plane.p; }
  return w;
}

// run scan-to-map association of the given slots against `grid` with `gates` (one launch), compact, fetch counts.  The
// context's association workspace is scratch; the map, gates and slots are the caller's (the window path passes the
// context's own, the odometry its own).
void associate_slots(glio_ctx* c, const GridBuild& grid, const AssocGates& gates, bool keep_debug, const std::vector<Slot*>& slots,
                     const std::vector<std::array<double, 7>>& lidar_poses, int64_t* n_match) {
  if (c->scans_pending) { GLIO_CUDA_TRY(cudaStreamWaitEvent(c->st, c->ev_scans, 0)); c->scans_pending = false; }
  Trace tr(c->st, "associate");
  const int nseg = (int)slots.size();
  std::vector<SegDesc> segs(nseg);
  std::vector<CompactDst> dst(nseg);
  int64_t Qt = 0;
  for (int s = 0; s < nseg; ++s) {
    Slot& sl = *slots[s];
    GLIO_REQUIRE(sl.scan.n > 0 && sl.scan.ptr, GLIO_ERR_STATE, "slot has no scan");
    segs[s] = make_seg(sl.scan, Qt, lidar_poses[s].data());
    dst[s] = sl.planes.plane_dst(sl.scan.n);
    Qt += sl.scan.n;
  }
  ensure_work(c, Qt, false, keep_debug);
  c->d_segs.reserve(nseg); c->d_dst.reserve(nseg); c->d_counts.reserve(nseg); c->h_counts.reserve(nseg);
  GLIO_CUDA_TRY(cudaMemcpyAsync(c->d_segs.p, segs.data(), nseg * sizeof(SegDesc), cudaMemcpyHostToDevice, c->st));
  GLIO_CUDA_TRY(cudaMemcpyAsync(c->d_dst.p, dst.data(), nseg * sizeof(CompactDst), cudaMemcpyHostToDevice, c->st));
  AssocWork w = make_work(c, Qt, false, keep_debug);
  tr.mark("setup+h2d");
  assoc_run(grid, c->d_segs.p, nseg, w, gates, nullptr, 0, c->cell_count, c->cell_pos, c->scan_tmp, c->st, c->lc);
  tr.mark("assoc_run");
  compact_run(w, c->d_segs.p, nseg, c->w_flags.p, c->w_pos.p, c->scan_tmp, c->d_dst.p, c->d_counts.p, c->st, c->lc);
  tr.mark("compact");
  GLIO_CUDA_TRY(cudaMemcpyAsync(c->h_counts.p, c->d_counts.p, nseg * sizeof(int), cudaMemcpyDeviceToHost, c->st));
  if (keep_debug)
    for (int s = 0; s < nseg; ++s) capture_debug(c, slots[s]->dbg, w, w.plane, 4, segs[s].offset, slots[s]->scan.n);
  GLIO_CUDA_TRY(cudaStreamSynchronize(c->st));
  for (int s = 0; s < nseg; ++s) {
    CorrList& l = slots[s]->planes;
    l.n = c->h_counts.p[s];
    if (n_match) n_match[s] = l.n;
  }
  tr.mark("done");
}

// the context's own window association: its map, its gates, slots 0..
void associate_ctx_slots(glio_ctx* c, const std::vector<int>& ids, const std::vector<std::array<double, 7>>& lidar_poses, int64_t* n_match) {
  GLIO_REQUIRE(c->map.valid, GLIO_ERR_STATE, "glio_set_map must be called before association");
  std::vector<Slot*> sl;
  for (int id : ids) sl.push_back(&c->slot(id));
  const AssocGates gates{c->prm.kd_max_radius, c->prm.surf_dist_thres, c->prm.weight_min};
  associate_slots(c, c->map.grid, gates, c->prm.keep_debug != 0, sl, lidar_poses, n_match);
}

// The work items of one evaluation kernel, one block each: every owner's (keyframe's or pair's) residuals cut into runs, owners in
// order.  start[o] = first item of owner o, start[owners] = the item count.
template <class Item>
struct ItemPlan {
  std::vector<Item> items;
  std::vector<int> start;
  explicit ItemPlan(int owners) : start(owners + 1, 0) {}
  // owner o (called once per owner, in order) with n residuals, in runs of per; item(first, count) makes one run's item
  template <class MakeItem>
  void cut(int o, int64_t n, int64_t per, MakeItem item) {
    for (int64_t f = 0; f < n; f += per) items.push_back(item(f, (int32_t)std::min<int64_t>(per, n - f)));
    start[o + 1] = (int)items.size();
  }
  // items and start table into d_items / d_start, d_partials sized for nacc sums per item; synchronises (both are host vectors)
  void upload(glio_ctx* c, DevBuf<Item>& d_items, DevBuf<int>& d_start, DevBuf<double>& d_partials, int nacc) const {
    d_items.reserve(items.size() + 1); d_start.reserve(start.size()); d_partials.reserve((items.size() + 1) * nacc);
    if (!items.empty()) GLIO_CUDA_TRY(cudaMemcpyAsync(d_items.p, items.data(), items.size() * sizeof(Item), cudaMemcpyHostToDevice, c->st));
    GLIO_CUDA_TRY(cudaMemcpyAsync(d_start.p, start.data(), start.size() * sizeof(int), cudaMemcpyHostToDevice, c->st));
    GLIO_CUDA_TRY(cudaStreamSynchronize(c->st));
  }
};

// the ticket of the unary kernels' last-block election, zero between launches
void init_ticket(glio_ctx* c) {
  if (!c->d_ticket.p) { c->d_ticket.reserve(1); GLIO_CUDA_TRY(cudaMemsetAsync(c->d_ticket.p, 0, sizeof(unsigned int), c->st)); }
}

// K2 work items of the given slots (slot k = keyframe k, nullptr = none)
ItemPlan<EvalItem> plan_items(const std::vector<const Slot*>& slots, int eval_slots) {
  const int W = (int)slots.size();
  auto active = [](const Slot* sl) { return sl ? sl->planes.active() : CorrView{}; };
  // item size: the whole launch should be about one wave of 2 resident blocks per SM (less per-item reduction
  // overhead, no wave-quantisation tail), but never below GLIO_ITEM_MAX residuals per item
  int64_t n_total = 0;
  for (int k = 0; k < W; ++k) n_total += active(slots[k]).n;
  int64_t item_size = (n_total + eval_slots - 1) / std::max(eval_slots, 1);
  item_size = std::max<int64_t>(GLIO_ITEM_MAX, ((item_size + 255) / 256) * 256);
  ItemPlan<EvalItem> plan(W);
  for (int k = 0; k < W; ++k) {
    const CorrView v = active(slots[k]);
    const int64_t parts = std::max<int64_t>(1, (v.n + item_size - 1) / item_size);
    const int64_t per = ((v.n + parts - 1) / parts + 255) / 256 * 256;      // equal, 256-aligned parts
    plan.cut(k, v.n, per, [&](int64_t f, int32_t count) { return EvalItem{v.cpw + f, v.nsd + f, count, k}; });
  }
  return plan;
}

// The work items of one evaluation target in device memory, and the constants its residuals are evaluated with.
struct EvalTarget {
  const EvalItem* d_items; int n_items; const int* d_kf_item_start; double* d_partials;
  EvalParams ep;
};

// uploads a K2 plan into the given device buffers; reserves the context's per-evaluation buffers for W keyframes
void upload_items(glio_ctx* c, int W, const ItemPlan<EvalItem>& plan, DevBuf<EvalItem>& d_items, DevBuf<int>& d_start,
                  DevBuf<double>& d_partials) {
  c->d_out.reserve((size_t)W * GLIO_NACC); c->h_out.reserve((size_t)W * GLIO_NACC);
  c->d_poses.reserve((size_t)W * 7); c->h_poses.reserve((size_t)W * 7);
  init_ticket(c);
  plan.upload(c, d_items, d_start, d_partials, GLIO_NACC);
}

void build_items(glio_ctx* c, int W) {
  if (!c->items_dirty && c->items_W == W) return;
  std::vector<const Slot*> sl(W, nullptr);
  for (int k = 0; k < W && (size_t)k < c->slots.size(); ++k) sl[k] = c->slots[k].get();
  const ItemPlan<EvalItem> plan = plan_items(sl, c->eval_slots);
  c->n_items = (int)plan.items.size();
  upload_items(c, W, plan, c->d_items, c->d_kf_item_start, c->d_partials);
  c->items_dirty = false;
  c->items_W = W;
}

EvalParams eval_params(const glio_ctx* c) {
  EvalParams ep;
  for (int k = 0; k < 4; ++k) ep.q_lb[k] = c->prm.q_lb[k];
  for (int k = 0; k < 3; ++k) ep.t_lb[k] = c->prm.t_lb[k];
  ep.lidar_const = c->prm.lidar_const;
  ep.huber_delta = c->prm.huber_delta;
  ep.unit_score = c->prm.unit_score != 0 ? 1 : 0;
  return ep;
}

// the W x 28 layout (per keyframe: 21 upper-triangular H, 6 g, 1 cost) as full 6x6 H, g and per-keyframe cost, each nullable
void unpack_blocks(const double* o28, int W, double* H, double* g, double* cost) {
  for (int k = 0; k < W; ++k) {
    const double* o = o28 + (size_t)k * GLIO_NACC;
    if (H) {
      int idx = 0;
      for (int p = 0; p < 6; ++p) for (int q = p; q < 6; ++q) { H[36 * k + 6 * p + q] = o[idx]; H[36 * k + 6 * q + p] = o[idx]; ++idx; }
    }
    if (g) for (int p = 0; p < 6; ++p) g[6 * k + p] = o[21 + p];
    if (cost) cost[k] = o[27];
  }
}

void fill_summary(const SolverSummary& S, int n, glio_solver_summary* summary, glio_iteration* iter_log, int iter_cap, double* step_log, int64_t step_cap) {
  if (summary) {
      memset(summary, 0, sizeof(*summary));
      summary->termination = S.termination; summary->num_iterations = (int)S.iterations.size();
      summary->num_successful_steps = S.num_successful_steps; summary->num_unsuccessful_steps = S.num_unsuccessful_steps;
      summary->num_evaluations = S.num_evaluations; summary->num_jacobian_evaluations = S.num_jacobian_evaluations;
      summary->num_linear_solves = S.num_linear_solves; summary->num_valid_steps = (int)(S.steps.size() / (size_t)n);
      summary->initial_cost = S.initial_cost; summary->final_cost = S.final_cost;
      summary->eval_seconds = S.eval_seconds; summary->linear_solver_seconds = S.linear_solver_seconds; summary->total_seconds = S.total_seconds;
      snprintf(summary->message, sizeof(summary->message), "%s", S.message.c_str());
    }
    if (iter_log) for (int i = 0; i < (int)S.iterations.size() && i < iter_cap; ++i) {
      const IterationRecord& r = S.iterations[i];
      glio_iteration& q = iter_log[i];
      q.iteration = r.iteration; q.step_is_valid = r.step_is_valid; q.step_is_successful = r.step_is_successful; q.reserved = 0;
      q.cost = r.cost; q.cost_change = r.cost_change; q.gradient_max_norm = r.gradient_max_norm; q.gradient_norm = r.gradient_norm;
      q.step_norm = r.step_norm; q.relative_decrease = r.relative_decrease; q.trust_region_radius = r.trust_region_radius; q.mu = r.mu;
    }
    if (step_log) memcpy(step_log, S.steps.data(), sizeof(double) * (size_t)std::min<int64_t>(step_cap, (int64_t)S.steps.size()));
}

// device evaluation of all active unary residuals -> c->h_out (W x 28: 21 upper-tri H, 6 g, 1 cost), synchronised
// launch half: returns the epoch to wait for (0: nothing was launched, h_out already holds zeros).  tgt = nullptr evaluates the
// context's own slots with its glio_params; otherwise the target's items and constants (the odometry's).
// An asynchronous marginalisation owns the pinned pose and result buffers (h_poses, h_out) until its worker has copied the
// device result: its kernel (and, above EV_MAXW keyframes, its pose upload) may still be queued.  Wait for that copy.
void wait_marg_copied(glio_ctx* c) {
  if (!c->marg_pending) return;
  while (!c->marg_pending->copied.load(std::memory_order_acquire)) {
#if defined(__x86_64__)
    __builtin_ia32_pause();
#endif
  }
}

// K2e work items of slots 0..W-1 (GLIO_ITEM_MAX residuals each, keyframe order) over their active edges
ItemPlan<EdgeItem> plan_edge_items(const glio_ctx* c, int W) {
  ItemPlan<EdgeItem> plan(W);
  for (int k = 0; k < W; ++k) {
    const CorrView e = (size_t)k < c->slots.size() && c->slots[k] ? c->slots[k]->edges.active() : CorrView{};
    plan.cut(k, e.n, GLIO_ITEM_MAX, [&](int64_t f, int32_t count) { return EdgeItem{e.cpw + f, e.pa + f, e.pb + f, count, k}; });
  }
  return plan;
}

// Queues the edge blocks of one solve / marginalisation evaluation (poses already in c->h_poses): the pose upload, K2e and the copy
// of its result into c->h_eout, all on the main stream ahead of K2.  Returns false when slots 0..W-1 hold no edge.
bool edge_blocks_launch(glio_ctx* c, int W, int jac_kind, bool want_jac) {
  if (c->edge_items_dirty || c->edge_items_W != W) {
    const ItemPlan<EdgeItem> plan = plan_edge_items(c, W);
    plan.upload(c, c->se_items, c->se_start, c->se_part, GLIO_NACC);
    c->n_edge_items = (int)plan.items.size(); c->edge_items_W = W; c->edge_items_dirty = false;
  }
  if (c->n_edge_items == 0) return false;
  c->se_out.reserve((size_t)W * GLIO_NACC); c->se_poses.reserve((size_t)W * 7); c->h_eout.reserve((size_t)W * GLIO_NACC);
  init_ticket(c);
  GLIO_CUDA_TRY(cudaMemcpyAsync(c->se_poses.p, c->h_poses.p, (size_t)W * 7 * sizeof(double), cudaMemcpyHostToDevice, c->st));
  eval_edge_run(c->se_items.p, c->n_edge_items, W, c->se_poses.p, eval_params(c), jac_kind, want_jac, c->se_part.p, c->se_out.p, c->se_start.p,
                c->d_ticket.p, c->st, c->lc);
  GLIO_CUDA_TRY(cudaMemcpyAsync(c->h_eout.p, c->se_out.p, (size_t)W * GLIO_NACC * sizeof(double), cudaMemcpyDeviceToHost, c->st));
  return true;
}

void add_edge_blocks(glio_ctx* c, int W) {
  for (size_t i = 0; i < (size_t)W * GLIO_NACC; ++i) c->h_out.p[i] += c->h_eout.p[i];
}

// with_edges: a solve or marginalisation evaluation of the context's own slots, which adds their edge blocks when
// glio_window_use_edges is on
unsigned int eval_unary_launch(glio_ctx* c, int W, const double* poses_body, int jac_kind, bool want_jac, const EvalTarget* tgt = nullptr,
                               bool with_edges = false) {
  wait_marg_copied(c);
  const bool own_slots = tgt == nullptr;
  EvalTarget own{};
  if (!tgt) {
    build_items(c, W);
    own = EvalTarget{c->d_items.p, c->n_items, c->d_kf_item_start.p, c->d_partials.p, eval_params(c)};
    tgt = &own;
  }
  // Zero-copy round trip: the W poses travel in the kernel parameters, the last block writes the W x 28 result into
  // pinned host memory and raises an epoch flag the host spins on.  This replaces H2D copy + launch + D2H copy +
  // stream synchronise on the per-iteration path, and lets the caller evaluate its host factors while the kernel runs.
  memcpy(c->h_poses.p, poses_body, (size_t)W * 7 * sizeof(double));
  const bool edges = with_edges && own_slots && c->use_edges && edge_blocks_launch(c, W, jac_kind, want_jac);
  if (tgt->n_items <= 0) {
    GLIO_CUDA_TRY(cudaStreamSynchronize(c->st));
    memset(c->h_out.p, 0, (size_t)W * GLIO_NACC * sizeof(double));
    if (edges) add_edge_blocks(c, W);
    return 0u;
  }
  if (!c->h_flag.p) { c->h_flag.reserve(4); memset(c->h_flag.p, 0, 4 * sizeof(unsigned int)); }
  const unsigned int epoch = ++c->eval_epoch;
  if (edges) { c->edge_epoch = epoch; c->edge_W = W; }
  if (W > EV_MAXW) GLIO_CUDA_TRY(cudaMemcpyAsync(c->d_poses.p, c->h_poses.p, (size_t)W * 7 * sizeof(double), cudaMemcpyHostToDevice, c->st));
  eval_unary_run(tgt->d_items, tgt->n_items, W, c->d_poses.p, tgt->ep, jac_kind, want_jac, tgt->d_partials, c->h_out.p,
                 tgt->d_kf_item_start, c->d_ticket.p, c->st, c->lc, c->h_flag.p, epoch, c->h_poses.p);
  (void)cudaStreamQuery(c->st);            // pushes the launch to the device now (otherwise it may sit in the driver's queue until the next API call)
  return epoch;
}

void eval_unary_wait(glio_ctx* c, unsigned int epoch) {
  if (!epoch) return;
  volatile unsigned int* flag = c->h_flag.p;
  const auto t0 = std::chrono::steady_clock::now();
  for (unsigned long long spins = 0; *flag != epoch; ++spins) {
#if defined(__x86_64__)
    __builtin_ia32_pause();
#endif
    if ((spins & 0x3ffull) == 0x3ffull) {
      const cudaError_t q = cudaStreamQuery(c->st);
      if (q != cudaSuccess && q != cudaErrorNotReady) GLIO_CUDA_TRY(q);
      if (q == cudaSuccess && *flag != epoch) throw Error{GLIO_ERR_CUDA, "eval_unary: kernel finished without raising the completion flag"};
      if (std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count() > 30.0) throw Error{GLIO_ERR_CUDA, "eval_unary: timed out waiting for the device"};
    }
  }
  std::atomic_thread_fence(std::memory_order_acquire);
  if (epoch == c->edge_epoch) add_edge_blocks(c, c->edge_W);   // K2e and its copy ran before K2 on the same stream
}

// device evaluation of all active unary residuals -> c->h_out (W x 28: 21 upper-tri H, 6 g, 1 cost), synchronised
void eval_unary_blocks(glio_ctx* c, int W, const double* poses_body, int jac_kind, bool want_jac) {
  eval_unary_wait(c, eval_unary_launch(c, W, poses_body, jac_kind, want_jac));
}

// Queues the read-out of an evaluation's n_diag diagonal and n_off off-diagonal block values: with reduce and a sharded run's hook,
// their sums over the ranks (the off values only with want_jac and n_off > 0), then their copies into pinned memory
void reduce_and_fetch(glio_ctx* c, bool reduce, bool want_jac, double* d_diag, double* h_diag, int64_t n_diag, double* d_off, double* h_off,
                      int64_t n_off, const char* diag_err, const char* off_err) {
  const bool hook = reduce && c->allreduce, off = want_jac && n_off > 0;
  GLIO_REQUIRE(!hook || c->allreduce(c->allreduce_user, d_diag, n_diag, (void*)c->st) == 0, GLIO_ERR_NCCL, diag_err);
  GLIO_REQUIRE(!hook || !off || c->allreduce(c->allreduce_user, d_off, n_off, (void*)c->st) == 0, GLIO_ERR_NCCL, off_err);
  GLIO_CUDA_TRY(cudaMemcpyAsync(h_diag, d_diag, (size_t)n_diag * sizeof(double), cudaMemcpyDeviceToHost, c->st));
  if (off) GLIO_CUDA_TRY(cudaMemcpyAsync(h_off, d_off, (size_t)n_off * sizeof(double), cudaMemcpyDeviceToHost, c->st));
}

// Device evaluation of the IMU blocks of list L -> L.h_diag (K x 241), L.h_off (n_pairs x 225), at the poses d_poses (already queued)
// and speed_bias, which is queued here; jac_kind 1 gives the ambient x, y, z quaternion columns.  With reduce (the batch list) the
// IMU buffers are summed over the ranks of a sharded run after whatever the caller queued before, one call per buffer.  Queued only;
// a synchronisation of the stream, or the completion flag of a K2 queued after it, makes the result visible.  Returns the
// off-diagonal block count.
int imu_blocks_launch(glio_ctx* c, ImuFactorList& L, int K, const double* d_poses, const double* speed_bias, int jac_kind, bool want_jac,
                      bool reduce) {
  const int Pi = (int)L.pairs.size();
  L.d_sb.reserve((size_t)K * 9); L.h_sb.reserve((size_t)K * 9);
  L.d_diag.reserve((size_t)K * GLIO_NACC_IMU_KF); L.h_diag.reserve((size_t)K * GLIO_NACC_IMU_KF);
  L.d_off.reserve((size_t)(Pi + 1) * 225); L.h_off.reserve((size_t)(Pi + 1) * 225);
  memcpy(L.h_sb.p, speed_bias, (size_t)K * 9 * sizeof(double));
  GLIO_CUDA_TRY(cudaMemcpyAsync(L.d_sb.p, L.h_sb.p, (size_t)K * 9 * sizeof(double), cudaMemcpyHostToDevice, c->st));
  eval_imu_run(L.d_f.p, L.d_fstart.p, Pi, K, L.max_kf + 1, L.d_inc_start.p, L.d_inc.p, d_poses, L.d_sb.p, jac_kind, want_jac, L.d_sums.p,
               L.d_diag.p, L.d_off.p, c->st, c->lc);
  reduce_and_fetch(c, reduce, want_jac, L.d_diag.p, L.h_diag.p, (int64_t)K * GLIO_NACC_IMU_KF, L.d_off.p, L.h_off.p, (int64_t)Pi * 225,
                   "allreduce hook failed (IMU diag)", "allreduce hook failed (IMU off)");
  return Pi;
}

// the half bandwidth of list L's blocks at 15 columns per keyframe: (the widest pair's span + 1) * 15 - 1, 0 for no pair
int imu_half_bandwidth(const ImuFactorList& L) {
  int span = 0;
  for (const auto& p : L.pairs) span = std::max(span, p.second - p.first);
  return span > 0 ? (span + 1) * 15 - 1 : 0;
}

// list L's blocks of an evaluation that has arrived into the 15-column band: the cost, then with want_jac each keyframe's 15 x 15
// lower triangle and g, then each pair's (a, b) block, stored transposed (rows of b, a < b)
void add_imu_blocks(const ImuFactorList& L, int K, bool want_jac, BandMat* H, double* g, double& ct) {
  for (int k = 0; k < K; ++k) ct += L.h_diag.p[(size_t)k * GLIO_NACC_IMU_KF + 240];
  if (!want_jac) return;
  const int w = H->hb + 1;
  double* a = H->a.data();
  for (int k = 0; k < K; ++k) {
    const double* o = L.h_diag.p + (size_t)k * GLIO_NACC_IMU_KF;
    for (int p = 0; p < 15; ++p) {
      double* row = a + (size_t)(15 * k + p) * w + (H->hb - p);
      for (int q = 0; q <= p; ++q) row[q] += o[15 * p + q];
      g[15 * k + p] += o[225 + p];
    }
  }
  for (size_t pi = 0; pi < L.pairs.size(); ++pi) {
    const int ka = L.pairs[pi].first, kb = L.pairs[pi].second;
    const double* ob = L.h_off.p + pi * 225;              // d2 cost / d x_a[p] d x_b[q]
    for (int q = 0; q < 15; ++q) { double* row = a + (size_t)(15 * kb + q) * w + (15 * ka - (15 * kb + q) + H->hb); for (int p = 0; p < 15; ++p) row[p] += ob[15 * p + q]; }
  }
}

// the W window poses into the device buffer the window's K2i reads, from pinned memory
void upload_window_imu_poses(glio_ctx* c, int W, const double* poses) {
  c->wimu_poses.reserve((size_t)W * 7); c->h_wimu_poses.reserve((size_t)W * 7);
  memcpy(c->h_wimu_poses.p, poses, (size_t)W * 7 * sizeof(double));
  GLIO_CUDA_TRY(cudaMemcpyAsync(c->wimu_poses.p, c->h_wimu_poses.p, (size_t)W * 7 * sizeof(double), cudaMemcpyHostToDevice, c->st));
}

// The window's IMU blocks at one solve evaluation (tangent columns): the poses and speed-bias states, K2i and the copies of its
// blocks into pinned memory, all queued on the main stream ahead of the K2 the caller queues next, whose completion flag covers them
void window_imu_launch(glio_ctx* c, int W, const double* poses, const double* speed_bias, bool want_jac) {
  wait_marg_copied(c);                   // a pending marginalisation's upload may still read the pinned buffers
  upload_window_imu_poses(c, W, poses);
  imu_blocks_launch(c, c->window_imu, W, c->wimu_poses.p, speed_bias, 0, want_jac, false);
}

// The marginalisation's IMU part (Estimator.cpp:2520-2534): the ImuFactor KF0 -> KF1 with the ambient x, y, z quaternion columns
// that ThreadsConstructA reads (MarginalizationFactor.cpp:3-29).  K2i runs over pair {0, 1} alone and its 706 sums are copied into
// c->h_wimu_marg, queued ahead of K2.  Factors that do not touch slot 0 take no part; an active factor (0, k), k != 1, is
// GLIO_ERR_ARG: its other speed-bias block is not in the marginalisation ordering.  Returns false when no active factor is (0, 1).
bool window_imu_marg_launch(glio_ctx* c, const double* poses, const double* speed_bias) {
  ImuFactorList& M = c->window_imu;
  GLIO_REQUIRE(!c->wimu_slot0_elsewhere, GLIO_ERR_ARG, "marginalisation: an active IMU factor joins slot 0 to a slot other than 1");
  const int p01 = c->wimu_pair01;
  if (p01 < 0) return false;
  wait_marg_copied(c);
  upload_window_imu_poses(c, 2, poses);
  M.d_sb.reserve(18); M.h_sb.reserve(18); c->h_wimu_marg.reserve(GLIO_NACC_IMU);
  memcpy(M.h_sb.p, speed_bias, 18 * sizeof(double));
  GLIO_CUDA_TRY(cudaMemcpyAsync(M.d_sb.p, M.h_sb.p, 18 * sizeof(double), cudaMemcpyHostToDevice, c->st));
  eval_imu_pair_sums_run(M.d_f.p, M.d_fstart.p + p01, 1, c->wimu_poses.p, M.d_sb.p, 1, true, M.d_sums.p, c->st, c->lc);
  GLIO_CUDA_TRY(cudaMemcpyAsync(c->h_wimu_marg.p, M.d_sums.p, GLIO_NACC_IMU * sizeof(double), cudaMemcpyDeviceToHost, c->st));
  return true;
}

// pair {0, 1}'s sums s (706: aa, bb, ab row-major, g) into A (N x N) and b at the marginalisation ordering, where KF0's
// [t, q, sb] is [0, 15) and KF1's [15, 30) (marg.h)
void add_marg_imu(std::vector<double>& A, std::vector<double>& b, int N, const double* s) {
  for (int p = 0; p < 15; ++p)
    for (int q = 0; q < 15; ++q) {
      A[(size_t)p * N + q] += s[15 * p + q];
      A[(size_t)(15 + p) * N + 15 + q] += s[225 + 15 * p + q];
      A[(size_t)p * N + 15 + q] += s[450 + 15 * p + q];
      A[(size_t)(15 + q) * N + p] += s[450 + 15 * p + q];
    }
  for (int l = 0; l < 30; ++l) b[l] += s[675 + l];
}

}  // namespace

extern "C" {

void glio_default_params(glio_params* p) {
  if (!p) return;
  memset(p, 0, sizeof(*p));
  p->kd_max_radius = 1.5; p->surf_dist_thres = 0.18; p->lidar_const = 7.5; p->weight_min = 0.3; p->huber_delta = 1.0;
  p->q_lb[0] = 1.0; p->t_lb[2] = 0.28;          // GLIO/config/config_urban_hk.yaml:90-97
  p->batch_max_radius = 1.5; p->batch_dist_thres = 0.18; p->batch_score = 2.5;
  p->cell_size = 0.f; p->keep_debug = 0; p->unit_score = 0;
}

int glio_create(int device, const glio_params* params, glio_ctx** out) {
  if (!out) return GLIO_ERR_ARG;
  *out = nullptr;
  glio_ctx* c = nullptr;
  int rc = guarded(nullptr, [&] {
    int ndev = 0;
    cudaError_t e = cudaGetDeviceCount(&ndev);
    if (e != cudaSuccess || ndev <= 0) throw Error{GLIO_ERR_NO_DEVICE, std::string("no CUDA device: ") + cudaGetErrorString(e) + " (glio_b200 has no CPU fallback)"};
    GLIO_REQUIRE(device >= 0 && device < ndev, GLIO_ERR_ARG, "device index out of range");
    GLIO_CUDA_TRY(cudaSetDevice(device));
    c = new glio_ctx();
    c->device = device;
    if (params) c->prm = *params; else glio_default_params(&c->prm);
    if (const char* e = getenv("GLIO_PTS_PER_CELL")) { const float v = (float)atof(e); if (v > 0.1f && v < 1000.f) c->pts_per_cell = v; }
    GLIO_CUDA_TRY(cudaStreamCreateWithFlags(&c->st, cudaStreamNonBlocking));
    GLIO_CUDA_TRY(cudaStreamCreateWithFlags(&c->st_copy, cudaStreamNonBlocking));
    GLIO_CUDA_TRY(cudaEventCreateWithFlags(&c->ev_scans, cudaEventDisableTiming));
    GLIO_CUDA_TRY(cudaEventCreateWithFlags(&c->ev_main, cudaEventDisableTiming));
    { int sms = kNumSMs; if (cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device) == cudaSuccess && sms > 0) c->eval_slots = 2 * sms; }
  });
  if (rc != GLIO_OK) { delete c; return rc; }
  *out = c;
  return GLIO_OK;
}

void glio_destroy(glio_ctx* c) {
  if (!c) return;
  DeviceGuard dev; dev.use(c->device);
  while (!c->odoms.empty()) glio_odom_destroy(c->odoms.back());   // an odometry still attached (it detaches itself)
  while (!c->loops.empty()) glio_loop_destroy(c->loops.back());   // likewise a loop object
  if (c->marg_thread.joinable()) {
    if (c->marg_pending) { glio_marg_prior* dropped = nullptr; glio_marg_job_wait(c->marg_pending, &dropped); if (dropped) glio_marg_prior_destroy(dropped); }
    { std::lock_guard<std::mutex> lk(c->marg_mu); c->marg_quit = true; }
    c->marg_cv.notify_one();
    c->marg_thread.join();
  }
  // nothing queued may still use the context's buffers when `delete c` frees them
  if (c->st_copy) cudaStreamSynchronize(c->st_copy);
  if (c->st) cudaStreamSynchronize(c->st);
  if (c->ev_map) cudaEventDestroy(c->ev_map);
  if (c->ev_sel) cudaEventDestroy(c->ev_sel);
  for (auto& r : c->lc.recs) { cudaEventDestroy(r.a); cudaEventDestroy(r.b); }
  for (auto& e : c->lc.pool) cudaEventDestroy(e);
  c->lc.recs.clear(); c->lc.pool.clear();
  if (c->ev_scans) cudaEventDestroy(c->ev_scans);
  if (c->ev_main) cudaEventDestroy(c->ev_main);
  if (c->st_copy) cudaStreamDestroy(c->st_copy);
  if (c->st) cudaStreamDestroy(c->st);
  delete c;
}

const char* glio_last_error(const glio_ctx* c) { return c ? c->err.c_str() : tl_err.c_str(); }

int glio_synchronize(glio_ctx* c) {
  if (!c) return GLIO_ERR_ARG;
  return guarded(c, [&] { GLIO_CUDA_TRY(cudaStreamSynchronize(c->st_copy)); GLIO_CUDA_TRY(cudaStreamSynchronize(c->st)); });
}
void* glio_stream(glio_ctx* c) { return c ? (void*)c->st : nullptr; }
int64_t glio_launch_count(const glio_ctx* c) { return c ? c->lc.n : 0; }

int glio_profile_enable(glio_ctx* c, int on) {
  if (!c) return GLIO_ERR_ARG;
  return guarded(c, [&] {
    GLIO_CUDA_TRY(cudaStreamSynchronize(c->st));
    for (auto& r : c->lc.recs) { c->lc.pool.push_back(r.a); c->lc.pool.push_back(r.b); }
    c->lc.recs.clear();
    c->lc.prof = on != 0;
    // events are created up front: cudaEventCreate inside the timed region would distort what is being measured
    if (on) while (c->lc.pool.size() < 16384) { cudaEvent_t e; GLIO_CUDA_TRY(cudaEventCreate(&e)); c->lc.pool.push_back(e); }
  });
}

int glio_profile_get(glio_ctx* c, const char* kernel_name, double* ms_total, int64_t* launches) {
  if (!c || !kernel_name) return GLIO_ERR_ARG;
  return guarded(c, [&] {
    GLIO_CUDA_TRY(cudaStreamSynchronize(c->st));
    double tot = 0; int64_t cnt = 0;
    for (auto& r : c->lc.recs) {
      if (strcmp(r.name, kernel_name) != 0) continue;
      float ms = 0.f;
      if (cudaEventElapsedTime(&ms, r.a, r.b) == cudaSuccess) { tot += ms; ++cnt; }
    }
    if (ms_total) *ms_total = tot;
    if (launches) *launches = cnt;
  });
}

int glio_get_stats(glio_ctx* c, int64_t* knn_fallback_queries, int /*reset*/) {
  if (!c) return GLIO_ERR_ARG;
  if (knn_fallback_queries) *knn_fallback_queries = 0;    // the box search has no second pass
  return GLIO_OK;
}

int glio_get_params(const glio_ctx* c, glio_params* out) {
  if (!c || !out) return GLIO_ERR_ARG;
  *out = c->prm;
  return GLIO_OK;
}

// direct upload of a slot's match list (association done elsewhere, e.g. by the unmodified Estimator): the Ceres shim
// uses this to move LidarPlaneNormFactor residual blocks onto the device.
int glio_set_matches(glio_ctx* c, int slot, const float* cp, const float* nsd, const float* weight, int64_t n) {
  if (!c) return GLIO_ERR_ARG;
  return guarded(c, [&] {
    CorrList& l = c->slot(slot).planes;
    l.clear();
    if (n <= 0) return;
    GLIO_REQUIRE(cp && nsd && weight, GLIO_ERR_ARG, "null match arrays");
    upload_matches(c, l, n, cp, weight, nsd, nullptr);
  });
}

int glio_get_match_counts(glio_ctx* c, int W, int64_t* n_match, int64_t* n_active) {
  if (!c) return GLIO_ERR_ARG;
  return guarded(c, [&] {
    for (int k = 0; k < W; ++k) {
      const CorrList& l = c->slot(k).planes;
      if (n_match) n_match[k] = l.n;
      if (n_active) n_active[k] = l.n_active();
    }
  });
}

void glio_lidar_pose(const glio_params* prm, const double pose_body[7], double t2[3], double q2[4]) {
  lidar_pose_in_map(prm->q_lb, prm->t_lb, pose_body, t2, q2);
}

}  // extern "C"

// M points on the device become the map's grid (glio_set_map, glio_set_edge_map and the local-map builds)
static void map_build(glio_ctx* c, FeatureMap& m, const float* d, int stride, int64_t M) {
  grid_build(m.grid, d, stride, M, nullptr, nullptr, c->prm.cell_size, c->pts_per_cell, c->st, c->lc);
  m.valid = true; m.n = M;
}

extern "C" {

int glio_set_map(glio_ctx* c, const float* xyz, int64_t M, int stride, int mem) {
  if (!c) return GLIO_ERR_ARG;
  return guarded(c, [&] {
    GLIO_REQUIRE(M >= 5, GLIO_ERR_ARG, "map needs at least 5 points");
    const float* d;
    if (mem != GLIO_DEVICE && c->pf_ptr == xyz && c->pf_M == M && c->pf_stride == stride) {
      // the upload was started by glio_map_prefetch: wait for it on the main stream, no second copy
      GLIO_CUDA_TRY(cudaStreamWaitEvent(c->st, c->ev_map, 0));
      std::swap(c->map.stage, c->map_stage2);
      d = c->map.stage.p;
    } else d = stage_points(c, c->map.stage, xyz, M, stride, mem);
    c->pf_ptr = nullptr;
    map_build(c, c->map, d, stride, M);
  });
}

// Start the host->device copy of the NEXT local map on the copy stream (returns at once).  A following glio_set_map with the same
// pointer, count and stride uses the staged copy.  The caller must not modify the host buffer until that glio_set_map.
int glio_map_prefetch(glio_ctx* c, const float* xyz, int64_t M, int stride) {
  if (!c) return GLIO_ERR_ARG;
  return guarded(c, [&] {
    GLIO_REQUIRE(xyz != nullptr && M >= 5 && stride >= 3 && stride <= 64, GLIO_ERR_ARG, "glio_map_prefetch: bad arguments");
    if (!c->ev_map) GLIO_CUDA_TRY(cudaEventCreateWithFlags(&c->ev_map, cudaEventDisableTiming));
    c->map_stage2.reserve((size_t)M * stride);
    GLIO_CUDA_TRY(cudaMemcpyAsync(c->map_stage2.p, xyz, (size_t)M * stride * sizeof(float), cudaMemcpyHostToDevice, c->st_copy));
    GLIO_CUDA_TRY(cudaEventRecord(c->ev_map, c->st_copy));
    c->pf_ptr = xyz; c->pf_M = M; c->pf_stride = stride;
  });
}

}  // extern "C"

// the context's two local maps (surf and corner) share these
static int localmap_clear(glio_ctx* c, FeatureMap& m) {
  return guarded(c, [&] {
    GLIO_CUDA_TRY(cudaStreamSynchronize(c->st));
    m.lm.clear();
  });
}

static int localmap_push(glio_ctx* c, FeatureMap& m, int at_front, const float* cloud_xyz, int64_t n, int stride, int mem, const double t[3],
                         const double q[4]) {
  return guarded(c, [&] {
    GLIO_REQUIRE(t && q, GLIO_ERR_ARG, "null pose");
    const float* d = stage_points(c, m.lm_stage, cloud_xyz, n, stride, mem);
    m.lm.push(at_front != 0, d, stride, n, t, q, c->st, c->lc);              // transformCloud: float(q*double(p)+t)
    if (mem != GLIO_DEVICE) GLIO_CUDA_TRY(cudaStreamSynchronize(c->st));    // the staging buffer is reused by the next push
  });
}

static int localmap_pop_front(glio_ctx* c, FeatureMap& m) {
  return guarded(c, [&] {
    GLIO_REQUIRE(!m.lm.frames.empty(), GLIO_ERR_STATE, "local map holds no keyframe cloud");
    m.lm.pop_front();
  });
}

// *surf_local_map += *recent_surf_keyframes[i] (Estimator.cpp:3605-3608), ds_filter_surf_map.filter (:3617-3618); leaf <= 0, or
// PCL's pass-through when the voxel grid would overflow, leaves the concatenation as it is.  name: "local map" or "corner local map"
static int localmap_build(glio_ctx* c, FeatureMap& m, const char* name, float leaf, int64_t* n_map) {
  return guarded(c, [&] {
    GLIO_REQUIRE(m.lm.n_points() >= 5, GLIO_ERR_STATE, std::string(name) + " needs at least 5 points");
    const float* pts = nullptr; int stride = 0; bool filtered = false;
    const int64_t n = m.lm.build(leaf, &pts, &stride, &filtered, c->st, c->lc);
    GLIO_REQUIRE(!filtered || n >= 5, GLIO_ERR_STATE, "down-sampled " + std::string(name) + " has fewer than 5 points");
    map_build(c, m, pts, stride, n);                                          // kd_tree_surf_local_map->setInputCloud
    if (n_map) *n_map = n;
  });
}

extern "C" {

// ---- local map maintenance on the device (Estimator.cpp:3529-3631 buildLocalMapWithLandMark, :3615-3618 downSampleCloud) ----
int glio_localmap_clear(glio_ctx* c) {
  if (!c) return GLIO_ERR_ARG;
  return localmap_clear(c, c->map);
}

int glio_localmap_push(glio_ctx* c, int at_front, const float* cloud_xyz, int64_t n, int stride, int mem, const double t[3], const double q[4]) {
  if (!c) return GLIO_ERR_ARG;
  return localmap_push(c, c->map, at_front, cloud_xyz, n, stride, mem, t, q);
}

int glio_localmap_pop_front(glio_ctx* c) {
  if (!c) return GLIO_ERR_ARG;
  return localmap_pop_front(c, c->map);
}

int glio_localmap_size(glio_ctx* c, int* n_frames, int64_t* n_points) {
  if (!c) return GLIO_ERR_ARG;
  if (n_frames) *n_frames = (int)c->map.lm.frames.size();
  if (n_points) *n_points = c->map.lm.n_points();
  return GLIO_OK;
}

int glio_localmap_build(glio_ctx* c, float leaf, int64_t* n_map) {
  if (!c) return GLIO_ERR_ARG;
  return localmap_build(c, c->map, "local map", leaf, n_map);
}

int glio_get_map(glio_ctx* c, int64_t capacity, float* xyz, int64_t* n_out) {
  if (!c) return GLIO_ERR_ARG;
  return guarded(c, [&] {
    GLIO_REQUIRE(c->map.valid, GLIO_ERR_STATE, "no map set");
    const int64_t n = std::min<int64_t>(capacity, c->map.n);
    if (n_out) *n_out = c->map.n;
    if (n <= 0 || !xyz) return;
    std::vector<float4> h((size_t)n);
    GLIO_CUDA_TRY(cudaMemcpyAsync(h.data(), c->map.grid.tmp4.p, (size_t)n * sizeof(float4), cudaMemcpyDeviceToHost, c->st));
    GLIO_CUDA_TRY(cudaStreamSynchronize(c->st));
    unpack_float4(h.data(), n, xyz);
  });
}

int glio_assoc_scan_to_map(glio_ctx* c, int slot, const float* scan_xyz, int64_t Q, int stride, int mem,
                           const double t[3], const double q[4], int64_t* n_match) {
  if (!c) return GLIO_ERR_ARG;
  return guarded(c, [&] {
    GLIO_REQUIRE(t && q, GLIO_ERR_ARG, "null pose");
    stage_points(c, c->slot(slot).scan, scan_xyz, Q, stride, mem);
    std::vector<std::array<double, 7>> lp(1);
    for (int k = 0; k < 3; ++k) lp[0][k] = t[k];
    for (int k = 0; k < 4; ++k) lp[0][3 + k] = q[k];
    associate_ctx_slots(c, std::vector<int>{slot}, lp, n_match);
  });
}

int glio_window_set_scans(glio_ctx* c, int W, const float* const* scans, const int64_t* Q, int stride, int mem) {
  if (!c) return GLIO_ERR_ARG;
  return guarded(c, [&] {
    GLIO_REQUIRE(W > 0 && scans && Q, GLIO_ERR_ARG, "bad window arguments");
    GLIO_REQUIRE(stride >= 3 && stride <= 64, GLIO_ERR_ARG, "stride_floats must be in [3,64]");
    // The call returns at once and the next association waits for the uploads.  The matches of the previous association stay
    // valid (they hold their own copies of the points), so the scans of the NEXT window can be handed over while the current
    // window is still being solved.
    std::vector<PointSet*> sets(W);
    for (int k = 0; k < W; ++k) {
      sets[k] = &c->slot(k).scan;
      GLIO_REQUIRE(scans[k] != nullptr && Q[k] > 0, GLIO_ERR_ARG, "null or empty point array");
    }
    upload_points_async(c, sets, scans, Q, stride, mem);
  });
}

// One keyframe's scan into one slot (copy stream for host buffers, like glio_window_set_scans): what a sliding window needs per
// new keyframe - the other W-1 scans are already resident.
int glio_window_set_scan(glio_ctx* c, int slot, const float* scan, int64_t Q, int stride, int mem) {
  if (!c) return GLIO_ERR_ARG;
  return guarded(c, [&] {
    GLIO_REQUIRE(scan != nullptr && Q > 0, GLIO_ERR_ARG, "null or empty point array");
    GLIO_REQUIRE(stride >= 3 && stride <= 64, GLIO_ERR_ARG, "stride_floats must be in [3,64]");
    upload_points_async(c, {&c->slot(slot).scan}, &scan, &Q, stride, mem);
  });
}

// slideWindow (GLIO/src/Estimator.cpp: the oldest keyframe leaves, every other one moves down one slot): O(1) per slot, no
// copies; the matches, corner scans and edges of the slots move with them.  The new keyframe's scan then goes into slot W-1 with
// glio_window_set_scan (and its corner scan with glio_window_set_edge_scan).
int glio_window_slide(glio_ctx* c, int W) {
  if (!c) return GLIO_ERR_ARG;
  return guarded(c, [&] {
    GLIO_REQUIRE(W >= 2 && W <= 4096, GLIO_ERR_ARG, "bad window size");
    c->slot(W - 1);
    GLIO_CUDA_TRY(cudaStreamSynchronize(c->st_copy));
    std::unique_ptr<Slot> first = std::move(c->slots[0]);
    for (int k = 0; k + 1 < W; ++k) c->slots[k] = std::move(c->slots[k + 1]);
    c->slots[W - 1] = std::move(first);                       // its buffers are reused by the next upload
    if (c->slots[W - 1]) {
      Slot& s = *c->slots[W - 1];
      s.scan.clear(); s.planes.clear();
      s.corners.clear(); s.edges.clear();                 // the dropped keyframe's corners and edges leave with it
      s.dbg.Q = 0; s.edge_dbg.Q = 0;                      // and its debug views
    }
    c->items_dirty = true; c->edge_items_dirty = true;    // the plans follow the slots' order, which changed
  });
}

// The corner scan of one keyframe, with the upload rules of glio_window_set_scan.
int glio_window_set_edge_scan(glio_ctx* c, int slot, const float* xyz, int64_t Q, int stride, int mem) {
  if (!c) return GLIO_ERR_ARG;
  return guarded(c, [&] {
    GLIO_REQUIRE(xyz != nullptr && Q > 0, GLIO_ERR_ARG, "null or empty point array");
    GLIO_REQUIRE(stride >= 3 && stride <= 64, GLIO_ERR_ARG, "stride_floats must be in [3,64]");
    upload_points_async(c, {&c->slot(slot).corners}, &xyz, &Q, stride, mem);
  });
}

void glio_edge_default_options(glio_edge_options* o) {
  if (!o) return;
  o->max_sqdist = 1.0; o->min_ratio = 3.0; o->half_length = 0.1; o->score = 1.0;
}

}  // extern "C"

namespace {

// the options of an edge association call (NULL: the defaults), validated
glio_edge_options edge_options_or_default(const glio_edge_options* options) {
  glio_edge_options o; if (options) o = *options; else glio_edge_default_options(&o);
  GLIO_REQUIRE(std::isfinite(o.max_sqdist) && o.max_sqdist > 0.0 && std::isfinite(o.min_ratio) && o.min_ratio >= 0.0 &&
               std::isfinite(o.half_length) && o.half_length > 0.0 && std::isfinite(o.score), GLIO_ERR_ARG,
               "glio_edge_options: need max_sqdist > 0, min_ratio >= 0, half_length > 0 and a finite score");
  return o;
}

// K1e / K1be over planned segments: ensure_work, one search + line-fit launch against `grid` (pair mode when oth_local is set),
// compaction of every segment's valid records into dst[segment] and one host synchronisation; c->h_counts then holds the
// per-segment edge counts.  dbg (window mode, keep_debug): each segment's debug views, captured from the work space.
void edge_assoc_launch(glio_ctx* c, const GridBuild& grid, const std::vector<SegDesc>& segs, const std::vector<EdgeDst>& dst, int64_t Qt,
                       const glio_edge_options& o, const float* oth_local, int oth_stride, const std::vector<AssocDebug*>* dbg) {
  const int nseg = (int)segs.size();
  const bool keep_debug = dbg != nullptr;
  ensure_work(c, Qt, false, keep_debug);
  c->w_pa.reserve((size_t)Qt); c->w_pb.reserve((size_t)Qt);
  if (keep_debug) c->w_eig.reserve((size_t)Qt * 3);
  c->d_segs.reserve(nseg); c->d_edst.reserve(nseg); c->d_counts.reserve(nseg); c->h_counts.reserve(nseg);
  GLIO_CUDA_TRY(cudaMemcpyAsync(c->d_segs.p, segs.data(), nseg * sizeof(SegDesc), cudaMemcpyHostToDevice, c->st));
  GLIO_CUDA_TRY(cudaMemcpyAsync(c->d_edst.p, dst.data(), nseg * sizeof(EdgeDst), cudaMemcpyHostToDevice, c->st));
  AssocWork w = make_work(c, Qt, false, keep_debug);
  const EdgeFitParams ep{o.max_sqdist, o.min_ratio, o.half_length};
  edge_assoc_run(grid, c->d_segs.p, nseg, w, ep, c->w_pa.p, c->w_pb.p, keep_debug ? c->w_eig.p : nullptr, oth_local, oth_stride, c->cell_count,
                 c->cell_pos, c->scan_tmp, c->st, c->lc);
  compact_count(w, c->d_segs.p, nseg, c->w_flags.p, c->w_pos.p, c->scan_tmp, c->d_counts.p, c->st, c->lc);
  compact_edge_scatter(w, c->d_segs.p, c->w_pos.p, c->w_pa.p, c->w_pb.p, (float)o.score, c->d_edst.p, c->st, c->lc);
  GLIO_CUDA_TRY(cudaMemcpyAsync(c->h_counts.p, c->d_counts.p, nseg * sizeof(int), cudaMemcpyDeviceToHost, c->st));
  if (keep_debug)
    for (int s = 0; s < nseg; ++s) capture_debug(c, *(*dbg)[s], w, c->w_eig.p, 3, segs[s].offset, segs[s].count);
  GLIO_CUDA_TRY(cudaStreamSynchronize(c->st));
}

}  // namespace

extern "C" {

int glio_set_edge_map(glio_ctx* c, const float* xyz, int64_t M, int stride, int mem) {
  if (!c) return GLIO_ERR_ARG;
  return guarded(c, [&] {
    GLIO_REQUIRE(M >= 5, GLIO_ERR_ARG, "corner map needs at least 5 points");
    map_build(c, c->edge_map, stage_points(c, c->edge_map.stage, xyz, M, stride, mem), stride, M);
  });
}

int glio_edge_localmap_clear(glio_ctx* c) {
  if (!c) return GLIO_ERR_ARG;
  return localmap_clear(c, c->edge_map);
}

int glio_edge_localmap_push(glio_ctx* c, int at_front, const float* cloud_xyz, int64_t n, int stride, int mem, const double t[3], const double q[4]) {
  if (!c) return GLIO_ERR_ARG;
  return localmap_push(c, c->edge_map, at_front, cloud_xyz, n, stride, mem, t, q);
}

int glio_edge_localmap_pop_front(glio_ctx* c) {
  if (!c) return GLIO_ERR_ARG;
  return localmap_pop_front(c, c->edge_map);
}

int glio_edge_localmap_build(glio_ctx* c, float leaf, int64_t* n_map) {
  if (!c) return GLIO_ERR_ARG;
  return localmap_build(c, c->edge_map, "corner local map", leaf, n_map);
}

int glio_window_associate_edges(glio_ctx* c, int W, const double* poses_body, const glio_edge_options* options, int64_t* n_edge) {
  if (!c) return GLIO_ERR_ARG;
  return guarded(c, [&] {
    GLIO_REQUIRE(W > 0 && W <= 4096 && poses_body, GLIO_ERR_ARG, "bad window arguments");
    const glio_edge_options o = edge_options_or_default(options);
    GLIO_REQUIRE(c->edge_map.valid, GLIO_ERR_STATE, "glio_set_edge_map must be called before edge association");
    for (int k = 0; k < W; ++k)
      GLIO_REQUIRE((size_t)k < c->slots.size() && c->slots[k] && c->slots[k]->corners.n > 0 && c->slots[k]->corners.ptr, GLIO_ERR_STATE,
                   "slot has no corner scan");
    if (c->scans_pending) { GLIO_CUDA_TRY(cudaStreamWaitEvent(c->st, c->ev_scans, 0)); c->scans_pending = false; }
    std::vector<SegDesc> segs(W);
    int64_t Qt = 0;
    for (int k = 0; k < W; ++k) {
      double lp[7];
      lidar_pose_in_map(c->prm.q_lb, c->prm.t_lb, poses_body + 7 * k, lp, lp + 3);   // Estimator.cpp:2216-2217
      segs[k] = make_seg(c->slots[k]->corners, Qt, lp);
      Qt += c->slots[k]->corners.n;
    }
    GLIO_REQUIRE(Qt < ((int64_t)1 << 31), GLIO_ERR_ARG, "glio_window_associate_edges: too many corner points in one window");
    // the slots' edge lists are replaced from here on: they count as empty until the counts arrive (an error below leaves them
    // empty, never pointing at memory that does not hold them)
    std::vector<EdgeDst> dst(W);
    std::vector<AssocDebug*> dbg(W);
    for (int k = 0; k < W; ++k) {
      Slot& sl = *c->slots[k];
      sl.edges.clear();
      dst[k] = sl.edges.edge_dst(sl.corners.n);
      dbg[k] = &sl.edge_dbg;
    }
    edge_assoc_launch(c, c->edge_map.grid, segs, dst, Qt, o, nullptr, 0, c->prm.keep_debug ? &dbg : nullptr);
    for (int k = 0; k < W; ++k) {
      CorrList& e = c->slots[k]->edges;
      e.n = c->h_counts.p[k]; e.has_src = true;
      if (n_edge) n_edge[k] = e.n;
    }
  });
}

}  // extern "C"

namespace {

// copy-out of an edge list (glio_get_edges / glio_batch_get_edges): all arrays NULL only counts
void copy_edges_out(glio_ctx* c, const CorrList& e, int64_t capacity, float* cp, float* pa, float* pb, double* s, int32_t* src, int64_t* n_out) {
  const int64_t n = e.n;
  if (n_out) *n_out = n;
  if (!cp && !pa && !pb && !s && !src) return;             // a count query
  GLIO_REQUIRE(capacity >= n, GLIO_ERR_ARG, "capacity smaller than the edge count");
  if (n == 0) return;
  std::vector<float4> h0(n), h1(n), h2(n);
  GLIO_CUDA_TRY(cudaMemcpyAsync(h0.data(), e.rec.cpw.p, n * sizeof(float4), cudaMemcpyDeviceToHost, c->st));
  GLIO_CUDA_TRY(cudaMemcpyAsync(h1.data(), e.rec.pa.p, n * sizeof(float4), cudaMemcpyDeviceToHost, c->st));
  GLIO_CUDA_TRY(cudaMemcpyAsync(h2.data(), e.rec.pb.p, n * sizeof(float4), cudaMemcpyDeviceToHost, c->st));
  if (src && e.has_src) GLIO_CUDA_TRY(cudaMemcpyAsync(src, e.src.p, n * sizeof(int32_t), cudaMemcpyDeviceToHost, c->st));
  GLIO_CUDA_TRY(cudaStreamSynchronize(c->st));
  unpack_float4(h0.data(), n, cp);
  unpack_float4(h1.data(), n, pa);
  unpack_float4(h2.data(), n, pb);
  for (int64_t i = 0; i < n; ++i) {
    if (s) s[i] = (double)h0[i].w;
    if (src && !e.has_src) src[i] = -1;
  }
}

// upload of an edge list (glio_set_edges / glio_batch_set_pair_edges): (cp, s) / pa / pb as float4, n > 0
void upload_edges(glio_ctx* c, CorrList& e, int64_t n, const float* cp, const float* pa, const float* pb, const double* s) {
  GLIO_REQUIRE(cp && pa && pb && s, GLIO_ERR_ARG, "null edge arrays");
  std::vector<float4> h0(n), h1(n), h2(n);
  for (int64_t i = 0; i < n; ++i) {
    h0[i] = make_float4(cp[3 * i], cp[3 * i + 1], cp[3 * i + 2], (float)s[i]);
    h1[i] = make_float4(pa[3 * i], pa[3 * i + 1], pa[3 * i + 2], 0.f);
    h2[i] = make_float4(pb[3 * i], pb[3 * i + 1], pb[3 * i + 2], 0.f);
  }
  e.rec.reserve(e.kind, n);
  GLIO_CUDA_TRY(cudaMemcpyAsync(e.rec.cpw.p, h0.data(), n * sizeof(float4), cudaMemcpyHostToDevice, c->st));
  GLIO_CUDA_TRY(cudaMemcpyAsync(e.rec.pa.p, h1.data(), n * sizeof(float4), cudaMemcpyHostToDevice, c->st));
  GLIO_CUDA_TRY(cudaMemcpyAsync(e.rec.pb.p, h2.data(), n * sizeof(float4), cudaMemcpyHostToDevice, c->st));
  GLIO_CUDA_TRY(cudaStreamSynchronize(c->st));
  e.n = n;
}

// glio_get_assoc_debug / glio_get_edge_debug: a slot's views of its last plane (nfit = 4) or edge (nfit = 3) association
int read_assoc_debug(glio_ctx* c, int slot, AssocDebug Slot::*view, int nfit, const char* q_mismatch, int64_t Q, uint8_t* status, int32_t* idx5,
                     float* sqd5, float* pm, double* fit) {
  if (!c) return GLIO_ERR_ARG;
  return guarded(c, [&] {
    GLIO_REQUIRE(c->prm.keep_debug, GLIO_ERR_STATE, "context was created without keep_debug");
    const AssocDebug& d = c->slot(slot).*view;
    GLIO_REQUIRE(d.Q == Q && Q > 0, GLIO_ERR_ARG, q_mismatch);
    if (status) GLIO_CUDA_TRY(cudaMemcpyAsync(status, d.status.p, Q, cudaMemcpyDeviceToHost, c->st));
    if (idx5) GLIO_CUDA_TRY(cudaMemcpyAsync(idx5, d.idx5.p, 5 * Q * sizeof(int32_t), cudaMemcpyDeviceToHost, c->st));
    if (sqd5) GLIO_CUDA_TRY(cudaMemcpyAsync(sqd5, d.sqd5.p, 5 * Q * sizeof(float), cudaMemcpyDeviceToHost, c->st));
    if (fit) GLIO_CUDA_TRY(cudaMemcpyAsync(fit, d.fit.p, nfit * Q * sizeof(double), cudaMemcpyDeviceToHost, c->st));
    std::vector<float4> h;
    if (pm) { h.resize(Q); GLIO_CUDA_TRY(cudaMemcpyAsync(h.data(), d.pm.p, Q * sizeof(float4), cudaMemcpyDeviceToHost, c->st)); }
    GLIO_CUDA_TRY(cudaStreamSynchronize(c->st));
    if (pm) unpack_float4(h.data(), Q, pm);
  });
}

}  // namespace

extern "C" {

int glio_get_edges(glio_ctx* c, int slot, int64_t capacity, float* cp, float* pa, float* pb, double* s, int32_t* src, int64_t* n_out) {
  if (!c) return GLIO_ERR_ARG;
  return guarded(c, [&] {
    copy_edges_out(c, c->slot(slot).edges, capacity, cp, pa, pb, s, src, n_out);
  });
}

int glio_get_edge_debug(glio_ctx* c, int slot, int64_t Q, uint8_t* status, int32_t* idx5, float* sqd5, float* pm, double* eig) {
  return read_assoc_debug(c, slot, &Slot::edge_dbg, 3, "Q does not match the slot's last edge association", Q, status, idx5, sqd5, pm, eig);
}

int glio_window_associate(glio_ctx* c, int W, const double* poses_body, int64_t* n_match) {
  if (!c) return GLIO_ERR_ARG;
  return guarded(c, [&] {
    GLIO_REQUIRE(W > 0 && poses_body, GLIO_ERR_ARG, "bad window arguments");
    std::vector<int> ids(W);
    std::vector<std::array<double, 7>> lp(W);
    for (int k = 0; k < W; ++k) {
      ids[k] = k;
      lidar_pose_in_map(c->prm.q_lb, c->prm.t_lb, poses_body + 7 * k, &lp[k][0], &lp[k][3]);   // Estimator.cpp:2216-2217
    }
    associate_ctx_slots(c, ids, lp, n_match);
  });
}

int glio_get_matches(glio_ctx* c, int slot, int64_t capacity, float* cp, float* nsd, float* weight, int32_t* src, int64_t* n_out) {
  if (!c) return GLIO_ERR_ARG;
  return guarded(c, [&] { copy_matches_out(c, c->slot(slot).planes, capacity, cp, weight, nsd, nullptr, src, n_out); });
}

int glio_get_assoc_debug(glio_ctx* c, int slot, int64_t Q, uint8_t* status, int32_t* idx5, float* sqd5, float* pm, double* plane) {
  return read_assoc_debug(c, slot, &Slot::dbg, 4, "Q does not match the slot's last association", Q, status, idx5, sqd5, pm, plane);
}

int glio_select(glio_ctx* c, int slot, const int32_t* keep, int64_t n) {
  if (!c) return GLIO_ERR_ARG;
  return guarded(c, [&] { select_keep(c, c->slot(slot).planes, keep, n); });
}

int glio_eval_unary(glio_ctx* c, int W, const double* poses_body, int jac_kind, double* H, double* g, double* cost) {
  if (!c) return GLIO_ERR_ARG;
  return guarded(c, [&] {
    GLIO_REQUIRE(W > 0 && W <= 4096 && poses_body, GLIO_ERR_ARG, "bad arguments");
    GLIO_REQUIRE(jac_kind == 0 || jac_kind == 1, GLIO_ERR_ARG, "jac_kind must be 0 or 1");
    const bool want_jac = (H != nullptr) || (g != nullptr);
    eval_unary_blocks(c, W, poses_body, jac_kind, want_jac);
    unpack_blocks(c->h_out.p, W, H, g, cost);
  });
}

// ---- K3: marginalisation of KF0 (MarginalizationInfo::PreMarginalize + Marginalize, MarginalizationFactor.cpp:107-202)
}  // extern "C"

namespace {

// host half: the device blocks (W x 28 doubles: 21 upper-triangular H, 6 g, cost) join A/b, then Schur + decomposition + prior
glio_marg_prior* marg_finish_host(int W, double eps, std::vector<double>& A, std::vector<double>& b, const double* hout,
                                  const double* x0_pose, const double* x0_sb) {
  const int N = 6 * W + 18, m = 15, n = N - m;
  static const int ut[6][6] = {{0, 1, 2, 3, 4, 5}, {1, 6, 7, 8, 9, 10}, {2, 7, 11, 12, 13, 14}, {3, 8, 12, 15, 16, 17}, {4, 9, 13, 16, 18, 19}, {5, 10, 14, 17, 19, 20}};
  for (int k = 0; k < W; ++k) {
    const double* o = hout + (size_t)k * GLIO_NACC;
    const int base = marg_index_t(k);                       // t at base, q at base + 3 in every keyframe of this ordering
    for (int p = 0; p < 6; ++p) { b[base + p] += o[21 + p]; for (int q = 0; q < 6; ++q) A[(size_t)(base + p) * N + base + q] += o[ut[p][q]]; }
  }
  std::vector<double> LJ((size_t)n * n), lr(n);
  if (marginalize_dense(A.data(), b.data(), N, m, eps, LJ.data(), lr.data()) != GLIO_OK) return nullptr;
  return glio_marg_prior_create(W, LJ.data(), lr.data(), x0_pose, x0_sb);
}

// device half + the caller's host factors: queues the LiDAR re-evaluation of every keyframe with the ambient x,y,z quaternion
// columns (Estimator.cpp:2538-2576), after the window's IMU factor KF0 -> KF1 when glio_window_use_imu_factors is on (*with_imu
// tells whether it was queued), and evaluates the host callback while the kernels run
unsigned int marg_begin(glio_ctx* c, int W, const double* poses, const double* speed_bias, glio_host_marg_fn host_marg, void* user,
                        std::vector<double>& A, std::vector<double>& b, bool* with_imu) {
  const int N = 6 * W + 18;
  *with_imu = c->window_imu.use && !c->window_imu.pairs.empty() && window_imu_marg_launch(c, poses, speed_bias);
  const unsigned int epoch = eval_unary_launch(c, W, poses, 1, true, nullptr, true);
  A.assign((size_t)N * N, 0.0); b.assign(N, 0.0);
  if (host_marg) GLIO_REQUIRE(host_marg(user, W, poses, speed_bias, A.data(), b.data()) == 0, GLIO_ERR_STATE, "host_marg callback failed");
  return epoch;
}

void marg_worker(glio_ctx* c) {
  cudaSetDevice(c->device);
#if defined(__linux__)
  cpu_set_t base; CPU_ZERO(&base);
  const bool have_base = pthread_getaffinity_np(pthread_self(), sizeof(base), &base) == 0;
  int excluded = -1;
#endif
  for (;;) {
    glio_marg_job* j = nullptr;
    {
      std::unique_lock<std::mutex> lk(c->marg_mu);
      c->marg_cv.wait(lk, [&] { return c->marg_queued != nullptr || c->marg_quit; });
      if (c->marg_quit && !c->marg_queued) return;
      j = c->marg_queued; c->marg_queued = nullptr;
    }
#if defined(__linux__)
    // The submitting thread is about to queue the next window's kernels: a worker woken onto ITS core would preempt it for the
    // whole host half and the GPU would idle meanwhile.  Keep off that core (the rest of the process mask stays allowed).
    if (have_base && j->submit_cpu >= 0 && j->submit_cpu != excluded && CPU_COUNT(&base) > 1) {
      cpu_set_t m = base; CPU_CLR(j->submit_cpu, &m);
      if (CPU_COUNT(&m) > 0 && pthread_setaffinity_np(pthread_self(), sizeof(m), &m) == 0) excluded = j->submit_cpu;
    }
#endif
    try {
      eval_unary_wait(c, j->epoch);
      j->out.assign(c->h_out.p, c->h_out.p + (size_t)j->W * GLIO_NACC);
      if (j->with_imu) j->imu.assign(c->h_wimu_marg.p, c->h_wimu_marg.p + GLIO_NACC_IMU);
      j->copied.store(1, std::memory_order_release);
      if (j->with_imu) add_marg_imu(j->A, j->b, 6 * j->W + 18, j->imu.data());
      j->prior = marg_finish_host(j->W, j->eps, j->A, j->b, j->out.data(), j->x0_pose.data(), j->x0_sb.data());
      if (!j->prior) { j->rc = GLIO_ERR_STATE; j->err = "marginalisation failed (decomposition or prior)"; }
    } catch (const Error& e) { j->rc = e.code; j->err = e.msg; }
    catch (const std::exception& e) { j->rc = GLIO_ERR_STATE; j->err = e.what(); }
    j->copied.store(1, std::memory_order_release);
    j->done.store(1, std::memory_order_release);
  }
}

}  // namespace

extern "C" {

int glio_window_marginalize(glio_ctx* c, int W, const double* poses, const double* speed_bias, glio_host_marg_fn host_marg, void* user,
                            double eps, glio_marg_prior** prior_out) {
  if (!c || !prior_out) return GLIO_ERR_ARG;
  *prior_out = nullptr;
  return guarded(c, [&] {
    GLIO_REQUIRE(W >= 2 && W <= 4096 && poses && speed_bias, GLIO_ERR_ARG, "glio_window_marginalize: need W >= 2, poses and speed_bias");
    std::vector<double> A, b;
    bool with_imu = false;
    const unsigned int epoch = marg_begin(c, W, poses, speed_bias, host_marg, user, A, b, &with_imu);
    eval_unary_wait(c, epoch);
    if (with_imu) add_marg_imu(A, b, 6 * W + 18, c->h_wimu_marg.p);
    glio_marg_prior* made = marg_finish_host(W, eps, A, b, c->h_out.p, poses + 7, speed_bias + 9);
    GLIO_REQUIRE(made != nullptr, GLIO_ERR_STATE, "marginalisation failed (decomposition or prior)");
    *prior_out = made;
  });
}

// The same pass with its host half on the context's worker thread: returns as soon as the device half is queued and the host
// callback has run; the Schur complement, the decomposition and the prior are computed while the caller hands the next window's
// association to the GPU.  One job at a time per context; glio_marg_job_wait joins it (and must be called before the next solve
// needs the prior).  Results are identical to glio_window_marginalize.
int glio_window_marginalize_async(glio_ctx* c, int W, const double* poses, const double* speed_bias, glio_host_marg_fn host_marg, void* user,
                                  double eps, glio_marg_job** job_out) {
  if (!c || !job_out) return GLIO_ERR_ARG;
  *job_out = nullptr;
  return guarded(c, [&] {
    GLIO_REQUIRE(W >= 2 && W <= 4096 && poses && speed_bias, GLIO_ERR_ARG, "glio_window_marginalize_async: need W >= 2, poses and speed_bias");
    GLIO_REQUIRE(c->marg_pending == nullptr, GLIO_ERR_STATE, "glio_window_marginalize_async: the previous job has not been waited for");
    std::unique_ptr<glio_marg_job> j(new glio_marg_job());
    j->ctx = c; j->W = W; j->eps = eps;
    j->x0_pose.assign(poses + 7, poses + 7 * (size_t)W); j->x0_sb.assign(speed_bias + 9, speed_bias + 18);
    j->epoch = marg_begin(c, W, poses, speed_bias, host_marg, user, j->A, j->b, &j->with_imu);
#if defined(__linux__)
    j->submit_cpu = sched_getcpu();
#endif
    if (!c->marg_thread.joinable()) c->marg_thread = std::thread(marg_worker, c);
    { std::lock_guard<std::mutex> lk(c->marg_mu); c->marg_queued = j.get(); }
    c->marg_cv.notify_one();
    c->marg_pending = j.get();
    *job_out = j.release();
  });
}

int glio_marg_job_wait(glio_marg_job* j, glio_marg_prior** prior_out) {
  if (!j) return GLIO_ERR_ARG;
  if (prior_out) *prior_out = nullptr;
  for (unsigned long long spins = 0; !j->done.load(std::memory_order_acquire); ++spins) {
#if defined(__x86_64__)
    __builtin_ia32_pause();
#endif
    if ((spins & 0xfffull) == 0xfffull) std::this_thread::yield();
  }
  glio_ctx* c = j->ctx;
  if (c && c->marg_pending == j) c->marg_pending = nullptr;
  const int rc = j->rc;
  if (rc != GLIO_OK) { if (c) c->err = j->err; if (j->prior) glio_marg_prior_destroy(j->prior); }
  else if (prior_out) *prior_out = j->prior;
  else if (j->prior) glio_marg_prior_destroy(j->prior);
  delete j;
  return rc;
}

// ---- front-end feature extraction (SURVEY 8 f-4): Preprocessing::cloudHandler, GLIO/src/Preprocessing.cpp:529-655
int glio_extract_features(glio_ctx* c, const float* cloud_xyzi, int64_t n, int stride, int intensity_offset, int mem, int n_scans, const int32_t* scan_start,
                          const int32_t* scan_end, int ds_rate, double edge_thres, double surf_thres, float ds_v, float* curvature, int8_t* label,
                          int32_t* sharp, int64_t* n_sharp, int32_t* less_sharp, int64_t* n_less_sharp, int32_t* flat, int64_t* n_flat,
                          int32_t* less_flat, int64_t* n_less_flat, float* less_flat_ds, int64_t* n_less_flat_ds) {
  if (!c) return GLIO_ERR_ARG;
  return guarded(c, [&] {
    GLIO_REQUIRE(cloud_xyzi && n > 10 && n < ((int64_t)1 << 30), GLIO_ERR_ARG, "glio_extract_features: bad cloud");
    GLIO_REQUIRE(stride >= 4 && stride <= 64 && intensity_offset >= 3 && intensity_offset < stride, GLIO_ERR_ARG, "glio_extract_features: stride_floats must be >= 4 and 3 <= intensity_offset < stride");
    GLIO_REQUIRE(n_scans > 0 && n_scans <= 1024 && scan_start && scan_end && ds_rate >= 1 && ds_v > 0.f, GLIO_ERR_ARG, "glio_extract_features: bad ring table");
    for (int r = 0; r < n_scans; ++r) GLIO_REQUIRE(scan_start[r] >= 5 && scan_end[r] < n - 5 && scan_end[r] - scan_start[r] < n, GLIO_ERR_ARG, "glio_extract_features: ring range outside [5, n-6]");
    {
      // the processed rings run concurrently (one CTA each): a ring's neighbour suppression marks points up to 5 past its
      // range, so ordered by start the next processed ring must begin at least 5 points after the previous one ends
      std::vector<std::pair<int32_t, int>> used;
      for (int r = 0; r < n_scans; r += ds_rate)
        if (scan_end[r] - scan_start[r] >= 6) used.push_back({scan_start[r], r});
      std::sort(used.begin(), used.end());
      for (size_t k = 1; k < used.size(); ++k) {
        const int p = used[k - 1].second, q = used[k].second;
        if (scan_start[q] < scan_end[p] + 5) {
          char b[256];
          snprintf(b, sizeof(b), "glio_extract_features: rings %d [%d, %d] and %d [%d, %d] %s (processed rings need scan_start >= previous scan_end + 5)",
                   p, scan_start[p], scan_end[p], q, scan_start[q], scan_end[q], scan_start[q] < scan_end[p] ? "overlap" : "are closer than 5 points");
          throw Error{GLIO_ERR_ARG, b};
        }
      }
    }
    FeatArgs a{};
    const float* d_cloud = cloud_xyzi;
    if (mem != GLIO_DEVICE) { c->f_cloud.reserve((size_t)n * stride); GLIO_CUDA_TRY(cudaMemcpyAsync(c->f_cloud.p, cloud_xyzi, (size_t)n * stride * sizeof(float), cudaMemcpyHostToDevice, c->st)); d_cloud = c->f_cloud.p; }
    c->f_curv.reserve(n); c->f_label.reserve(n); c->f_picked.reserve(n); c->f_scan.reserve((size_t)2 * n_scans);
    c->f_ring.reserve((size_t)n_scans * (FEAT_MAX_SHARP + FEAT_MAX_LESS_SHARP + FEAT_MAX_FLAT)); c->f_lf.reserve(n); c->f_ds.reserve(n);
    c->f_counts.reserve((size_t)5 * n_scans + (size_t)5 * (n_scans + 1) + 4);
    c->f_out.reserve((size_t)n_scans * (FEAT_MAX_SHARP + FEAT_MAX_LESS_SHARP + FEAT_MAX_FLAT) + n); c->f_outds.reserve(n);
    GLIO_CUDA_TRY(cudaMemcpyAsync(c->f_scan.p, scan_start, n_scans * sizeof(int32_t), cudaMemcpyHostToDevice, c->st));
    GLIO_CUDA_TRY(cudaMemcpyAsync(c->f_scan.p + n_scans, scan_end, n_scans * sizeof(int32_t), cudaMemcpyHostToDevice, c->st));
    a.cloud = d_cloud; a.stride = stride; a.ioff = intensity_offset; a.n = n; a.n_scans = n_scans; a.scan_start = c->f_scan.p; a.scan_end = c->f_scan.p + n_scans; a.ds_rate = ds_rate;
    a.edge_thres = edge_thres; a.surf_thres = surf_thres; a.ds_v = ds_v;
    a.curv = c->f_curv.p; a.label = c->f_label.p; a.picked = c->f_picked.p;
    a.ring_sharp = c->f_ring.p; a.ring_less_sharp = a.ring_sharp + (size_t)n_scans * FEAT_MAX_SHARP; a.ring_flat = a.ring_less_sharp + (size_t)n_scans * FEAT_MAX_LESS_SHARP;
    a.ring_less_flat = c->f_lf.p; a.ring_ds = c->f_ds.p;
    a.counts = c->f_counts.p; a.offsets = c->f_counts.p + 5 * n_scans; a.err = c->f_counts.p + 5 * n_scans + 5 * (n_scans + 1);
    a.out_sharp = c->f_out.p; a.out_less_sharp = a.out_sharp + (size_t)n_scans * FEAT_MAX_SHARP; a.out_flat = a.out_less_sharp + (size_t)n_scans * FEAT_MAX_LESS_SHARP;
    a.out_less_flat = a.out_flat + (size_t)n_scans * FEAT_MAX_FLAT; a.out_ds = c->f_outds.p;
    features_run(a, c->st, c->lc);
    std::vector<int32_t> tot((size_t)5 * (n_scans + 1) + 1);
    GLIO_CUDA_TRY(cudaMemcpyAsync(tot.data(), a.offsets, tot.size() * sizeof(int32_t), cudaMemcpyDeviceToHost, c->st));
    GLIO_CUDA_TRY(cudaStreamSynchronize(c->st));
    const int32_t err = tot[(size_t)5 * (n_scans + 1)];
    GLIO_REQUIRE(err == 0, GLIO_ERR_ARG, err == 1 ? "glio_extract_features: a ring sector has more than 4096 points" : "glio_extract_features: a ring has more than 8192 less-flat points");
    const int64_t cnt[5] = {tot[0 * (n_scans + 1) + n_scans], tot[1 * (n_scans + 1) + n_scans], tot[2 * (n_scans + 1) + n_scans], tot[3 * (n_scans + 1) + n_scans], tot[4 * (n_scans + 1) + n_scans]};
    if (n_sharp) *n_sharp = cnt[0];
    if (n_less_sharp) *n_less_sharp = cnt[1];
    if (n_flat) *n_flat = cnt[2];
    if (n_less_flat) *n_less_flat = cnt[3];
    if (n_less_flat_ds) *n_less_flat_ds = cnt[4];
    if (curvature) GLIO_CUDA_TRY(cudaMemcpyAsync(curvature, a.curv, n * sizeof(float), cudaMemcpyDeviceToHost, c->st));
    if (label) GLIO_CUDA_TRY(cudaMemcpyAsync(label, a.label, n, cudaMemcpyDeviceToHost, c->st));
    if (sharp && cnt[0]) GLIO_CUDA_TRY(cudaMemcpyAsync(sharp, a.out_sharp, cnt[0] * sizeof(int32_t), cudaMemcpyDeviceToHost, c->st));
    if (less_sharp && cnt[1]) GLIO_CUDA_TRY(cudaMemcpyAsync(less_sharp, a.out_less_sharp, cnt[1] * sizeof(int32_t), cudaMemcpyDeviceToHost, c->st));
    if (flat && cnt[2]) GLIO_CUDA_TRY(cudaMemcpyAsync(flat, a.out_flat, cnt[2] * sizeof(int32_t), cudaMemcpyDeviceToHost, c->st));
    if (less_flat && cnt[3]) GLIO_CUDA_TRY(cudaMemcpyAsync(less_flat, a.out_less_flat, cnt[3] * sizeof(int32_t), cudaMemcpyDeviceToHost, c->st));
    if (less_flat_ds && cnt[4]) GLIO_CUDA_TRY(cudaMemcpyAsync(less_flat_ds, a.out_ds, cnt[4] * sizeof(float4), cudaMemcpyDeviceToHost, c->st));
    GLIO_CUDA_TRY(cudaStreamSynchronize(c->st));
  });
}

// ---- front-end sweep preparation (SURVEY 8 f-5): Preprocessing::cloudHandler, GLIO/src/Preprocessing.cpp:387-526
int glio_prepare_scan(glio_ctx* c, const float* raw, int64_t n, int stride, int mem, int n_scans, const double q_imu[4],
                      const double q_lb[4], float* out_xyzi, int out_mem, int64_t out_capacity, int64_t* n_out,
                      int32_t* scan_start, int32_t* scan_end) {
  if (!c) return GLIO_ERR_ARG;
  return guarded(c, [&] {
    GLIO_REQUIRE(raw && n > 0 && n < ((int64_t)1 << 30), GLIO_ERR_ARG, "glio_prepare_scan: bad sweep");
    GLIO_REQUIRE(stride >= 3 && stride <= 64, GLIO_ERR_ARG, "glio_prepare_scan: stride_floats must be in [3,64]");
    GLIO_REQUIRE(n_scans == 16 || n_scans == 32 || n_scans == 64, GLIO_ERR_ARG, "glio_prepare_scan: n_scans must be 16, 32 or 64 (wrong scan number)");
    GLIO_REQUIRE(n_out && out_capacity >= 0 && (out_xyzi || out_capacity == 0), GLIO_ERR_ARG, "glio_prepare_scan: bad output arguments");
    // a GLIO_DEVICE pointer must be memory of the context's GPU that the kernels can address: a host pointer, another GPU's
    // memory or a misaligned output is an argument error, never a fault
    auto on_device = [c](const void* p) { return on_ctx_device(c, p); };
    GLIO_REQUIRE(mem != GLIO_DEVICE || on_device(raw), GLIO_ERR_ARG, "glio_prepare_scan: mem = GLIO_DEVICE but raw is not device memory of the context's GPU");
    GLIO_REQUIRE(((uintptr_t)raw & 3) == 0, GLIO_ERR_ARG, "glio_prepare_scan: raw must be 4-byte aligned");
    GLIO_REQUIRE(out_mem != GLIO_DEVICE || !out_xyzi || on_device(out_xyzi), GLIO_ERR_ARG, "glio_prepare_scan: out_mem = GLIO_DEVICE but out_xyzi is not device memory of the context's GPU");
    GLIO_REQUIRE(out_mem != GLIO_DEVICE || ((uintptr_t)out_xyzi & 15) == 0, GLIO_ERR_ARG, "glio_prepare_scan: a device out_xyzi must be 16-byte aligned (float4 stores)");
    ScanPrepArgs a{};
    // per-sweep rotation constants (:186-191): qIMU (NaN -> identity, :415-417), q_lb, q_lb.inverse(), Identity.dot(qIMU)
    const double ident[4] = {1.0, 0.0, 0.0, 0.0};
    const double* qi = q_imu ? q_imu : ident;
    if (std::isnan(qi[0]) || std::isnan(qi[1]) || std::isnan(qi[2]) || std::isnan(qi[3])) qi = ident;
    const double* ql = q_lb ? q_lb : ident;
    for (int d = 0; d < 4; ++d) { a.q_imu[d] = qi[d]; a.q_lb[d] = ql[d]; }
    const double n2 = ((ql[1] * ql[1] + ql[2] * ql[2]) + ql[3] * ql[3]) + ql[0] * ql[0];       // coeffs() = x, y, z, w
    if (n2 > 0.0) { a.q_lb_inv[0] = ql[0] / n2; a.q_lb_inv[1] = -ql[1] / n2; a.q_lb_inv[2] = -ql[2] / n2; a.q_lb_inv[3] = -ql[3] / n2; }
    a.dot = ((0.0 * qi[1] + 0.0 * qi[2]) + 0.0 * qi[3]) + 1.0 * qi[0];
    const double absd = std::fabs(a.dot);
    a.slerp_linear = absd >= 1.0 - std::numeric_limits<double>::epsilon();
    a.theta = std::acos(absd); a.sin_theta = std::sin(a.theta);

    a.raw = raw;
    if (mem != GLIO_DEVICE) {
      c->sp_raw.reserve((size_t)n * stride);
      GLIO_CUDA_TRY(cudaMemcpyAsync(c->sp_raw.p, raw, (size_t)n * stride * sizeof(float), cudaMemcpyHostToDevice, c->st));
      a.raw = c->sp_raw.p;
    }
    a.stride = stride; a.n = n; a.n_scans = n_scans; a.nb = (int)((n + 255) / 256);
    c->sp_ring.reserve(n); c->sp_ori.reserve(n);
    c->sp_hist.reserve((size_t)n_scans * a.nb); c->sp_hscan.reserve((size_t)n_scans * a.nb);
    c->sp_small.reserve(5 + 2 * 64); c->sp_consts.reserve(1);
    if (!c->sp_hits.p) { c->sp_hits.reserve(1); GLIO_CUDA_TRY(cudaMemsetAsync(c->sp_hits.p, 0, sizeof(unsigned long long), c->st)); }
    a.consts = c->sp_consts.p; a.small = c->sp_small.p; a.ring = c->sp_ring.p; a.ori = c->sp_ori.p;
    a.hist = c->sp_hist.p; a.hscan = c->sp_hscan.p; a.scan_tmp = &c->sp_scan_tmp; a.guard_hits = c->sp_hits.p;
    if (out_mem == GLIO_DEVICE) { a.out = reinterpret_cast<float4*>(out_xyzi); a.out_capacity = out_capacity; }
    else { c->sp_out.reserve(n); a.out = c->sp_out.p; a.out_capacity = n; }
    scanprep_run(a, c->st, c->lc);
    std::vector<int32_t> small((size_t)5 + 2 * n_scans);
    GLIO_CUDA_TRY(cudaMemcpyAsync(small.data(), a.small, small.size() * sizeof(int32_t), cudaMemcpyDeviceToHost, c->st));
    GLIO_CUDA_TRY(cudaStreamSynchronize(c->st));
    GLIO_REQUIRE(small[3] != 0, GLIO_ERR_ARG, "glio_prepare_scan: no point of the sweep is finite and at least 3 m from the sensor");
    const int64_t m = small[4];
    *n_out = m;
    if (scan_start) std::memcpy(scan_start, small.data() + 5, n_scans * sizeof(int32_t));
    if (scan_end) std::memcpy(scan_end, small.data() + 5 + n_scans, n_scans * sizeof(int32_t));
    GLIO_REQUIRE(m <= out_capacity, GLIO_ERR_ARG, "glio_prepare_scan: out_capacity is smaller than the number of kept points");
    if (out_mem != GLIO_DEVICE && m > 0) {
      GLIO_CUDA_TRY(cudaMemcpyAsync(out_xyzi, a.out, (size_t)m * sizeof(float4), cudaMemcpyDeviceToHost, c->st));
      GLIO_CUDA_TRY(cudaStreamSynchronize(c->st));
    }
  });
}

int glio_scanprep_stats(glio_ctx* c, int64_t* guard_hits, int reset) {
  if (!c) return GLIO_ERR_ARG;
  return guarded(c, [&] {
    unsigned long long h = 0;
    if (c->sp_hits.p) {
      GLIO_CUDA_TRY(cudaMemcpyAsync(&h, c->sp_hits.p, sizeof(h), cudaMemcpyDeviceToHost, c->st));
      GLIO_CUDA_TRY(cudaStreamSynchronize(c->st));
      if (reset) GLIO_CUDA_TRY(cudaMemsetAsync(c->sp_hits.p, 0, sizeof(h), c->st));
    }
    if (guard_hits) *guard_hits = (int64_t)h;
  });
}

int glio_imu_sweep_rotation(glio_imu_state* st, const double* stamps, const double* gyro_xyz, int64_t n_buf, double t_scan_next,
                            double q_wxyz[4]) {
  return guarded(nullptr, [&] {
    GLIO_REQUIRE(st && q_wxyz && n_buf >= 0 && (n_buf == 0 || (stamps && gyro_xyz)), GLIO_ERR_ARG, "glio_imu_sweep_rotation: bad arguments");
    GLIO_REQUIRE(st->idx_imu >= 0 && st->idx_imu <= n_buf, GLIO_ERR_ARG, "glio_imu_sweep_rotation: idx_imu is past the end of the buffer");
    GLIO_REQUIRE(n_buf > 0 || !st->first_imu, GLIO_ERR_ARG, "glio_imu_sweep_rotation: empty IMU buffer after the first sample");
    imu_sweep_rotation(st, stamps, gyro_xyz, n_buf, t_scan_next, q_wxyz);
  });
}

void glio_default_solver_options(glio_solver_options* o) {
  if (!o) return;
  memset(o, 0, sizeof(*o));
  o->max_num_iterations = 15; o->dogleg_type = 0; o->use_nonmonotonic_steps = 0; o->max_consecutive_nonmonotonic_steps = 5;
  o->initial_trust_region_radius = 1e4; o->max_trust_region_radius = 1e16; o->min_trust_region_radius = 1e-32;
  o->min_relative_decrease = 1e-3; o->min_lm_diagonal = 1e-6; o->max_lm_diagonal = 1e32; o->max_num_consecutive_invalid_steps = 5;
  o->jacobi_scaling = 1; o->function_tolerance = 1e-6; o->gradient_tolerance = 1e-10; o->parameter_tolerance = 1e-8;
  o->fuse_candidate_jacobian = 1;
}

static SolverOptions solver_options_from(const glio_solver_options& o) {
  SolverOptions so;
  so.max_num_iterations = o.max_num_iterations; so.dogleg_type = o.dogleg_type; so.use_nonmonotonic_steps = o.use_nonmonotonic_steps != 0;
  so.max_consecutive_nonmonotonic_steps = o.max_consecutive_nonmonotonic_steps;
  so.initial_trust_region_radius = o.initial_trust_region_radius; so.max_trust_region_radius = o.max_trust_region_radius;
  so.min_trust_region_radius = o.min_trust_region_radius; so.min_relative_decrease = o.min_relative_decrease;
  so.min_lm_diagonal = o.min_lm_diagonal; so.max_lm_diagonal = o.max_lm_diagonal;
  so.max_num_consecutive_invalid_steps = o.max_num_consecutive_invalid_steps; so.jacobi_scaling = o.jacobi_scaling != 0;
  so.function_tolerance = o.function_tolerance; so.gradient_tolerance = o.gradient_tolerance; so.parameter_tolerance = o.parameter_tolerance;
  so.fuse_candidate_jacobian = o.fuse_candidate_jacobian != 0;
  GLIO_REQUIRE(o.trust_region_strategy == 0 || o.trust_region_strategy == 1, GLIO_ERR_ARG, "trust_region_strategy must be 0 (DOGLEG) or 1 (LEVENBERG_MARQUARDT)");
  so.trust_region_strategy = o.trust_region_strategy;
  return so;
}

// W keyframes as the minimizer sees them: t (3), q (4, tangent 3) and, with speed-bias, 9 more per keyframe.  The ambient
// state holds them in that order, na doubles per keyframe; the tangent has nt per keyframe.
struct StateLayout {
  int W; bool sb; int nt, na;
  StateLayout(int W_, bool sb_) : W(W_), sb(sb_), nt(sb_ ? 15 : 6), na(sb_ ? 16 : 7) {}
  std::vector<ParamBlock> blocks() const {
    std::vector<ParamBlock> b;
    for (int k = 0; k < W; ++k) {
      b.push_back(ParamBlock{na * k, 3, nt * k, 3, false, nullptr});
      b.push_back(ParamBlock{na * k + 3, 4, nt * k + 3, 3, true, nullptr});
      if (sb) b.push_back(ParamBlock{na * k + 7, 9, nt * k + 6, 9, false, nullptr});
    }
    return b;
  }
  // poses (W x 7) and, with speed-bias, speed_bias (W x 9) into the ambient state x
  void pack(const double* poses, const double* speed_bias, double* x) const {
    for (int k = 0; k < W; ++k) {
      for (int i = 0; i < 7; ++i) x[(size_t)na * k + i] = poses[7 * k + i];
      if (sb) for (int i = 0; i < 9; ++i) x[(size_t)na * k + 7 + i] = speed_bias[9 * k + i];
    }
  }
  void unpack(const double* x, double* poses, double* speed_bias) const {
    for (int k = 0; k < W; ++k) {
      for (int i = 0; i < 7; ++i) poses[7 * k + i] = x[(size_t)na * k + i];
      if (sb) for (int i = 0; i < 9; ++i) speed_bias[9 * k + i] = x[(size_t)na * k + 7 + i];
    }
  }
};

// each keyframe's 21 upper-triangular H entries of the W x 28 layout onto the band's diagonal blocks, nt columns per keyframe
static void add_diag_blocks(BandMat* H, const double* o28, int W, int nt) {
  for (int k = 0; k < W; ++k) {
    const double* ob = o28 + (size_t)k * GLIO_NACC;
    int idx = 0;
    for (int p = 0; p < 6; ++p) for (int q = p; q < 6; ++q) { H->at(nt * k + q, nt * k + p) += ob[idx]; ++idx; }
  }
}

// The minimizer over W poses (and speed-bias states) with the LiDAR blocks of `tgt` (nullptr: the context's slots and glio_params,
// plus the window's IMU chain when glio_window_use_imu_factors is on) plus the host factors.  Throws on error; poses / speed_bias
// are in/out.
static void solve_core(glio_ctx* c, int W, double* poses, double* speed_bias, glio_host_factors_fn host_factors, glio_host_factors_band_fn host_band,
                       int hb_hint, void* user, const SolverOptions& so, const EvalTarget* tgt, SolverSummary& S) {
    const bool sb = speed_bias != nullptr;
    const StateLayout L(W, sb);
    const int nt = L.nt, n = W * nt;
    const bool add_imu = tgt == nullptr && c->window_imu.use && !c->window_imu.pairs.empty();
    GLIO_REQUIRE(!add_imu || sb, GLIO_ERR_ARG, "window solve: the IMU factors need speed_bias");
    GLIO_REQUIRE(!add_imu || c->window_imu.max_kf < W, GLIO_ERR_ARG, "window solve: an IMU factor references a slot outside [0, W)");
    const int imu_hb = add_imu ? imu_half_bandwidth(c->window_imu) : 0;   // the band must cover the IMU pairs whatever the callback writes
    TrustRegionDogleg solver(L.blocks(), so);
    std::vector<double> x((size_t)W * L.na), pz((size_t)W * 7), sz((size_t)W * 9);
    L.pack(poses, speed_bias, x.data());
    std::vector<double> Hd;       // dense scratch for the host callback's n x n interface
    int hb_fixed = -1;
    EvalFn eval = [&](const double* xa, bool want_jac, double* cost, BandMat* H, double* g) -> bool {
      L.unpack(xa, pz.data(), sz.data());
      // the device evaluates the IMU chain and the LiDAR residuals while the host evaluates its own factors
      if (add_imu) window_imu_launch(c, W, pz.data(), sz.data(), want_jac);
      const unsigned int epoch = eval_unary_launch(c, W, pz.data(), 0, want_jac, tgt, true);
      double ct = 0;
      if (want_jac) std::fill(g, g + n, 0.0);
      auto add_device = [&]() {
        eval_unary_wait(c, epoch);
        for (int k = 0; k < W; ++k) ct += c->h_out.p[(size_t)k * GLIO_NACC + 27];
        if (want_jac) for (int k = 0; k < W; ++k) for (int p = 0; p < 6; ++p) g[nt * k + p] += c->h_out.p[(size_t)k * GLIO_NACC + 21 + p];
      };
      if (host_band) {
        // host factors accumulate straight into the band matrix (no dense n x n scratch)
        if (want_jac) H->reset(n, hb_hint >= 5 ? std::max(hb_hint, imu_hb) : n - 1);
        const int hrc = host_band(user, W, pz.data(), sb ? sz.data() : nullptr, want_jac ? 1 : 0, want_jac ? H->a.data() : nullptr, want_jac ? H->hb : 0, g, &ct);
        add_device();
        if (hrc != 0) return false;
        if (want_jac) add_diag_blocks(H, c->h_out.p, W, nt);
        if (add_imu) add_imu_blocks(c->window_imu, W, want_jac, H, g, ct);
        *cost = ct;
        return std::isfinite(ct);
      }
      int hrc = 0;
      if (host_factors) {
        if (want_jac) Hd.assign((size_t)n * n, 0.0);
        hrc = host_factors(user, W, pz.data(), sb ? sz.data() : nullptr, want_jac ? 1 : 0, want_jac ? Hd.data() : nullptr, g, &ct);
      }
      add_device();
      if (hrc != 0) return false;
      if (want_jac) {
        // band of J^T J from what the callback actually wrote, re-derived at EVERY Jacobian evaluation (an entry that turns
        // non-zero later must not be dropped); the LiDAR blocks need 5
        {
          int w = 5;
          if (host_factors) for (int i = 0; i < n; ++i) for (int j = 0; j < i - w; ++j) if (Hd[(size_t)i * n + j] != 0.0 || Hd[(size_t)j * n + i] != 0.0) { w = i - j; break; }
          hb_fixed = std::max(hb_fixed, std::max(w, imu_hb));
        }
        H->reset(n, hb_fixed);
        const int hb = H->hb;
        if (host_factors) for (int i = 0; i < n; ++i) for (int j = std::max(0, i - hb); j <= i; ++j) H->at(i, j) = Hd[(size_t)i * n + j];
        add_diag_blocks(H, c->h_out.p, W, nt);
      }
      if (add_imu) add_imu_blocks(c->window_imu, W, want_jac, H, g, ct);
      *cost = ct;
      return std::isfinite(ct);
    };
    solver.solve(x.data(), eval, &S);
    L.unpack(x.data(), poses, speed_bias);
}

static int window_solve_impl(glio_ctx* c, int W, double* poses, double* speed_bias, glio_host_factors_fn host_factors,
                             glio_host_factors_band_fn host_band, int hb_hint, void* user,
                             const glio_solver_options* options, glio_solver_summary* summary, glio_iteration* iter_log, int iter_cap,
                             double* step_log, int64_t step_cap) {
  if (!c) return GLIO_ERR_ARG;
  return guarded(c, [&] {
    GLIO_REQUIRE(W > 0 && W <= 4096 && poses, GLIO_ERR_ARG, "bad arguments");
    glio_solver_options o; if (options) o = *options; else glio_default_solver_options(&o);
    const SolverOptions so = solver_options_from(o);
    SolverSummary S;
    solve_core(c, W, poses, speed_bias, host_factors, host_band, hb_hint, user, so, nullptr, S);
    fill_summary(S, W * (speed_bias ? 15 : 6), summary, iter_log, iter_cap, step_log, step_cap);
  });
}

int glio_window_solve(glio_ctx* c, int W, double* poses, double* speed_bias, glio_host_factors_fn host_factors, void* user,
                      const glio_solver_options* options, glio_solver_summary* summary, glio_iteration* iter_log, int iter_cap,
                      double* step_log, int64_t step_cap) {
  return window_solve_impl(c, W, poses, speed_bias, host_factors, nullptr, -1, user, options, summary, iter_log, iter_cap, step_log, step_cap);
}

int glio_window_solve_band(glio_ctx* c, int W, double* poses, double* speed_bias, glio_host_factors_band_fn host_factors, int half_bandwidth,
                           void* user, const glio_solver_options* options, glio_solver_summary* summary, glio_iteration* iter_log,
                           int iter_cap, double* step_log, int64_t step_cap) {
  return window_solve_impl(c, W, poses, speed_bias, nullptr, host_factors, half_bandwidth, user, options, summary, iter_log, iter_cap, step_log, step_cap);
}

int glio_eval_unary_residuals(glio_ctx* c, int slot, const double pose_body[7], int jac_kind, int64_t capacity, double* r, double* J, int64_t* n_out) {
  if (!c) return GLIO_ERR_ARG;
  return guarded(c, [&] {
    const CorrView v = c->slot(slot).planes.active();
    const int64_t n = v.n;
    if (n_out) *n_out = n;
    GLIO_REQUIRE(capacity >= n, GLIO_ERR_ARG, "capacity smaller than the residual count");
    if (n == 0) return;
    wait_marg_copied(c);               // h_poses may still feed a pending marginalisation's upload
    c->d_r.reserve(n); c->d_J.reserve(6 * n); c->d_poses.reserve(7); c->h_poses.reserve(7);
    memcpy(c->h_poses.p, pose_body, 7 * sizeof(double));
    GLIO_CUDA_TRY(cudaMemcpyAsync(c->d_poses.p, c->h_poses.p, 7 * sizeof(double), cudaMemcpyHostToDevice, c->st));
    eval_unary_residuals_run(v.cpw, v.nsd, n, c->d_poses.p, eval_params(c), jac_kind, c->d_r.p, c->d_J.p, c->st, c->lc);
    if (r) GLIO_CUDA_TRY(cudaMemcpyAsync(r, c->d_r.p, n * sizeof(double), cudaMemcpyDeviceToHost, c->st));
    if (J) GLIO_CUDA_TRY(cudaMemcpyAsync(J, c->d_J.p, 6 * n * sizeof(double), cudaMemcpyDeviceToHost, c->st));
    GLIO_CUDA_TRY(cudaStreamSynchronize(c->st));
  });
}


// ------------------------------------------------------------------------------------------------------------
// batch path: frames, pair association (K1b), binary evaluation (K2b)
// ------------------------------------------------------------------------------------------------------------
int glio_batch_clear(glio_ctx* c) {
  if (!c) return GLIO_ERR_ARG;
  return guarded(c, [&] {
    GLIO_CUDA_TRY(cudaStreamSynchronize(c->st));
    c->frames.clear(); c->pairs.clear(); c->pair_index.clear(); c->bin_dirty = true; c->bedge_dirty = true;
    c->pose.clear(); c->dd.clear(); c->imu.clear();
  });
}

int glio_batch_set_frame(glio_ctx* c, int frame, const float* scan_xyz, int64_t Q, int stride, int mem, const double pose[7]) {
  if (!c) return GLIO_ERR_ARG;
  return guarded(c, [&] {
    GLIO_REQUIRE(frame >= 0 && pose, GLIO_ERR_ARG, "bad frame arguments");
    auto& fp = c->frames[frame];
    if (!fp) fp.reset(new glio_ctx::Frame());
    stage_points(c, fp->surf.pts, scan_xyz, Q, stride, mem);
    fp->set_pose(pose);
  });
}

// pose-only update (association always uses the poses registered here — the reference uses pose_info_keyframe, quirk Q8)
int glio_batch_set_pose(glio_ctx* c, int frame, const double pose[7]) {
  if (!c) return GLIO_ERR_ARG;
  return guarded(c, [&] {
    auto it = c->frames.find(frame);
    GLIO_REQUIRE(it != c->frames.end() && pose, GLIO_ERR_ARG, "unknown frame");
    it->second->set_pose(pose);
  });
}

}  // extern "C"

namespace {

// the listed pairs grouped by searched frame (one grid, one launch per group), each group in list order; every pair must join
// two distinct known frames
std::map<int, std::vector<int64_t>> pairs_by_searched_frame(glio_ctx* c, const int32_t* pairs_cur, const int32_t* pairs_oth, int64_t n_pairs) {
  std::map<int, std::vector<int64_t>> by_oth;
  for (int64_t i = 0; i < n_pairs; ++i) {
    GLIO_REQUIRE(c->frames.count(pairs_cur[i]) && c->frames.count(pairs_oth[i]) && pairs_cur[i] != pairs_oth[i], GLIO_ERR_ARG,
                 "pair references an unknown frame");
    by_oth[pairs_oth[i]].push_back(i);
  }
  return by_oth;
}

// the grid of a searched frame's world cloud (body pose applied directly to the stored points, quirk Q7), built when stale
const GridBuild& searched_grid(glio_ctx* c, const glio_ctx::Frame& f, glio_ctx::FrameCloud& fc) {
  if (!fc.grid_valid) {
    grid_build(fc.grid, fc.pts.ptr, fc.pts.stride, fc.pts.n, f.pose, f.pose + 3, c->prm.cell_size, c->pts_per_cell, c->st, c->lc);
    fc.grid_valid = true;
  }
  return fc.grid;
}

// the pair (cur, oth) of the pair list, appended with no matches and no edges when it is not there yet
glio_ctx::Pair& pair_entry(glio_ctx* c, int cur, int oth) {
  const std::pair<int, int> key(cur, oth);
  auto it = c->pair_index.find(key);
  if (it != c->pair_index.end()) return *c->pairs[it->second];
  c->pair_index[key] = (int)c->pairs.size();
  c->pairs.emplace_back(new glio_ctx::Pair(cur, oth, &c->bin_dirty, &c->bedge_dirty));
  c->bin_dirty = true;
  return *c->pairs.back();
}

// the pair (cur, oth) of the pair list; GLIO_ERR_ARG when it is not there
glio_ctx::Pair& find_pair(glio_ctx* c, int cur, int oth) {
  auto it = c->pair_index.find(std::make_pair(cur, oth));
  GLIO_REQUIRE(it != c->pair_index.end(), GLIO_ERR_ARG, "pair is not on the pair list");
  return *c->pairs[it->second];
}

// the LiDAR pair list as (cur, oth)
std::vector<std::pair<int, int>> lidar_pairs(const glio_ctx* c) {
  std::vector<std::pair<int, int>> t;
  t.reserve(c->pairs.size());
  for (const auto& p : c->pairs) t.emplace_back(p->cur, p->oth);
  return t;
}

// a pair table into the caller's arrays (glio_batch_pair_list, glio_batch_pose_pair_list, glio_batch_dd_psr_pair_list): NULL
// arrays only count; a capacity below the pair count is GLIO_ERR_ARG with the text err
void copy_pair_table(const std::vector<std::pair<int, int>>& t, int64_t capacity, int32_t* a, int32_t* b, int64_t* n_pairs, const char* err) {
  const int64_t n = (int64_t)t.size();
  if (n_pairs) *n_pairs = n;
  if (!a && !b) return;
  GLIO_REQUIRE(capacity >= n, GLIO_ERR_ARG, err);
  for (int64_t k = 0; k < n; ++k) { if (a) a[k] = t[k].first; if (b) b[k] = t[k].second; }
}

}  // namespace

extern "C" {

int glio_batch_associate_pairs(glio_ctx* c, const int32_t* pairs_cur, const int32_t* pairs_oth, int64_t n_pairs, int64_t* n_match) {
  if (!c) return GLIO_ERR_ARG;
  return guarded(c, [&] {
    GLIO_REQUIRE(n_pairs > 0 && pairs_cur && pairs_oth, GLIO_ERR_ARG, "bad pair list");
    AssocGates gates{c->prm.batch_max_radius, c->prm.batch_dist_thres, c->prm.weight_min};
    for (auto& grp : pairs_by_searched_frame(c, pairs_cur, pairs_oth, n_pairs)) {
      glio_ctx::Frame& fo = *c->frames[grp.first];
      const GridBuild& grid = searched_grid(c, fo, fo.surf);
      const int nseg = (int)grp.second.size();
      std::vector<SegDesc> segs(nseg);
      int64_t Qt = 0;
      for (int s = 0; s < nseg; ++s) {
        const glio_ctx::Frame& fc = *c->frames[pairs_cur[grp.second[s]]];
        segs[s] = make_seg(fc.surf.pts, Qt, fc.pose);
        Qt += fc.surf.pts.n;
      }
      ensure_work(c, Qt, true, c->prm.keep_debug != 0);
      c->d_segs.reserve(nseg); c->d_dst.reserve(nseg); c->d_counts.reserve(nseg); c->h_counts.reserve(nseg);
      GLIO_CUDA_TRY(cudaMemcpyAsync(c->d_segs.p, segs.data(), nseg * sizeof(SegDesc), cudaMemcpyHostToDevice, c->st));
      AssocWork w = make_work(c, Qt, true, c->prm.keep_debug != 0);
      assoc_run(grid, c->d_segs.p, nseg, w, gates, fo.surf.pts.ptr, fo.surf.pts.stride, c->cell_count, c->cell_pos, c->scan_tmp, c->st, c->lc);
      compact_count(w, c->d_segs.p, nseg, c->w_flags.p, c->w_pos.p, c->scan_tmp, c->d_counts.p, c->st, c->lc);
      GLIO_CUDA_TRY(cudaMemcpyAsync(c->h_counts.p, c->d_counts.p, nseg * sizeof(int), cudaMemcpyDeviceToHost, c->st));
      GLIO_CUDA_TRY(cudaStreamSynchronize(c->st));
      std::vector<CompactDst> dst(nseg);
      for (int s = 0; s < nseg; ++s) {
        const int64_t i = grp.second[s];
        CorrList& l = pair_entry(c, pairs_cur[i], pairs_oth[i]).planes;
        l.n = c->h_counts.p[s];
        dst[s] = l.plane_dst(std::max<int64_t>(l.n, 1));
        if (n_match) n_match[i] = l.n;
      }
      GLIO_CUDA_TRY(cudaMemcpyAsync(c->d_dst.p, dst.data(), nseg * sizeof(CompactDst), cudaMemcpyHostToDevice, c->st));
      compact_scatter(w, c->d_segs.p, nseg, c->w_pos.p, c->d_dst.p, c->st, c->lc);
      GLIO_CUDA_TRY(cudaStreamSynchronize(c->st));   // dst/segs are stack vectors
    }
  });
}

int glio_batch_associate(glio_ctx* c, int cur, const int32_t* oth, int n_oth, int64_t* n_match) {
  if (!c || !oth || n_oth <= 0) return GLIO_ERR_ARG;
  std::vector<int32_t> cc(n_oth, cur);
  return glio_batch_associate_pairs(c, cc.data(), oth, n_oth, n_match);
}

int glio_batch_pair_list(glio_ctx* c, int64_t capacity, int32_t* cur, int32_t* oth, int64_t* n_pairs) {
  if (!c) return GLIO_ERR_ARG;
  return guarded(c, [&] { copy_pair_table(lidar_pairs(c), capacity, cur, oth, n_pairs, "capacity smaller than the pair count"); });
}

int glio_batch_get_matches(glio_ctx* c, int cur, int oth, int64_t capacity, float* cp, float* weight, double* normal_cent, int32_t* src, int64_t* n_out) {
  if (!c) return GLIO_ERR_ARG;
  return guarded(c, [&] { copy_matches_out(c, find_pair(c, cur, oth).planes, capacity, cp, weight, nullptr, normal_cent, src, n_out); });
}

int glio_batch_select(glio_ctx* c, int cur, int oth, const int32_t* keep, int64_t n) {
  if (!c) return GLIO_ERR_ARG;
  return guarded(c, [&] { select_keep(c, find_pair(c, cur, oth).planes, keep, n); });
}

// ---- K1be / K2be: scan-to-multiscan edge association and binary point-to-edge factors
int glio_batch_set_edge_frame(glio_ctx* c, int frame, const float* xyz, int64_t Q, int stride, int mem) {
  if (!c) return GLIO_ERR_ARG;
  return guarded(c, [&] {
    auto it = c->frames.find(frame);
    GLIO_REQUIRE(it != c->frames.end(), GLIO_ERR_STATE, "glio_batch_set_edge_frame: frame was not set with glio_batch_set_frame");
    GLIO_REQUIRE(Q >= 0 && stride >= 3 && stride <= 64, GLIO_ERR_ARG, "glio_batch_set_edge_frame: need Q >= 0 and stride_floats in [3,64]");
    glio_ctx::Frame& f = *it->second;
    PointSet& ps = f.corners.pts;
    if (Q > 0) stage_points(c, ps, xyz, Q, stride, mem);
    else { ps.clear(); ps.stride = stride; }
    f.has_edge = true; f.corners.grid_valid = false;
  });
}

// K1be over the listed pairs, one group per searched frame: its corner grid (built once, reused by every pair that searches it),
// one search + line-fit launch for all the group's queries, compaction straight into the pairs' edge lists, one host
// synchronisation for the counts.
int glio_batch_associate_edges_pairs(glio_ctx* c, const int32_t* pairs_cur, const int32_t* pairs_oth, int64_t n_pairs,
                                     const glio_edge_options* options, int64_t* n_edge) {
  if (!c) return GLIO_ERR_ARG;
  return guarded(c, [&] {
    GLIO_REQUIRE(n_pairs > 0 && pairs_cur && pairs_oth, GLIO_ERR_ARG, "bad pair list");
    const glio_edge_options o = edge_options_or_default(options);
    const auto by_oth = pairs_by_searched_frame(c, pairs_cur, pairs_oth, n_pairs);
    for (int64_t i = 0; i < n_pairs; ++i)
      GLIO_REQUIRE(c->frames[pairs_cur[i]]->has_edge && c->frames[pairs_oth[i]]->has_edge, GLIO_ERR_STATE,
                   "pair frame has no corner scan (glio_batch_set_edge_frame)");
    for (auto& grp : by_oth) {
      glio_ctx::Frame& fo = *c->frames[grp.first];
      // the group's pairs; their edge lists count as empty until the counts arrive
      std::vector<glio_ctx::Pair*> prs;
      for (int64_t i : grp.second) {
        glio_ctx::Pair& pr = pair_entry(c, pairs_cur[i], pairs_oth[i]);
        pr.edges.clear();
        prs.push_back(&pr);
        if (n_edge) n_edge[i] = 0;
      }
      if (fo.corners.pts.n == 0) continue;      // nothing to search: every query fails the radius gate
      std::vector<SegDesc> segs;
      std::vector<EdgeDst> dst;
      std::vector<int64_t> seg_item;
      int64_t Qt = 0;
      for (size_t s = 0; s < grp.second.size(); ++s) {
        const glio_ctx::Frame& fc = *c->frames[pairs_cur[grp.second[s]]];
        if (fc.corners.pts.n == 0) continue;
        segs.push_back(make_seg(fc.corners.pts, Qt, fc.pose));     // body pose applied directly to the stored points (quirk Q7)
        dst.push_back(prs[s]->edges.edge_dst(fc.corners.pts.n));
        seg_item.push_back((int64_t)s);
        Qt += fc.corners.pts.n;
      }
      if (segs.empty()) continue;
      GLIO_REQUIRE(Qt < ((int64_t)1 << 31), GLIO_ERR_ARG, "glio_batch_associate_edges_pairs: too many corner points searching one frame");
      const GridBuild& grid = searched_grid(c, fo, fo.corners);
      edge_assoc_launch(c, grid, segs, dst, Qt, o, fo.corners.pts.ptr, fo.corners.pts.stride, nullptr);
      for (size_t s = 0; s < segs.size(); ++s) {
        CorrList& e = prs[seg_item[s]]->edges;
        e.n = c->h_counts.p[s]; e.has_src = true;
        if (n_edge) n_edge[grp.second[seg_item[s]]] = e.n;
      }
    }
  });
}

int glio_batch_get_edges(glio_ctx* c, int cur, int oth, int64_t capacity, float* cp, float* pa, float* pb, double* s, int32_t* src, int64_t* n) {
  if (!c) return GLIO_ERR_ARG;
  return guarded(c, [&] {
    copy_edges_out(c, find_pair(c, cur, oth).edges, capacity, cp, pa, pb, s, src, n);
  });
}

int glio_batch_set_pair_edges(glio_ctx* c, int cur, int oth, const float* cp, const float* pa, const float* pb, const double* s, int64_t n) {
  if (!c) return GLIO_ERR_ARG;
  return guarded(c, [&] {
    GLIO_REQUIRE(cur >= 0 && oth >= 0 && cur != oth, GLIO_ERR_ARG, "bad pair");
    GLIO_REQUIRE(n >= 0 && (n == 0 || (cp && pa && pb && s)), GLIO_ERR_ARG, "null edge arrays");
    CorrList& e = pair_entry(c, cur, oth).edges;
    e.clear();
    if (n > 0) upload_edges(c, e, n, cp, pa, pb, s);
  });
}

}  // extern "C"

namespace {

// Philox key domains: one per rule and record kind, so plane and edge samples with the same seed, stream and nonce are independent
enum {
  SEL_DOMAIN_WINDOW = 0, SEL_DOMAIN_STARTEND = 1, SEL_DOMAIN_ADD = 2,
  SEL_DOMAIN_WINDOW_EDGES = 3, SEL_DOMAIN_STARTEND_EDGES = 4, SEL_DOMAIN_ADD_EDGES = 5
};

void check_select_options(const glio_select_options* o) {
  GLIO_REQUIRE(o != nullptr, GLIO_ERR_ARG, "null selection options");
  GLIO_REQUIRE(o->feature_res_num >= 1 && o->feature_res_num <= GLIO_SEL_MAX, GLIO_ERR_ARG, "feature_res_num must be in [1, 4096]");
  GLIO_REQUIRE(o->rand_set_num >= 1, GLIO_ERR_ARG, "rand_set_num must be >= 1");
  GLIO_REQUIRE(o->batch_feature_res_num >= 1 && o->batch_feature_res_num <= GLIO_SEL_MAX, GLIO_ERR_ARG, "batch_feature_res_num must be in [1, 4096]");
  GLIO_REQUIRE(o->batch_rand_set_num >= o->batch_feature_res_num, GLIO_ERR_ARG, "batch_rand_set_num must be >= batch_feature_res_num");
}

// one k_sel_sample launch over the planned segments: the table goes up in one copy from pinned memory, nothing waits for the
// stream.  The staging buffer is only rewritten once the previous call's copy has run (an event, not a stream synchronisation).
void select_launch(glio_ctx* c, const std::vector<SelSeg>& segs, int k_max, uint64_t domain, uint64_t seed, uint64_t nonce) {
  if (segs.empty()) return;
  if (!c->ev_sel) GLIO_CUDA_TRY(cudaEventCreateWithFlags(&c->ev_sel, cudaEventDisableTiming));
  else GLIO_CUDA_TRY(cudaEventSynchronize(c->ev_sel));
  c->h_sel_segs.reserve(segs.size()); c->d_sel_segs.reserve(segs.size());
  memcpy(c->h_sel_segs.p, segs.data(), segs.size() * sizeof(SelSeg));
  GLIO_CUDA_TRY(cudaMemcpyAsync(c->d_sel_segs.p, c->h_sel_segs.p, segs.size() * sizeof(SelSeg), cudaMemcpyHostToDevice, c->st));
  GLIO_CUDA_TRY(cudaEventRecord(c->ev_sel, c->st));
  select_sample_run(c->d_sel_segs.p, (int)segs.size(), k_max, seed, domain, nonce, c->st, c->lc);
}

// featureSelection's outcome (Estimator.cpp:3894-3992) for a list of n records, which follows from n alone: -1 keeps all of them
// (the reference returns), F keeps the F sampled ones, 0 keeps none (random_select off: the loop never runs)
int64_t window_select_count(int64_t n, const glio_select_options* o) {
  const int F = o->feature_res_num;
  return (n < 1 || n - 1 < F) ? -1 : o->random_select ? F : 0;
}

// the pairs (cur[i], oth[i]) of a batch selection call `fn`, with its arguments checked before anything changes: mode 0 or 1, the
// options, no pair with cur == oth or off the pair list, none listed twice, the list grouped by cur
std::vector<glio_ctx::Pair*> batch_select_pairs(glio_ctx* c, const std::string& fn, const int32_t* cur, const int32_t* oth, int64_t n_pairs,
                                                int mode, const glio_select_options* opt) {
  GLIO_REQUIRE(n_pairs >= 0 && (n_pairs == 0 || (cur && oth)), GLIO_ERR_ARG, fn + ": null pair arrays");
  GLIO_REQUIRE(mode == 0 || mode == 1, GLIO_ERR_ARG, fn + ": mode must be 0 (start/end) or 1 (incremental)");
  check_select_options(opt);
  std::vector<glio_ctx::Pair*> prs((size_t)n_pairs);
  std::set<const glio_ctx::Pair*> listed;
  std::set<int> runs_seen;
  for (int64_t i = 0; i < n_pairs; ++i) {
    GLIO_REQUIRE(cur[i] != oth[i], GLIO_ERR_ARG, fn + ": cur == oth");
    prs[i] = &find_pair(c, cur[i], oth[i]);
    GLIO_REQUIRE(listed.insert(prs[i]).second, GLIO_ERR_ARG, fn + ": pair listed twice");
    if (i == 0 || cur[i] != cur[i - 1])
      GLIO_REQUIRE(runs_seen.insert(cur[i]).second, GLIO_ERR_ARG, fn + ": pair list is not grouped by cur");
  }
  return prs;
}

// globalFeatureSelection_Batch (mode 0, Estimator.cpp:3994-4055) / globalFeatureSelectionAdd_Batch (mode 1, :4057-4116) for the
// listed pairs' record counts n[i], visited in list order: -1 keeps all records, B the B sampled ones.  A start/end pair that fails
// the size test ends the run of its cur (the reference's `return`), an incremental one only skips itself (`continue`).
std::vector<int64_t> batch_select_counts(const int32_t* cur, const std::vector<int64_t>& n, int mode, int B) {
  std::vector<int64_t> n_sel(n.size());
  bool stopped = false;
  for (size_t i = 0; i < n.size(); ++i) {
    if (i == 0 || cur[i] != cur[i - 1]) stopped = false;
    if (mode == 0) {
      if (!stopped && (n[i] - 1 < B || n[i] < 50)) stopped = true;
      n_sel[i] = stopped ? -1 : B;
    } else {
      n_sel[i] = n[i] <= B ? -1 : B;
    }
  }
  return n_sel;
}

uint64_t pair_stream(int32_t cur, int32_t oth) { return ((uint64_t)(uint32_t)cur << 32) | (uint32_t)oth; }

// The seeded selection of lists[i] with the outcomes n_sel[i] (-1 keeps every record, 0 none, k > 0 draws k records with
// stream[i]): one k_sel_sample launch in the given Philox domain; n_active[i] (nullable) receives each list's active count
void sample_lists(glio_ctx* c, const std::vector<CorrList*>& lists, const std::vector<int64_t>& n_sel, const std::vector<uint64_t>& stream,
                  int k, uint64_t domain, const glio_select_options* opt, int64_t* n_active) {
  std::vector<SelSeg> segs;
  for (size_t i = 0; i < lists.size(); ++i)
    if (n_sel[i] > 0) segs.push_back(lists[i]->sample_seg(k, stream[i]));
  select_launch(c, segs, k, domain, opt->seed, opt->nonce);
  for (size_t i = 0; i < lists.size(); ++i) {
    lists[i]->set_selection(n_sel[i]);
    if (n_active) n_active[i] = lists[i]->n_active();
  }
}

// featureSelection (Estimator.cpp:3894-3992) on one list of slots 0..W-1 (glio_select_random: the plane matches,
// glio_select_random_edges: the edges).  The outcome of every slot follows from its record count alone, so the host decides it
// here and only the sampled slots go to the device.
void select_random_slots(glio_ctx* c, CorrList Slot::*list, const char* fn, uint64_t domain, int W, const int64_t* stream_ids,
                         const glio_select_options* opt, int64_t* n_active) {
  GLIO_REQUIRE(W > 0 && W <= 4096 && stream_ids, GLIO_ERR_ARG, std::string(fn) + ": bad window arguments");
  check_select_options(opt);
  std::vector<CorrList*> lists(W);
  std::vector<int64_t> n_sel(W);
  std::vector<uint64_t> stream(W);
  for (int k = 0; k < W; ++k) {
    lists[k] = &(c->slot(k).*list);
    n_sel[k] = window_select_count(lists[k]->n, opt);
    stream[k] = (uint64_t)stream_ids[k];
  }
  sample_lists(c, lists, n_sel, stream, opt->feature_res_num, domain, opt, n_active);
}

// globalFeatureSelection_Batch (mode 0) / globalFeatureSelectionAdd_Batch (mode 1) on one list of the listed pairs
// (glio_batch_select_random: the plane matches, glio_batch_select_random_edges: the edges)
void select_random_pairs(glio_ctx* c, CorrList glio_ctx::Pair::*list, const char* fn, uint64_t domain, const int32_t* cur, const int32_t* oth,
                         int64_t n_pairs, int mode, const glio_select_options* opt, int64_t* n_active) {
  const std::vector<glio_ctx::Pair*> prs = batch_select_pairs(c, fn, cur, oth, n_pairs, mode, opt);
  std::vector<CorrList*> lists((size_t)n_pairs);
  std::vector<int64_t> n((size_t)n_pairs);
  std::vector<uint64_t> stream((size_t)n_pairs);
  for (int64_t i = 0; i < n_pairs; ++i) {
    lists[i] = &(prs[i]->*list);
    n[i] = lists[i]->n;
    stream[i] = pair_stream(cur[i], oth[i]);
  }
  const int Bn = opt->batch_feature_res_num;
  sample_lists(c, lists, batch_select_counts(cur, n, mode, Bn), stream, Bn, domain, opt, n_active);
}

}  // namespace

extern "C" {

void glio_select_default_options(glio_select_options* o) {
  if (!o) return;
  memset(o, 0, sizeof(*o));
  o->feature_res_num = 100; o->rand_set_num = 300; o->batch_feature_res_num = 25; o->batch_rand_set_num = 400;
  o->random_select = 1; o->seed = 0; o->nonce = 0;
}

int glio_select_random(glio_ctx* c, int W, const int64_t* stream_ids, const glio_select_options* opt, int64_t* n_active) {
  if (!c) return GLIO_ERR_ARG;
  return guarded(c, [&] { select_random_slots(c, &Slot::planes, "glio_select_random", SEL_DOMAIN_WINDOW, W, stream_ids, opt, n_active); });
}

int glio_select_random_edges(glio_ctx* c, int W, const int64_t* stream_ids, const glio_select_options* opt, int64_t* n_active) {
  if (!c) return GLIO_ERR_ARG;
  return guarded(c, [&] {
    select_random_slots(c, &Slot::edges, "glio_select_random_edges", SEL_DOMAIN_WINDOW_EDGES, W, stream_ids, opt, n_active);
  });
}

int glio_batch_select_random(glio_ctx* c, const int32_t* cur, const int32_t* oth, int64_t n_pairs, int mode, const glio_select_options* opt,
                             int64_t* n_active) {
  if (!c) return GLIO_ERR_ARG;
  return guarded(c, [&] {
    select_random_pairs(c, &glio_ctx::Pair::planes, "glio_batch_select_random", mode == 0 ? SEL_DOMAIN_STARTEND : SEL_DOMAIN_ADD, cur, oth,
                        n_pairs, mode, opt, n_active);
  });
}

int glio_batch_select_random_edges(glio_ctx* c, const int32_t* cur, const int32_t* oth, int64_t n_pairs, int mode, const glio_select_options* opt,
                                   int64_t* n_active) {
  if (!c) return GLIO_ERR_ARG;
  return guarded(c, [&] {
    select_random_pairs(c, &glio_ctx::Pair::edges, "glio_batch_select_random_edges",
                        mode == 0 ? SEL_DOMAIN_STARTEND_EDGES : SEL_DOMAIN_ADD_EDGES, cur, oth, n_pairs, mode, opt, n_active);
  });
}

int glio_get_selection(glio_ctx* c, int slot, int64_t capacity, int32_t* keep, int64_t* n) {
  if (!c) return GLIO_ERR_ARG;
  return guarded(c, [&] { copy_selection(c, c->slot(slot).planes, capacity, keep, n); });
}

int glio_batch_get_selection(glio_ctx* c, int cur, int oth, int64_t capacity, int32_t* keep, int64_t* n) {
  if (!c) return GLIO_ERR_ARG;
  return guarded(c, [&] { copy_selection(c, find_pair(c, cur, oth).planes, capacity, keep, n); });
}

int glio_get_edge_selection(glio_ctx* c, int slot, int64_t capacity, int32_t* keep, int64_t* n) {
  if (!c) return GLIO_ERR_ARG;
  return guarded(c, [&] { copy_selection(c, c->slot(slot).edges, capacity, keep, n); });
}

int glio_batch_get_edge_selection(glio_ctx* c, int cur, int oth, int64_t capacity, int32_t* keep, int64_t* n) {
  if (!c) return GLIO_ERR_ARG;
  return guarded(c, [&] { copy_selection(c, find_pair(c, cur, oth).edges, capacity, keep, n); });
}

}  // extern "C"

namespace {

// The incidence lists of a pair table for the block assembly, queued into d_kstart / d_inc: per keyframe k < n_kf, by a counting
// sort, its pairs in table order at inc[kstart[k] .. kstart[k+1]), role 0 where k is the pair's first keyframe, 1 where its second
void upload_incidence(glio_ctx* c, const std::vector<std::pair<int, int>>& pairs, int n_kf, DevBuf<int>& d_kstart, DevBuf<BinIncidence>& d_inc) {
  std::vector<int> kstart((size_t)n_kf + 1, 0);
  for (const auto& pr : pairs) { ++kstart[(size_t)pr.first + 1]; ++kstart[(size_t)pr.second + 1]; }
  for (size_t k = 1; k < kstart.size(); ++k) kstart[k] += kstart[k - 1];
  std::vector<BinIncidence> inc(2 * pairs.size());
  std::vector<int> fill(kstart.begin(), kstart.end() - 1);
  for (int p = 0; p < (int)pairs.size(); ++p) { inc[fill[pairs[p].first]++] = BinIncidence{p, 0}; inc[fill[pairs[p].second]++] = BinIncidence{p, 1}; }
  d_kstart.reserve(kstart.size()); d_inc.reserve(inc.size() + 1);
  GLIO_CUDA_TRY(cudaMemcpyAsync(d_kstart.p, kstart.data(), kstart.size() * sizeof(int), cudaMemcpyHostToDevice, c->st));
  if (!inc.empty()) GLIO_CUDA_TRY(cudaMemcpyAsync(d_inc.p, inc.data(), inc.size() * sizeof(BinIncidence), cudaMemcpyHostToDevice, c->st));
}

// work items + incidence lists of the binary evaluation (rebuilt when associations / selections change)
void build_bin_items(glio_ctx* c, int K) {
  if (!c->bin_dirty && c->bin_K == K) return;
  const int P = (int)c->pairs.size();
  ItemPlan<BinItem> plan(P);
  std::vector<std::pair<int, int>> kf_pairs(P);
  for (int p = 0; p < P; ++p) {
    const glio_ctx::Pair& pr = *c->pairs[p];
    GLIO_REQUIRE(pr.cur >= 0 && pr.oth >= 0 && pr.cur < K && pr.oth < K, GLIO_ERR_ARG, "pair references a keyframe outside [0, K)");
    const CorrView v = pr.planes.active();
    plan.cut(p, v.n, GLIO_ITEM_MAX, [&](int64_t f, int32_t count) { return BinItem{v.cpw + f, v.nc + 6 * f, count, pr.cur, pr.oth}; });
    kf_pairs[p] = {pr.cur, pr.oth};
  }
  c->n_bin_items = (int)plan.items.size();
  c->d_pair_sums.reserve((size_t)(P + 1) * GLIO_NACC_BIN);
  c->d_bin_diag.reserve((size_t)K * GLIO_NACC); c->d_bin_off.reserve((size_t)(P + 1) * 36); c->d_bin_poses.reserve((size_t)K * 7);
  c->h_bin_diag.reserve((size_t)K * GLIO_NACC); c->h_bin_off.reserve((size_t)(P + 1) * 36); c->h_bin_poses.reserve((size_t)K * 7);
  upload_incidence(c, kf_pairs, K, c->d_kf_inc_start, c->d_inc);
  plan.upload(c, c->d_bin_items, c->d_pair_item_start, c->d_bin_partials, GLIO_NACC_BIN);
  c->bin_dirty = false; c->bin_K = K;
}

// work items of the binary edge evaluation: each pair's active edges in runs of GLIO_ITEM_MAX, pairs in pair-list order (rebuilt
// when an edge list or its selection, K or the pair count changes, or the switch is turned; build_bin_items runs first and checks
// the pairs against K)
void build_bedge_items(glio_ctx* c, int K) {
  const int P = (int)c->pairs.size();
  if (!c->bedge_dirty && c->bedge_K == K && c->bedge_P == P) return;
  ItemPlan<BinEdgeItem> plan(P);
  for (int p = 0; p < P; ++p) {
    const glio_ctx::Pair& pr = *c->pairs[p];
    const CorrView e = pr.edges.active();
    plan.cut(p, e.n, GLIO_ITEM_MAX, [&](int64_t f, int32_t count) { return BinEdgeItem{e.cpw + f, e.pa + f, e.pb + f, count, pr.cur, pr.oth}; });
  }
  c->n_bedge_items = (int)plan.items.size();
  c->d_bedge_sums.reserve((size_t)(P + 1) * GLIO_NACC_BIN);
  plan.upload(c, c->d_bedge_items, c->d_bedge_pstart, c->d_bedge_partials, GLIO_NACC_BIN);
  c->bedge_dirty = false; c->bedge_K = K; c->bedge_P = P;
}

// the LiDAR part of a batch block evaluation: none (glio_eval_pose_factors, glio_eval_dd_psr_factors), the plane blocks
// (glio_eval_binary), plane + edge blocks (glio_batch_solve with glio_batch_use_edges on), or the edge blocks alone
// (glio_eval_binary_edge)
enum BinBlocks { BIN_NONE, BIN_PLANES, BIN_PLANES_EDGES, BIN_EDGES };

// Device evaluation of the batch blocks -> c->h_bin_diag (K x 28), c->h_bin_off: the LiDAR part, then the pose list when add_pose,
// then the DD list when add_dd.  The first group queued writes the diagonal buffer and the later ones add to it; the off-diagonal
// blocks of each group follow those of the groups before it.  With edges, each LiDAR pair's sums are S_plane + S_edge before the one
// block assembly, so the all-reduce is the same as without.  Everything is queued (kernels, the all-reduce of a sharded run, the
// copies to pinned host memory); a synchronisation of the stream makes the result visible.  Returns the off-diagonal block count.
// Without a LiDAR part the LiDAR pairs are neither read nor checked against K.
int eval_blocks_launch(glio_ctx* c, int K, const double* poses, bool want_jac, BinBlocks lidar, bool add_pose, bool add_dd) {
  if (lidar != BIN_NONE) build_bin_items(c, K);
  if (lidar == BIN_PLANES_EDGES || lidar == BIN_EDGES) build_bedge_items(c, K);
  const int P = lidar == BIN_NONE ? 0 : (int)c->pairs.size(), Pp = add_pose ? (int)c->pose.pairs.size() : 0;
  const int Pd = add_dd ? (int)c->dd.pairs.size() : 0, Pt = P + Pp + Pd;
  c->d_bin_diag.reserve((size_t)K * GLIO_NACC); c->d_bin_off.reserve((size_t)(Pt + 1) * 36); c->d_bin_poses.reserve((size_t)K * 7);
  c->h_bin_diag.reserve((size_t)K * GLIO_NACC); c->h_bin_off.reserve((size_t)(Pt + 1) * 36); c->h_bin_poses.reserve((size_t)K * 7);
  memcpy(c->h_bin_poses.p, poses, (size_t)K * 7 * sizeof(double));
  GLIO_CUDA_TRY(cudaMemcpyAsync(c->d_bin_poses.p, c->h_bin_poses.p, (size_t)K * 7 * sizeof(double), cudaMemcpyHostToDevice, c->st));
  const bool add_edges = lidar == BIN_PLANES_EDGES && c->n_bedge_items > 0;   // no edges: exactly the plane launches
  if (lidar == BIN_EDGES || add_edges)
    eval_binary_edge_run(c->d_bedge_items.p, c->n_bedge_items, c->d_bedge_pstart.p, P, c->d_bin_poses.p, want_jac, c->d_bedge_partials.p,
                         c->d_bedge_sums.p, c->st, c->lc);
  if (lidar == BIN_EDGES) {
    c->lc.begin("k_bin_assemble", c->st);
    pair_assemble_run<BinLayout>(c->d_bedge_sums.p, K, P, K, c->d_kf_inc_start.p, c->d_inc.p, want_jac, false, c->d_bin_diag.p, c->d_bin_off.p, c->st);
    c->lc.end(c->st);
  } else if (lidar != BIN_NONE)
    eval_binary_run(c->d_bin_items.p, c->n_bin_items, c->d_pair_item_start.p, P, K, c->d_bin_poses.p, c->prm.batch_score,
                    /*no loss on batch LiDAR factors, Estimator.cpp:2768*/ 0.0, want_jac, c->d_bin_partials.p, c->d_pair_sums.p,
                    c->d_kf_inc_start.p, c->d_inc.p, c->d_bin_diag.p, c->d_bin_off.p, c->st, c->lc, add_edges ? c->d_bedge_sums.p : nullptr);
  if (add_pose)
    eval_pose_run(c->d_pose_f.p, c->pose.d_fstart.p, Pp, K, c->pose.max_kf + 1, c->pose.d_inc_start.p, c->pose.d_inc.p, c->d_bin_poses.p,
                  want_jac, /*add*/ lidar != BIN_NONE, c->pose.d_sums.p, c->d_bin_diag.p, c->d_bin_off.p + (size_t)P * 36, c->st, c->lc);
  if (add_dd)
    eval_dd_psr_run(c->d_dd_f.p, c->dd.d_fstart.p, c->d_dd_sats.p, c->d_dd_w.p, c->dd_frame, Pd, K, c->dd.max_kf + 1,
                    c->dd.d_inc_start.p, c->dd.d_inc.p, c->d_bin_poses.p, want_jac, /*add*/ lidar != BIN_NONE || add_pose, c->dd.d_sums.p,
                    c->d_bin_diag.p, c->d_bin_off.p + (size_t)(P + Pp) * 36, c->st, c->lc);
  // keyframe-sharded: every rank holds the same pair lists, only its own pairs and factors carry residuals (SURVEY 8e "pose-block allreduce")
  reduce_and_fetch(c, true, want_jac, c->d_bin_diag.p, c->h_bin_diag.p, (int64_t)K * GLIO_NACC, c->d_bin_off.p, c->h_bin_off.p,
                   (int64_t)Pt * 36, "allreduce hook failed (diag)", "allreduce hook failed (off)");
  return Pt;
}

// an evaluation that adds a pair-factor list referencing a keyframe >= K is GLIO_ERR_ARG; who names the call
void require_lists_within(const glio_ctx* c, int K, bool add_pose, bool add_dd, const char* who) {
  GLIO_REQUIRE(!add_pose || c->pose.max_kf < K, GLIO_ERR_ARG, std::string(who) + ": a pose factor references a keyframe outside [0, K)");
  GLIO_REQUIRE(!add_dd || c->dd.max_kf < K, GLIO_ERR_ARG, std::string(who) + ": a DD factor references a keyframe outside [0, K)");
}

// glio_eval_binary, glio_eval_binary_edge, glio_eval_pose_factors, glio_eval_dd_psr_factors: one evaluation, its blocks on the host
// as 6x6 Hdiag / 6 g / total cost and the off-diagonal blocks
int eval_blocks_out(glio_ctx* c, const char* who, int K, const double* poses, BinBlocks lidar, bool add_pose, bool add_dd, double* Hdiag,
                    double* Hoff, double* g, double* cost) {
  if (!c) return GLIO_ERR_ARG;
  return guarded(c, [&] {
    GLIO_REQUIRE(K > 0 && poses, GLIO_ERR_ARG, "bad arguments");
    require_lists_within(c, K, add_pose, add_dd, who);
    const int n_off = eval_blocks_launch(c, K, poses, Hdiag || Hoff || g, lidar, add_pose, add_dd);
    GLIO_CUDA_TRY(cudaStreamSynchronize(c->st));
    unpack_blocks(c->h_bin_diag.p, K, Hdiag, g, nullptr);
    double ct = 0;
    for (int k = 0; k < K; ++k) ct += c->h_bin_diag.p[(size_t)k * GLIO_NACC + 27];
    if (Hoff) memcpy(Hoff, c->h_bin_off.p, (size_t)n_off * 36 * sizeof(double));
    if (cost) *cost = ct;
  });
}

// The pair plan of a factor list with keyframes i, j and an active flag (pose and DD factors): the distinct unordered pairs
// (a, b), a < b, in order of first appearance; the active factors' list positions grouped by pair, list order inside a pair
// (order[fstart[p] .. fstart[p+1])).
struct PairPlan {
  std::vector<std::pair<int, int>> pairs;
  std::vector<int> fstart, order;
  int max_kf = -1;
};
template <class F>
PairPlan plan_factor_pairs(const F* f, int64_t n) {
  PairPlan pl;
  std::map<std::pair<int, int>, int> index;
  std::vector<int> fpair((size_t)n), count;
  for (int64_t k = 0; k < n; ++k) {
    const std::pair<int, int> key(std::min(f[k].i, f[k].j), std::max(f[k].i, f[k].j));
    auto it = index.emplace(key, (int)pl.pairs.size()).first;
    if (it->second == (int)pl.pairs.size()) { pl.pairs.push_back(key); count.push_back(0); }
    fpair[k] = it->second;
    if (f[k].active) ++count[it->second];
    pl.max_kf = std::max(pl.max_kf, key.second);
  }
  const int Pn = (int)pl.pairs.size();
  pl.fstart.assign(Pn + 1, 0);
  for (int p = 0; p < Pn; ++p) pl.fstart[p + 1] = pl.fstart[p] + count[p];
  pl.order.resize((size_t)pl.fstart[Pn]);
  std::vector<int> pos(pl.fstart.begin(), pl.fstart.end() - 1);
  for (int64_t k = 0; k < n; ++k)
    if (f[k].active) pl.order[pos[fpair[k]]++] = (int)k;
  return pl;
}

// A new pair-factor list from n records (glio_batch_set_pose_factors, glio_batch_set_dd_psr_factors), after the checks every
// record shares (i != j, both in [0, max_kf); ij_err otherwise): its pair plan, the incidence lists of keyframes 0 .. max_kf of the
// list, and its active records grouped by pair into d_f, queued on the stream into buffers of their own.  The caller queues its own payload, synchronises, and only then hands the
// buffers to the context, so a failed call leaves the previous list and its buffers as they were.
template <class F, class Rec>
PairFactorList upload_pair_factors(glio_ctx* c, const Rec* f, int64_t n, int max_kf, int nacc, const char* ij_err, DevBuf<F>& d_f) {
  for (int64_t k = 0; k < n; ++k)
    GLIO_REQUIRE(f[k].i >= 0 && f[k].j >= 0 && f[k].i < max_kf && f[k].j < max_kf && f[k].i != f[k].j, GLIO_ERR_ARG, ij_err);
  PairPlan pl = plan_factor_pairs(f, n);
  std::vector<F> grouped(pl.order.size());
  for (size_t q = 0; q < grouped.size(); ++q) memcpy(&grouped[q], &f[pl.order[q]], sizeof(F));
  PairFactorList l;
  d_f.reserve(grouped.size() + 1); l.d_fstart.reserve(pl.fstart.size()); l.d_sums.reserve((pl.pairs.size() + 1) * nacc);
  if (!grouped.empty()) GLIO_CUDA_TRY(cudaMemcpyAsync(d_f.p, grouped.data(), grouped.size() * sizeof(F), cudaMemcpyHostToDevice, c->st));
  GLIO_CUDA_TRY(cudaMemcpyAsync(l.d_fstart.p, pl.fstart.data(), pl.fstart.size() * sizeof(int), cudaMemcpyHostToDevice, c->st));
  upload_incidence(c, pl.pairs, pl.max_kf + 1, l.d_inc_start, l.d_inc);
  l.pairs.swap(pl.pairs); l.max_kf = pl.max_kf;
  return l;
}

static_assert(sizeof(glio_imu_factor) == sizeof(ImuFactor) && offsetof(glio_imu_factor, sum_dt) == offsetof(ImuFactor, sum_dt) &&
              offsetof(glio_imu_factor, delta_q) == offsetof(ImuFactor, delta_q) && offsetof(glio_imu_factor, dp_dba) == offsetof(ImuFactor, dp_dba) &&
              offsetof(glio_imu_factor, dv_dbg) == offsetof(ImuFactor, dv_dbg) && offsetof(glio_imu_factor, sqrt_info) == offsetof(ImuFactor, sqrt_info),
              "ImuFactor must have glio_imu_factor's layout");

// Replaces IMU list L (glio_batch_set_imu_factors, glio_window_set_imu_factors; who names the call, max_name its index bound)
void set_imu_factors(glio_ctx* c, ImuFactorList& L, const glio_imu_factor* f, int64_t n, int max_kf, const char* who, const char* max_name) {
  const std::string w(who);
  // validate the whole list first: a refused call leaves the previous list in place
  GLIO_REQUIRE(n >= 0 && (n == 0 || f), GLIO_ERR_ARG, w + ": null factor array");
  GLIO_REQUIRE(n < ((int64_t)1 << 31), GLIO_ERR_ARG, w + ": too many factors");
  constexpr int nd = (int)((sizeof(glio_imu_factor) - offsetof(glio_imu_factor, sum_dt)) / sizeof(double));
  for (int64_t k = 0; k < n; ++k) {
    const double* d = &f[k].sum_dt;
    for (int m = 0; m < nd; ++m) GLIO_REQUIRE(std::isfinite(d[m]), GLIO_ERR_ARG, w + ": a non-finite field");
  }
  DevBuf<ImuFactor> d_f;
  PairFactorList l = upload_pair_factors(c, f, n, max_kf, GLIO_NACC_IMU, (w + ": need i != j, both in [0, " + max_name + ")").c_str(), d_f);
  GLIO_CUDA_TRY(cudaStreamSynchronize(c->st));   // also: no evaluation still reads the buffers released below
  L.d_f = std::move(d_f); L.take(std::move(l));
}

// an IMU evaluation that has arrived, on the host: Hdiag (K x 225), Hoff (n_off x 225), g (K x 15), the total cost
void imu_blocks_out(const ImuFactorList& L, int K, int n_off, double* Hdiag, double* Hoff, double* g, double* cost) {
  double ct = 0;
  for (int k = 0; k < K; ++k) {
    const double* o = L.h_diag.p + (size_t)k * GLIO_NACC_IMU_KF;
    if (Hdiag) memcpy(Hdiag + (size_t)225 * k, o, 225 * sizeof(double));
    if (g) memcpy(g + (size_t)15 * k, o + 225, 15 * sizeof(double));
    ct += o[240];
  }
  if (Hoff && n_off > 0) memcpy(Hoff, L.h_off.p, (size_t)n_off * 225 * sizeof(double));
  if (cost) *cost = ct;
}

}  // namespace

extern "C" {

int glio_eval_binary(glio_ctx* c, int K, const double* poses, double* Hdiag, double* Hoff, double* g, double* cost) {
  return eval_blocks_out(c, "glio_eval_binary", K, poses, BIN_PLANES, false, false, Hdiag, Hoff, g, cost);
}

int glio_eval_binary_edge(glio_ctx* c, int K, const double* poses, double* Hdiag, double* Hoff, double* g, double* cost) {
  return eval_blocks_out(c, "glio_eval_binary_edge", K, poses, BIN_EDGES, false, false, Hdiag, Hoff, g, cost);
}

int glio_batch_use_edges(glio_ctx* c, int on) {
  if (!c) return GLIO_ERR_ARG;
  c->batch_use_edges = on != 0; c->bedge_dirty = true;
  return GLIO_OK;
}

static_assert(sizeof(glio_pose_factor) == sizeof(PoseFactor) && offsetof(glio_pose_factor, dq) == offsetof(PoseFactor, dq) &&
              offsetof(glio_pose_factor, dp) == offsetof(PoseFactor, dp), "PoseFactor must have glio_pose_factor's layout");

int glio_batch_set_pose_factors(glio_ctx* c, const glio_pose_factor* f, int64_t n) {
  if (!c) return GLIO_ERR_ARG;
  return guarded(c, [&] {
    // validate the whole list first: a refused call leaves the previous list in place
    GLIO_REQUIRE(n >= 0 && (n == 0 || f), GLIO_ERR_ARG, "glio_batch_set_pose_factors: null factor array");
    GLIO_REQUIRE(n < ((int64_t)1 << 31), GLIO_ERR_ARG, "glio_batch_set_pose_factors: too many factors");
    for (int64_t k = 0; k < n; ++k)
      GLIO_REQUIRE(f[k].kind == GLIO_POSE_RELATIVE || f[k].kind == GLIO_POSE_DELTA_Q, GLIO_ERR_ARG, "glio_batch_set_pose_factors: need a known kind");
    DevBuf<PoseFactor> d_f;
    PairFactorList l = upload_pair_factors(c, f, n, GLIO_POSE_MAX_KF, GLIO_NACC_POSE,
                                           "glio_batch_set_pose_factors: need i != j, both in [0, GLIO_POSE_MAX_KF)", d_f);
    GLIO_CUDA_TRY(cudaStreamSynchronize(c->st));   // also: no evaluation still reads the buffers released below
    c->d_pose_f = std::move(d_f); c->pose.take(std::move(l));
  });
}

int glio_batch_pose_pair_list(glio_ctx* c, int64_t capacity, int32_t* a, int32_t* b, int64_t* n_pairs) {
  if (!c) return GLIO_ERR_ARG;
  return guarded(c, [&] { copy_pair_table(c->pose.pairs, capacity, a, b, n_pairs, "glio_batch_pose_pair_list: capacity too small"); });
}

int glio_eval_pose_factors(glio_ctx* c, int K, const double* poses, double* Hdiag, double* Hoff, double* g, double* cost) {
  return eval_blocks_out(c, "glio_eval_pose_factors", K, poses, BIN_NONE, true, false, Hdiag, Hoff, g, cost);
}

int glio_batch_use_pose_factors(glio_ctx* c, int on) {
  if (!c) return GLIO_ERR_ARG;
  c->pose.use = on != 0;
  return GLIO_OK;
}

static_assert(sizeof(glio_dd_psr_factor) == sizeof(DdPsrFactor) && offsetof(glio_dd_psr_factor, sat_offset) == offsetof(DdPsrFactor, sat_offset) &&
              offsetof(glio_dd_psr_factor, ratio) == offsetof(DdPsrFactor, ratio) && offsetof(glio_dd_psr_factor, station) == offsetof(DdPsrFactor, station),
              "DdPsrFactor must have glio_dd_psr_factor's layout");
static_assert(sizeof(glio_dd_psr_sat) == sizeof(DdPsrSat) && offsetof(glio_dd_psr_sat, psr_user) == offsetof(DdPsrSat, psr_user),
              "DdPsrSat must have glio_dd_psr_sat's layout");

int glio_batch_set_dd_psr_factors(glio_ctx* c, const glio_dd_psr_factor* f, int64_t n, const glio_dd_psr_sat* sats, int64_t n_sats,
                                  const double* W, int64_t n_w, const double* R_ecef_local, const double* anchor_ecef) {
  if (!c) return GLIO_ERR_ARG;
  return guarded(c, [&] {
    // validate the whole list first: a refused call leaves the previous list in place
    GLIO_REQUIRE(n >= 0 && (n == 0 || (f && R_ecef_local && anchor_ecef)), GLIO_ERR_ARG, "glio_batch_set_dd_psr_factors: null factor array or frame");
    GLIO_REQUIRE(n < ((int64_t)1 << 31), GLIO_ERR_ARG, "glio_batch_set_dd_psr_factors: too many factors");
    GLIO_REQUIRE(n_sats >= 0 && (n_sats == 0 || sats) && n_w >= 0 && (n_w == 0 || W), GLIO_ERR_ARG,
                 "glio_batch_set_dd_psr_factors: null satellite or weight array");
    for (int64_t k = 0; k < n; ++k) {
      const glio_dd_psr_factor& F = f[k];
      GLIO_REQUIRE(F.n_sat >= 2 && F.n_sat <= GLIO_DD_PSR_MAX_SAT && F.master >= 0 && F.master < F.n_sat, GLIO_ERR_ARG,
                   "glio_batch_set_dd_psr_factors: need 2 <= n_sat <= GLIO_DD_PSR_MAX_SAT and 0 <= master < n_sat");
      GLIO_REQUIRE(F.sat_offset >= 0 && F.sat_offset <= n_sats - F.n_sat, GLIO_ERR_ARG, "glio_batch_set_dd_psr_factors: satellites outside [0, n_sats)");
      const int64_t nw = (int64_t)(F.n_sat - 1) * (F.n_sat - 1);
      GLIO_REQUIRE(F.w_offset == -1 || (F.w_offset >= 0 && F.w_offset <= n_w - nw), GLIO_ERR_ARG,
                   "glio_batch_set_dd_psr_factors: weight outside [0, n_w) and not -1");
    }
    DevBuf<DdPsrFactor> d_f; DevBuf<DdPsrSat> d_sats; DevBuf<double> d_w;
    PairFactorList l = upload_pair_factors(c, f, n, GLIO_DD_PSR_MAX_KF, GLIO_NACC_DD,
                                           "glio_batch_set_dd_psr_factors: need i != j, both in [0, GLIO_DD_PSR_MAX_KF)", d_f);
    d_sats.reserve((size_t)n_sats + 1); d_w.reserve((size_t)n_w + 1);
    if (n_sats > 0) GLIO_CUDA_TRY(cudaMemcpyAsync(d_sats.p, sats, (size_t)n_sats * sizeof(DdPsrSat), cudaMemcpyHostToDevice, c->st));
    if (n_w > 0) GLIO_CUDA_TRY(cudaMemcpyAsync(d_w.p, W, (size_t)n_w * sizeof(double), cudaMemcpyHostToDevice, c->st));
    DdPsrFrame fr{};
    if (n > 0) { memcpy(fr.R, R_ecef_local, sizeof(fr.R)); memcpy(fr.anchor, anchor_ecef, sizeof(fr.anchor)); }
    GLIO_CUDA_TRY(cudaStreamSynchronize(c->st));   // also: no evaluation still reads the buffers released below
    c->d_dd_f = std::move(d_f); c->d_dd_sats = std::move(d_sats); c->d_dd_w = std::move(d_w); c->dd_frame = fr; c->dd.take(std::move(l));
  });
}

int glio_batch_dd_psr_pair_list(glio_ctx* c, int64_t capacity, int32_t* a, int32_t* b, int64_t* n_pairs) {
  if (!c) return GLIO_ERR_ARG;
  return guarded(c, [&] { copy_pair_table(c->dd.pairs, capacity, a, b, n_pairs, "glio_batch_dd_psr_pair_list: capacity too small"); });
}

int glio_eval_dd_psr_factors(glio_ctx* c, int K, const double* poses, double* Hdiag, double* Hoff, double* g, double* cost) {
  return eval_blocks_out(c, "glio_eval_dd_psr_factors", K, poses, BIN_NONE, false, true, Hdiag, Hoff, g, cost);
}

int glio_batch_use_dd_psr_factors(glio_ctx* c, int on) {
  if (!c) return GLIO_ERR_ARG;
  c->dd.use = on != 0;
  return GLIO_OK;
}

int glio_batch_set_imu_factors(glio_ctx* c, const glio_imu_factor* f, int64_t n) {
  if (!c) return GLIO_ERR_ARG;
  return guarded(c, [&] { set_imu_factors(c, c->imu, f, n, GLIO_IMU_MAX_KF, "glio_batch_set_imu_factors", "GLIO_IMU_MAX_KF"); });
}

int glio_batch_imu_pair_list(glio_ctx* c, int64_t capacity, int32_t* a, int32_t* b, int64_t* n_pairs) {
  if (!c) return GLIO_ERR_ARG;
  return guarded(c, [&] { copy_pair_table(c->imu.pairs, capacity, a, b, n_pairs, "glio_batch_imu_pair_list: capacity too small"); });
}

int glio_eval_imu_factors(glio_ctx* c, int K, const double* poses, const double* speed_bias, double* Hdiag, double* Hoff, double* g,
                          double* cost) {
  if (!c) return GLIO_ERR_ARG;
  return guarded(c, [&] {
    GLIO_REQUIRE(K > 0 && poses && speed_bias, GLIO_ERR_ARG, "glio_eval_imu_factors: need K > 0, poses and speed_bias");
    GLIO_REQUIRE(c->imu.max_kf < K, GLIO_ERR_ARG, "glio_eval_imu_factors: an IMU factor references a keyframe outside [0, K)");
    c->d_bin_poses.reserve((size_t)K * 7); c->h_bin_poses.reserve((size_t)K * 7);
    memcpy(c->h_bin_poses.p, poses, (size_t)K * 7 * sizeof(double));
    GLIO_CUDA_TRY(cudaMemcpyAsync(c->d_bin_poses.p, c->h_bin_poses.p, (size_t)K * 7 * sizeof(double), cudaMemcpyHostToDevice, c->st));
    const int n_off = imu_blocks_launch(c, c->imu, K, c->d_bin_poses.p, speed_bias, 0, Hdiag || Hoff || g, true);
    GLIO_CUDA_TRY(cudaStreamSynchronize(c->st));
    imu_blocks_out(c->imu, K, n_off, Hdiag, Hoff, g, cost);
  });
}

int glio_batch_use_imu_factors(glio_ctx* c, int on) {
  if (!c) return GLIO_ERR_ARG;
  c->imu.use = on != 0;
  return GLIO_OK;
}

// ---- the window's IMU chain (Estimator.cpp:2179-2193), from the caller's pre-integration
int glio_window_set_imu_factors(glio_ctx* c, const glio_imu_factor* f, int64_t n) {
  if (!c) return GLIO_ERR_ARG;
  return guarded(c, [&] {
    set_imu_factors(c, c->window_imu, f, n, 4096, "glio_window_set_imu_factors", "4096");
    // what the marginalisation needs of slot 0 (glio_window_marginalize)
    bool active01 = false, slot0_elsewhere = false;
    for (int64_t k = 0; k < n; ++k)
      if (f[k].active && std::min(f[k].i, f[k].j) == 0) (std::max(f[k].i, f[k].j) == 1 ? active01 : slot0_elsewhere) = true;
    c->wimu_pair01 = -1; c->wimu_slot0_elsewhere = slot0_elsewhere;
    for (size_t p = 0; active01 && p < c->window_imu.pairs.size(); ++p)
      if (c->window_imu.pairs[p] == std::make_pair(0, 1)) c->wimu_pair01 = (int)p;
  });
}

int glio_window_imu_pair_list(glio_ctx* c, int64_t capacity, int32_t* a, int32_t* b, int64_t* n_pairs) {
  if (!c) return GLIO_ERR_ARG;
  return guarded(c, [&] { copy_pair_table(c->window_imu.pairs, capacity, a, b, n_pairs, "glio_window_imu_pair_list: capacity too small"); });
}

int glio_eval_window_imu_factors(glio_ctx* c, int W, const double* poses, const double* speed_bias, int jac_kind, double* Hdiag,
                                 double* Hoff, double* g, double* cost) {
  if (!c) return GLIO_ERR_ARG;
  return guarded(c, [&] {
    GLIO_REQUIRE(W > 0 && W <= 4096 && poses && speed_bias, GLIO_ERR_ARG, "glio_eval_window_imu_factors: need 0 < W <= 4096, poses and speed_bias");
    GLIO_REQUIRE(jac_kind == 0 || jac_kind == 1, GLIO_ERR_ARG, "glio_eval_window_imu_factors: jac_kind must be 0 or 1");
    GLIO_REQUIRE(c->window_imu.max_kf < W, GLIO_ERR_ARG, "glio_eval_window_imu_factors: an IMU factor references a slot outside [0, W)");
    wait_marg_copied(c);
    upload_window_imu_poses(c, W, poses);
    const int n_off = imu_blocks_launch(c, c->window_imu, W, c->wimu_poses.p, speed_bias, jac_kind, Hdiag || Hoff || g, false);
    GLIO_CUDA_TRY(cudaStreamSynchronize(c->st));
    imu_blocks_out(c->window_imu, W, n_off, Hdiag, Hoff, g, cost);
  });
}

int glio_window_use_imu_factors(glio_ctx* c, int on) {
  if (!c) return GLIO_ERR_ARG;
  c->window_imu.use = on != 0;
  return GLIO_OK;
}

int glio_set_allreduce(glio_ctx* c, glio_allreduce_fn fn, void* user) {
  if (!c) return GLIO_ERR_ARG;
  c->allreduce = fn; c->allreduce_user = user;
  return GLIO_OK;
}

int glio_batch_declare_pairs(glio_ctx* c, const int32_t* pairs_cur, const int32_t* pairs_oth, int64_t n_pairs) {
  if (!c) return GLIO_ERR_ARG;
  return guarded(c, [&] {
    // validate the whole list first: a refused call leaves the pair list as it was
    GLIO_REQUIRE(n_pairs >= 0 && (n_pairs == 0 || (pairs_cur && pairs_oth)), GLIO_ERR_ARG, "glio_batch_declare_pairs: null pair arrays");
    for (int64_t i = 0; i < n_pairs; ++i)
      GLIO_REQUIRE(pairs_cur[i] >= 0 && pairs_oth[i] >= 0 && pairs_cur[i] != pairs_oth[i], GLIO_ERR_ARG,
                   "glio_batch_declare_pairs: pair indices must be >= 0 and distinct");
    for (int64_t i = 0; i < n_pairs; ++i) pair_entry(c, pairs_cur[i], pairs_oth[i]);
    c->bin_dirty = true;
  });
}

int glio_batch_set_pair_matches(glio_ctx* c, int cur, int oth, const float* cp, const double* normal_cent, const float* weight, int64_t n) {
  if (!c) return GLIO_ERR_ARG;
  return guarded(c, [&] {
    GLIO_REQUIRE(cur >= 0 && oth >= 0 && cur != oth, GLIO_ERR_ARG, "bad pair");
    GLIO_REQUIRE(n >= 0 && (n == 0 || (cp && normal_cent && weight)), GLIO_ERR_ARG, "null match arrays");
    CorrList& l = pair_entry(c, cur, oth).planes;
    l.clear();
    if (n > 0) upload_matches(c, l, n, cp, weight, nullptr, normal_cent);
  });
}

namespace {

// One batch problem as glio_batch_solve sees it: the state layout, the off-diagonal block order, the band's half bandwidth, and
// the evaluation of its normal equations into a host band (the host path) or into a device band (the device minimizer).
struct BatchProblem {
  glio_ctx* c; int K; bool sb; StateLayout L; int nt, n, hb;
  bool add_pose, add_dd, add_imu;
  glio_host_factors_band_fn host_factors; void* user;
  std::vector<std::pair<int, int>> off;
  std::vector<double> pz, sz;
  int n_blocks = 0; bool plan_ready = false;
  BandMat hcb;                      // the callback's band of the device path
  BatchProblem(glio_ctx* c_, int K_, bool sb_, glio_host_factors_band_fn hf, void* u, const char* who)
      : c(c_), K(K_), sb(sb_), L(K_, sb_), nt(L.nt), n(K_ * L.nt), host_factors(hf), user(u), pz((size_t)K_ * 7), sz((size_t)K_ * 9) {
    add_pose = c->pose.use && !c->pose.pairs.empty(); add_dd = c->dd.use && !c->dd.pairs.empty();
    add_imu = c->imu.use && !c->imu.pairs.empty();
    require_lists_within(c, K, add_pose, add_dd, who);
    GLIO_REQUIRE(!add_imu || sb, GLIO_ERR_ARG, std::string(who) + ": the IMU factors need speed_bias");
    GLIO_REQUIRE(!add_imu || c->imu.max_kf < K, GLIO_ERR_ARG, std::string(who) + ": an IMU factor references a keyframe outside [0, K)");
    // the keyframe pair of each off-diagonal block, in the evaluation's order: LiDAR pairs (cur, oth), then pose pairs (a, b), then
    // DD pairs (a, b)
    off = lidar_pairs(c);
    if (add_pose) off.insert(off.end(), c->pose.pairs.begin(), c->pose.pairs.end());
    if (add_dd) off.insert(off.end(), c->dd.pairs.begin(), c->dd.pairs.end());
    int span = 1;
    for (const auto& p : off) span = std::max(span, std::abs(p.first - p.second));
    if (add_imu) for (const auto& p : c->imu.pairs) span = std::max(span, p.second - p.first);
    hb = std::min((span + 1) * nt - 1, std::max(n - 1, 0));   // BandMat::reset's clamp
  }
  // the device blocks of one evaluation at the ambient state xa, and the host callback into the freshly reset band H (may be the
  // callback band of the device path); the cost as the host path sums it.  false: the callback failed.
  bool evaluate(const double* xa, bool want_jac, double* cost, BandMat* H, double* g) {
    L.unpack(xa, pz.data(), sz.data());
    // the device evaluates the LiDAR pairs (and a sharded run sums them over the ranks) while the host evaluates its own
    // factors into the freshly reset band; the device blocks are added when they have arrived
    eval_blocks_launch(c, K, pz.data(), want_jac, c->batch_use_edges ? BIN_PLANES_EDGES : BIN_PLANES, add_pose, add_dd);
    if (add_imu) imu_blocks_launch(c, c->imu, K, c->d_bin_poses.p, sz.data(), 0, want_jac, true);
    double ct = 0;
    int hrc = 0;
    if (want_jac) { H->reset(n, hb); std::fill(g, g + n, 0.0); }
    if (host_factors) hrc = host_factors(user, K, pz.data(), sb ? sz.data() : nullptr, want_jac ? 1 : 0, want_jac ? H->a.data() : nullptr, want_jac ? H->hb : 0, g, &ct);
    GLIO_CUDA_TRY(cudaStreamSynchronize(c->st));
    if (hrc != 0) return false;
    for (int k = 0; k < K; ++k) ct += c->h_bin_diag.p[(size_t)k * GLIO_NACC + 27];
    if (add_imu) for (int k = 0; k < K; ++k) ct += c->imu.h_diag.p[(size_t)k * GLIO_NACC_IMU_KF + 240];
    *cost = ct;
    return std::isfinite(ct);
  }
  // the host path: the blocks that have arrived added into H and g in the order LiDAR / pose / DD diagonal and off-diagonal, IMU
  void host_add(BandMat* H, double* g) {
    const int w = H->hb + 1;
    double* a = H->a.data();
    add_diag_blocks(H, c->h_bin_diag.p, K, nt);
    for (int k = 0; k < K; ++k) for (int p = 0; p < 6; ++p) g[nt * k + p] += c->h_bin_diag.p[(size_t)k * GLIO_NACC + 21 + p];
    for (size_t pi = 0; pi < off.size(); ++pi) {
      const int kc = off[pi].first, ko = off[pi].second;
      const double* ob = c->h_bin_off.p + pi * 36;                 // d2 cost / d x_cur[p] d x_oth[q]
      if (kc > ko) {                                               // rows of cur, six contiguous band entries each
        for (int p = 0; p < 6; ++p) { double* row = a + (size_t)(nt * kc + p) * w + (nt * ko - (nt * kc + p) + H->hb); for (int q = 0; q < 6; ++q) row[q] += ob[6 * p + q]; }
      } else if (kc < ko) {                                        // stored transposed: rows of oth
        for (int q = 0; q < 6; ++q) { double* row = a + (size_t)(nt * ko + q) * w + (nt * kc - (nt * ko + q) + H->hb); for (int p = 0; p < 6; ++p) row[p] += ob[6 * p + q]; }
      } else {
        for (int p = 0; p < 6; ++p) for (int q = 0; q < 6; ++q) H->add_sym(nt * kc + p, nt * ko + q, ob[6 * p + q]);
      }
    }
    if (add_imu) { double unused = 0; add_imu_blocks(c->imu, K, true, H, g, unused); }   // the IMU blocks after all others
  }
  bool host_eval(const double* xa, bool want_jac, double* cost, BandMat* H, double* g) {
    if (!evaluate(xa, want_jac, cost, H, g)) return false;
    if (want_jac) host_add(H, g);
    return true;
  }
  // the assembly plan of the device path (once per problem): per band block its contributions in the host path's order
  void build_plan() {
    if (plan_ready) return;
    std::map<std::pair<int, int>, std::vector<BandContrib>> per;
    for (int k = 0; k < K; ++k) per[{k, k}].push_back(BandContrib{BAND_DIAG6, k});
    for (size_t pi = 0; pi < off.size(); ++pi) {
      const int kc = off[pi].first, ko = off[pi].second;
      if (kc > ko) per[{kc, ko}].push_back(BandContrib{BAND_OFF6, (int)pi});
      else per[{ko, kc}].push_back(BandContrib{BAND_OFF6_T, (int)pi});
    }
    if (add_imu) {
      for (int k = 0; k < K; ++k) per[{k, k}].push_back(BandContrib{BAND_IMU_DIAG, k});
      for (size_t pi = 0; pi < c->imu.pairs.size(); ++pi) per[{c->imu.pairs[pi].second, c->imu.pairs[pi].first}].push_back(BandContrib{BAND_IMU_OFF_T, (int)pi});
    }
    std::vector<BandBlock> blocks; std::vector<BandContrib> contrib;
    for (auto& kv : per) {
      blocks.push_back(BandBlock{kv.first.first, kv.first.second, (int)contrib.size(), (int)(contrib.size() + kv.second.size())});
      contrib.insert(contrib.end(), kv.second.begin(), kv.second.end());
    }
    n_blocks = (int)blocks.size();
    c->dm_blocks.reserve(blocks.size() + 1); c->dm_contrib.reserve(contrib.size() + 1);
    GLIO_CUDA_TRY(cudaMemcpyAsync(c->dm_blocks.p, blocks.data(), blocks.size() * sizeof(BandBlock), cudaMemcpyHostToDevice, c->st));
    GLIO_CUDA_TRY(cudaMemcpyAsync(c->dm_contrib.p, contrib.data(), contrib.size() * sizeof(BandContrib), cudaMemcpyHostToDevice, c->st));
    GLIO_CUDA_TRY(cudaStreamSynchronize(c->st));
    plan_ready = true;
  }
  // the device path: the callback's band and g uploaded, then the device blocks gathered onto them (k_band_assemble) into d_H;
  // g comes back to the host
  bool device_eval(const double* xa, bool want_jac, double* cost, double* d_H, double* g) {
    if (!evaluate(xa, want_jac, cost, &hcb, g)) return false;
    if (!want_jac) return true;
    build_plan();
    const size_t nb = (size_t)n * (hb + 1);
    if (host_factors) GLIO_CUDA_TRY(cudaMemcpyAsync(d_H, hcb.a.data(), nb * sizeof(double), cudaMemcpyHostToDevice, c->st));
    else GLIO_CUDA_TRY(cudaMemsetAsync(d_H, 0, nb * sizeof(double), c->st));
    GLIO_CUDA_TRY(cudaMemcpyAsync(c->dm_g.p, g, (size_t)n * sizeof(double), cudaMemcpyHostToDevice, c->st));
    band_assemble_run(d_H, hb, nt, c->dm_blocks.p, n_blocks, c->dm_contrib.p, c->d_bin_diag.p, c->d_bin_off.p,
                      add_imu ? c->imu.d_diag.p : nullptr, add_imu ? c->imu.d_off.p : nullptr, c->dm_g.p, n, c->st, c->lc);
    GLIO_CUDA_TRY(cudaMemcpyAsync(g, c->dm_g.p, (size_t)n * sizeof(double), cudaMemcpyDeviceToHost, c->st));
    GLIO_CUDA_TRY(cudaStreamSynchronize(c->st));
    return true;
  }
};

// The minimizer's band operations on the device: H and Hc in c->dm_H, Hs, A; n-vectors through pinned staging
struct DeviceBandOps : BandOps {
  BatchProblem& P; glio_ctx* c; int n, hb; int cur = 0; bool bcr;
  explicit DeviceBandOps(BatchProblem& p) : P(p), c(p.c), n(p.n), hb(p.hb), bcr(p.c->batch_factorization == GLIO_FACTOR_BCR) {
    const size_t nb = (size_t)n * (hb + 1);
    if (bcr) {
      GLIO_REQUIRE(hb <= GLIO_BAND_BCR_MAX_HB, GLIO_ERR_ARG,
                   "glio_batch_solve: the device solver's BCR factorisation needs a half bandwidth <= GLIO_BAND_BCR_MAX_HB (256)");
      c->bcr.reserve(n, hb);
    } else {
      GLIO_REQUIRE(hb <= GLIO_BAND_MAX_HB, GLIO_ERR_ARG, "glio_batch_solve: the device solver needs a half bandwidth <= GLIO_BAND_MAX_HB (160)");
      c->dm_A.reserve(nb);
    }
    c->dm_H[0].reserve(nb); c->dm_H[1].reserve(nb); c->dm_Hs.reserve(nb);
    c->dm_g.reserve(n); c->dm_v1.reserve(n); c->dm_v2.reserve(n); c->dm_v3.reserve(n); c->dm_flag.reserve(1);
    c->dm_h1.reserve(n); c->dm_h2.reserve(n);
    P.hcb.reset(n, hb);
  }
  bool eval(const double* x, bool want_jac, double* cost, int slot, double* g) override {
    return P.device_eval(x, want_jac, cost, c->dm_H[slot ? 1 - cur : cur].p, g);
  }
  bool shape_ok(int) const override { return true; }
  void down(const double* d, double* h) {
    GLIO_CUDA_TRY(cudaMemcpyAsync(c->dm_h1.p, d, (size_t)n * sizeof(double), cudaMemcpyDeviceToHost, c->st));
    GLIO_CUDA_TRY(cudaStreamSynchronize(c->st));
    memcpy(h, c->dm_h1.p, (size_t)n * sizeof(double));
  }
  void up(const double* h, double* d) {
    memcpy(c->dm_h2.p, h, (size_t)n * sizeof(double));
    GLIO_CUDA_TRY(cudaMemcpyAsync(d, c->dm_h2.p, (size_t)n * sizeof(double), cudaMemcpyHostToDevice, c->st));
  }
  void diag(double* d) override {
    GLIO_CUDA_TRY(cudaMemcpy2DAsync(c->dm_h1.p, sizeof(double), c->dm_H[cur].p + hb, (hb + 1) * sizeof(double), sizeof(double), n,
                                    cudaMemcpyDeviceToHost, c->st));
    GLIO_CUDA_TRY(cudaStreamSynchronize(c->st));
    memcpy(d, c->dm_h1.p, (size_t)n * sizeof(double));
  }
  void scale(const double* s, double* hs_diag) override {
    up(s, c->dm_v1.p);
    band_scale_run(c->dm_H[cur].p, c->dm_Hs.p, c->dm_v1.p, n, hb, c->dm_v2.p, c->st, c->lc);
    down(c->dm_v2.p, hs_diag);
  }
  bool shifted_solve(const double* v, const double* rhs, double* y) override {
    up(v, c->dm_v1.p);
    GLIO_CUDA_TRY(cudaStreamSynchronize(c->st));   // the staging buffer is reused for rhs
    up(rhs, c->dm_v2.p);
    int ok = 0;
    if (bcr) {                                     // gathers Hs + diag(v * v) itself: no k_band_shift
      bcr_solve_run(c->bcr, c->dm_Hs.p, c->dm_v1.p, c->dm_v2.p, c->dm_v3.p, n, hb, c->st, c->lc);
      int bad = 1;
      GLIO_CUDA_TRY(cudaMemcpyAsync(&bad, c->bcr.flag.p, sizeof(int), cudaMemcpyDeviceToHost, c->st));
      down(c->dm_v3.p, y);
      return bad == 0;
    }
    band_shift_run(c->dm_Hs.p, c->dm_A.p, c->dm_v1.p, n, hb, c->st, c->lc);
    band_chol_solve_run(c->dm_A.p, c->dm_v2.p, c->dm_v3.p, n, hb, c->dm_flag.p, c->st, c->lc);
    GLIO_CUDA_TRY(cudaMemcpyAsync(&ok, c->dm_flag.p, sizeof(int), cudaMemcpyDeviceToHost, c->st));
    down(c->dm_v3.p, y);
    return ok == 1;
  }
  void symv(const double* x, double* y) override {
    up(x, c->dm_v1.p);
    band_symv_run(c->dm_Hs.p, c->dm_v1.p, c->dm_v2.p, n, hb, c->st, c->lc);
    down(c->dm_v2.p, y);
  }
  void swap() override { cur = 1 - cur; }
};

}  // namespace

int glio_batch_use_device_solver(glio_ctx* c, int on) {
  if (!c) return GLIO_ERR_ARG;
  c->batch_device_solver = on != 0;
  return GLIO_OK;
}

int glio_batch_device_factorization(glio_ctx* c, int kind) {
  if (!c || (kind != GLIO_FACTOR_SEQUENTIAL && kind != GLIO_FACTOR_BCR)) return GLIO_ERR_ARG;
  c->batch_factorization = kind;
  return GLIO_OK;
}

int glio_batch_solve(glio_ctx* c, int K, double* poses, double* speed_bias, glio_host_factors_band_fn host_factors, void* user,
                     const glio_solver_options* options, glio_solver_summary* summary, glio_iteration* iter_log, int iter_cap,
                     double* step_log, int64_t step_cap) {
  if (!c) return GLIO_ERR_ARG;
  return guarded(c, [&] {
    GLIO_REQUIRE(K > 0 && poses, GLIO_ERR_ARG, "bad arguments");
    glio_solver_options o;
    if (options) o = *options;
    else { glio_default_solver_options(&o); o.dogleg_type = 1; o.use_nonmonotonic_steps = 1; o.max_num_iterations = 100; }  // Estimator.cpp:3276-3281
    BatchProblem P(c, K, speed_bias != nullptr, host_factors, user, "glio_batch_solve");
    TrustRegionDogleg solver(P.L.blocks(), solver_options_from(o));
    std::vector<double> x((size_t)K * P.L.na);
    P.L.pack(poses, speed_bias, x.data());
    SolverSummary S;
    if (c->batch_device_solver) {
      DeviceBandOps ops(P);
      solver.solve(x.data(), ops, &S);
    } else {
      EvalFn eval = [&](const double* xa, bool want_jac, double* cost, BandMat* H, double* g) -> bool { return P.host_eval(xa, want_jac, cost, H, g); };
      solver.solve(x.data(), eval, &S);
    }
    P.L.unpack(x.data(), poses, speed_bias);
    fill_summary(S, P.n, summary, iter_log, iter_cap, step_log, step_cap);
  });
}

int glio_batch_normal_equations(glio_ctx* c, int K, const double* poses, const double* speed_bias, glio_host_factors_band_fn host_factors,
                                void* user, int on_device, int64_t capacity, double* Hband, int* hb, double* g, double* cost) {
  if (!c) return GLIO_ERR_ARG;
  return guarded(c, [&] {
    GLIO_REQUIRE(K > 0 && poses && hb && g && cost, GLIO_ERR_ARG, "glio_batch_normal_equations: need K > 0, poses, hb, g and cost");
    BatchProblem P(c, K, speed_bias != nullptr, host_factors, user, "glio_batch_normal_equations");
    *hb = P.hb;
    const size_t nb = (size_t)P.n * (P.hb + 1);
    GLIO_REQUIRE(Hband && capacity >= (int64_t)nb, GLIO_ERR_ARG, "glio_batch_normal_equations: capacity smaller than n * (hb + 1)");
    std::vector<double> x((size_t)K * P.L.na);
    P.L.pack(poses, speed_bias, x.data());
    bool ok;
    if (on_device) {
      GLIO_REQUIRE(P.hb <= GLIO_BAND_BCR_MAX_HB, GLIO_ERR_ARG,
                   "glio_batch_normal_equations: the device path needs hb <= GLIO_BAND_BCR_MAX_HB (256)");
      c->dm_H[0].reserve(nb); c->dm_g.reserve(P.n); P.hcb.reset(P.n, P.hb);
      ok = P.device_eval(x.data(), true, cost, c->dm_H[0].p, g);
      if (ok) {
        GLIO_CUDA_TRY(cudaMemcpyAsync(Hband, c->dm_H[0].p, nb * sizeof(double), cudaMemcpyDeviceToHost, c->st));
        GLIO_CUDA_TRY(cudaStreamSynchronize(c->st));
      }
    } else {
      BandMat H;
      ok = P.host_eval(x.data(), true, cost, &H, g);
      if (ok) memcpy(Hband, H.a.data(), nb * sizeof(double));
    }
    GLIO_REQUIRE(ok, GLIO_ERR_NUMERIC, "glio_batch_normal_equations: the host callback failed or the cost is not finite");
  });
}


int glio_band_solve(glio_ctx* c, int n, int hb, double* band, const double* b, double* x, int* ok) {
  if (!c) return GLIO_ERR_ARG;
  return guarded(c, [&] {
    GLIO_REQUIRE(n > 0 && band && b && x && ok, GLIO_ERR_ARG, "glio_band_solve: need n > 0 and band, b, x, ok");
    GLIO_REQUIRE(hb >= 0 && hb <= GLIO_BAND_MAX_HB, GLIO_ERR_ARG, "glio_band_solve: need 0 <= hb <= GLIO_BAND_MAX_HB (160)");
    const size_t nb = (size_t)n * (hb + 1);
    c->band_a.reserve(nb); c->band_b.reserve((size_t)n); c->band_x.reserve((size_t)n); c->band_flag.reserve(1);
    GLIO_CUDA_TRY(cudaMemcpyAsync(c->band_a.p, band, nb * sizeof(double), cudaMemcpyHostToDevice, c->st));
    GLIO_CUDA_TRY(cudaMemcpyAsync(c->band_b.p, b, (size_t)n * sizeof(double), cudaMemcpyHostToDevice, c->st));
    band_chol_solve_run(c->band_a.p, c->band_b.p, c->band_x.p, n, hb, c->band_flag.p, c->st, c->lc);
    GLIO_CUDA_TRY(cudaMemcpyAsync(band, c->band_a.p, nb * sizeof(double), cudaMemcpyDeviceToHost, c->st));
    GLIO_CUDA_TRY(cudaMemcpyAsync(x, c->band_x.p, (size_t)n * sizeof(double), cudaMemcpyDeviceToHost, c->st));
    GLIO_CUDA_TRY(cudaMemcpyAsync(ok, c->band_flag.p, sizeof(int), cudaMemcpyDeviceToHost, c->st));
    GLIO_CUDA_TRY(cudaStreamSynchronize(c->st));
  });
}

int glio_band_solve_bcr(glio_ctx* c, int n, int hb, const double* band, const double* b, double* x, int* ok) {
  if (!c) return GLIO_ERR_ARG;
  return guarded(c, [&] {
    GLIO_REQUIRE(n > 0 && band && b && x && ok, GLIO_ERR_ARG, "glio_band_solve_bcr: need n > 0 and band, b, x, ok");
    GLIO_REQUIRE(hb >= 0 && hb <= GLIO_BAND_BCR_MAX_HB, GLIO_ERR_ARG, "glio_band_solve_bcr: need 0 <= hb <= GLIO_BAND_BCR_MAX_HB (256)");
    const size_t nb = (size_t)n * (hb + 1);
    c->band_a.reserve(nb); c->band_b.reserve((size_t)n); c->band_x.reserve((size_t)n);
    GLIO_CUDA_TRY(cudaMemcpyAsync(c->band_a.p, band, nb * sizeof(double), cudaMemcpyHostToDevice, c->st));
    GLIO_CUDA_TRY(cudaMemcpyAsync(c->band_b.p, b, (size_t)n * sizeof(double), cudaMemcpyHostToDevice, c->st));
    bcr_solve_run(c->bcr, c->band_a.p, nullptr, c->band_b.p, c->band_x.p, n, hb, c->st, c->lc);
    int bad = 1;
    GLIO_CUDA_TRY(cudaMemcpyAsync(x, c->band_x.p, (size_t)n * sizeof(double), cudaMemcpyDeviceToHost, c->st));
    GLIO_CUDA_TRY(cudaMemcpyAsync(&bad, c->bcr.flag.p, sizeof(int), cudaMemcpyDeviceToHost, c->st));
    GLIO_CUDA_TRY(cudaStreamSynchronize(c->st));
    *ok = bad == 0 ? 1 : 0;
  });
}

// DeviceBandOps' scale, shift and symv on host buffers, in the device minimizer's own buffers (every solve fills them afresh) and
// with its staging pattern: s, then v, then x in dm_v1; hs_diag, then y in dm_v2.  One stream orders every reuse.
int glio_band_ops(glio_ctx* c, int n, int hb, const double* H, const double* s, const double* v, const double* x, double* Hs,
                  double* hs_diag, double* A, double* y) {
  if (!c) return GLIO_ERR_ARG;
  return guarded(c, [&] {
    GLIO_REQUIRE(n > 0 && H && s && v && x && Hs && hs_diag && A && y, GLIO_ERR_ARG,
                 "glio_band_ops: need n > 0 and H, s, v, x, Hs, hs_diag, A, y");
    GLIO_REQUIRE(hb >= 0 && hb <= GLIO_BAND_BCR_MAX_HB, GLIO_ERR_ARG, "glio_band_ops: need 0 <= hb <= GLIO_BAND_BCR_MAX_HB (256)");
    const size_t nb = (size_t)n * (hb + 1), bb = nb * sizeof(double), vb = (size_t)n * sizeof(double);
    c->dm_H[0].reserve(nb); c->dm_Hs.reserve(nb); c->dm_A.reserve(nb); c->dm_v1.reserve(n); c->dm_v2.reserve(n);
    GLIO_CUDA_TRY(cudaMemcpyAsync(c->dm_H[0].p, H, bb, cudaMemcpyHostToDevice, c->st));
    GLIO_CUDA_TRY(cudaMemcpyAsync(c->dm_v1.p, s, vb, cudaMemcpyHostToDevice, c->st));
    band_scale_run(c->dm_H[0].p, c->dm_Hs.p, c->dm_v1.p, n, hb, c->dm_v2.p, c->st, c->lc);
    GLIO_CUDA_TRY(cudaMemcpyAsync(hs_diag, c->dm_v2.p, vb, cudaMemcpyDeviceToHost, c->st));
    GLIO_CUDA_TRY(cudaMemcpyAsync(c->dm_v1.p, v, vb, cudaMemcpyHostToDevice, c->st));
    band_shift_run(c->dm_Hs.p, c->dm_A.p, c->dm_v1.p, n, hb, c->st, c->lc);
    GLIO_CUDA_TRY(cudaMemcpyAsync(c->dm_v1.p, x, vb, cudaMemcpyHostToDevice, c->st));
    band_symv_run(c->dm_Hs.p, c->dm_v1.p, c->dm_v2.p, n, hb, c->st, c->lc);
    GLIO_CUDA_TRY(cudaMemcpyAsync(y, c->dm_v2.p, vb, cudaMemcpyDeviceToHost, c->st));
    GLIO_CUDA_TRY(cudaMemcpyAsync(Hs, c->dm_Hs.p, bb, cudaMemcpyDeviceToHost, c->st));
    GLIO_CUDA_TRY(cudaMemcpyAsync(A, c->dm_A.p, bb, cudaMemcpyDeviceToHost, c->st));
    GLIO_CUDA_TRY(cudaStreamSynchronize(c->st));
    GLIO_CUDA_TRY(cudaGetLastError());
  });
}

// ---- K2e: edge correspondences are an input (the reference has no edge association, SURVEY fact 1)
int glio_set_edges(glio_ctx* c, int slot, const float* cp, const float* pa, const float* pb, const double* s, int64_t n) {
  if (!c) return GLIO_ERR_ARG;
  return guarded(c, [&] {
    CorrList& e = c->slot(slot).edges;
    e.clear();
    if (n > 0) upload_edges(c, e, n, cp, pa, pb, s);
  });
}

}  // extern "C"

static int eval_edge_impl(glio_ctx* c, int W, const double* poses_body, int jac_kind, double* H, double* g, double* cost) {
  if (!c) return GLIO_ERR_ARG;
  return guarded(c, [&] {
    GLIO_REQUIRE(W > 0 && W <= 4096 && poses_body, GLIO_ERR_ARG, "bad arguments");
    GLIO_REQUIRE(jac_kind == 0 || jac_kind == 1, GLIO_ERR_ARG, "jac_kind must be 0 or 1");
    // its own buffers: the solve path's cached K2e plan and h_eout stay untouched
    const ItemPlan<EdgeItem> plan = plan_edge_items(c, W);
    plan.upload(c, c->e_items, c->e_start, c->e_part, GLIO_NACC);
    c->e_out.reserve((size_t)W * GLIO_NACC); c->e_poses.reserve((size_t)W * 7);
    init_ticket(c);
    GLIO_CUDA_TRY(cudaMemcpyAsync(c->e_poses.p, poses_body, (size_t)W * 7 * sizeof(double), cudaMemcpyHostToDevice, c->st));
    const bool want_jac = H || g;
    eval_edge_run(c->e_items.p, (int)plan.items.size(), W, c->e_poses.p, eval_params(c), jac_kind, want_jac, c->e_part.p, c->e_out.p, c->e_start.p,
                  c->d_ticket.p, c->st, c->lc);
    std::vector<double> ho((size_t)W * GLIO_NACC);
    GLIO_CUDA_TRY(cudaMemcpyAsync(ho.data(), c->e_out.p, ho.size() * sizeof(double), cudaMemcpyDeviceToHost, c->st));
    GLIO_CUDA_TRY(cudaStreamSynchronize(c->st));
    unpack_blocks(ho.data(), W, H, g, cost);
  });
}

extern "C" {

int glio_eval_edge(glio_ctx* c, int W, const double* poses_body, double* H, double* g, double* cost) {
  return eval_edge_impl(c, W, poses_body, 0, H, g, cost);
}

int glio_eval_edge_kind(glio_ctx* c, int W, const double* poses_body, int jac_kind, double* H, double* g, double* cost) {
  return eval_edge_impl(c, W, poses_body, jac_kind, H, g, cost);
}

int glio_window_use_edges(glio_ctx* c, int on) {
  if (!c) return GLIO_ERR_ARG;
  return guarded(c, [&] {
    wait_marg_copied(c);
    c->use_edges = on != 0; c->edge_items_dirty = true;
  });
}

}  // extern "C"

// ------------------------------------------------------------------------------------------------------------
// front-end LiDAR odometry (SURVEY 8 f-6): LidarOdometry::run, GLIO/src/LidarOdometry.cpp:661-695
// ------------------------------------------------------------------------------------------------------------
struct glio_odom {
  glio_ctx* ctx = nullptr;
  glio_odom_options opt{};
  // the node's state; poses in its own layout q(w,x,y,z), t(x,y,z)
  bool initialized = false;             // system_initialized
  double abs_pose[7], rel_pose[7];
  int64_t n_poses = 0;                  // pose_cloud_frame->points.size()
  double last_pose[7];                  // pose_info_cloud_frame->points.back()
  bool kf = true;
  int64_t kf_num = 0, latest_frame_idx = 0;
  double trans_last_kf[3], quat_last_kf[4];
  // device state
  LocalMap lm;                          // recent_surf_frames, surf_from_map and down_size_filter_surf_map
  VoxelWork scan_vox;                   // down_size_filter_surf
  DevBuf<float> last_ds; int last_ds_stride = 3; int64_t last_ds_n = 0;   // surf_frames.back(): the previous sweep's surf_last_ds
  DevBuf<float4> in_surf, in_full, out_surf, out_full;                    // owned copy of the surf input, staging of host clouds
  const float* map_pts = nullptr; int map_stride = 3; int64_t map_n = 0;  // surf_from_map_ds of the last step
  GridBuild grid;                       // kd_tree_surf_last
  Slot slot;                            // surf_current_pts / surf_normal
  DevBuf<EvalItem> d_items; DevBuf<int> d_start; DevBuf<double> d_partials;

  void reset_state() {
    initialized = false;
    for (int k = 0; k < 7; ++k) { abs_pose[k] = k == 0 ? 1.0 : 0.0; rel_pose[k] = abs_pose[k]; last_pose[k] = abs_pose[k]; }
    n_poses = 0; kf = true; kf_num = 0; latest_frame_idx = 0;
    trans_last_kf[0] = trans_last_kf[1] = trans_last_kf[2] = 0.0;
    quat_last_kf[0] = 1.0; quat_last_kf[1] = quat_last_kf[2] = quat_last_kf[3] = 0.0;
    while (!lm.frames.empty()) lm.pop_front();   // buffers kept for the next run
    last_ds_n = 0; map_pts = nullptr; map_n = 0;
  }
};

namespace {

// VoxelGrid(0.2) of n device points (float4); *pts / *stride receive the filtered cloud, or the input when PCL passes it through
int64_t odom_voxel(glio_ctx* c, VoxelWork& w, const float4* in, int64_t n, const float** pts, int* stride) {
  if (n <= 0) { *pts = nullptr; *stride = 3; return 0; }
  const int64_t m = voxel_filter_run(w, in, n, 0.2f, c->st, c->lc);
  if (m >= 0) { *pts = w.out_xyz.p; *stride = 3; return m; }
  *pts = reinterpret_cast<const float*>(in); *stride = 4;
  return n;
}

void odom_step(glio_odom* o, const float4* surf, int64_t n_surf, const float4* full, int64_t n_full, float* surf_out, float* full_out,
               int out_mem, glio_odom_report* rep) {
  glio_ctx* c = o->ctx;
  glio_odom_report R;
  memset(&R, 0, sizeof(R));
  // outputs of this sweep, written only when the node publishes
  float4* so = nullptr; float4* fo = nullptr;
  if (out_mem == GLIO_DEVICE) { so = reinterpret_cast<float4*>(surf_out); fo = reinterpret_cast<float4*>(full_out); }
  else {
    if (surf_out && n_surf) { o->out_surf.reserve((size_t)n_surf); so = o->out_surf.p; }
    if (full_out && n_full) { o->out_full.reserve((size_t)n_full); fo = o->out_full.p; }
  }
  bool publish = false;
  double trans[3] = {0.0, 0.0, 0.0};
  int deskew = 0;
  if (!o->initialized) {
    // savePoses with abs_pose = identity and an empty surf_last_ds, then checkInitialization: the clouds pass through unchanged
    o->n_poses += 1;
    for (int k = 0; k < 7; ++k) o->last_pose[k] = o->abs_pose[k];
    o->last_ds_n = 0; o->map_n = 0;
    o->initialized = true;
    R.initialised = 1;
    publish = true;
  } else {
    odom_predict(o->abs_pose, o->rel_pose);                                    // poseInitialization
    // buildLocalMap (:267-288)
    const float* src = nullptr; int64_t src_n = 0;                              // float4 points, scan or world frame
    if (o->n_poses <= 1) { src = reinterpret_cast<const float*>(surf); src_n = n_surf; }   // the sweep's own surf cloud, scan frame
    else {
      const double t[3] = {o->last_pose[4], o->last_pose[5], o->last_pose[6]};
      const double q[4] = {o->last_pose[0], o->last_pose[1], o->last_pose[2], o->last_pose[3]};
      if (o->lm.frames.size() < 20) o->lm.push(false, o->last_ds.p, o->last_ds_stride, o->last_ds_n, t, q, c->st, c->lc);
      else if (o->latest_frame_idx != o->n_poses - 1) {
        o->lm.pop_front();
        o->latest_frame_idx = o->n_poses - 1;
        o->lm.push(false, o->last_ds.p, o->last_ds_stride, o->last_ds_n, t, q, c->st, c->lc);
      }
      bool filtered = false; int cat_stride = 4;
      src_n = o->lm.build(0.f, &src, &cat_stride, &filtered, c->st, c->lc);      // concatenation only (float4): the filter follows
    }
    // downSampleCloud (:305-313)
    o->map_n = odom_voxel(c, o->lm.vox, reinterpret_cast<const float4*>(src), src_n, &o->map_pts, &o->map_stride);
    const float* scan = nullptr; int scan_stride = 3;
    const int64_t scan_n = odom_voxel(c, o->scan_vox, surf, n_surf, &scan, &scan_stride);
    R.n_map = o->map_n; R.n_scan = scan_n;
    // updateTransformationWithCeres (:474-579)
    if (o->map_n < 10) R.skipped = 1;                                           // "Not enough feature points from the map"
    else {
      grid_build(o->grid, o->map_pts, o->map_stride, o->map_n, nullptr, nullptr, 0.f, c->pts_per_cell, c->st, c->lc);
      const int rounds = o->n_poses < 2 ? 8 : o->opt.scan_match_cnt;
      const AssocGates gates{1.0, 0.06, 0.4};
      EvalParams ep{};
      ep.q_lb[0] = 1.0; ep.lidar_const = 1.0; ep.huber_delta = 0.1; ep.unit_score = 1;       // LidarPlaneNormIncreFactor, HuberLoss(0.1)
      glio_solver_options go; glio_default_solver_options(&go);
      go.trust_region_strategy = 1; go.max_num_iterations = o->opt.max_num_iter;             // Ceres defaults: LEVENBERG_MARQUARDT
      SolverOptions sopt = solver_options_from(go);
      sopt.max_solver_time_in_seconds = o->opt.max_solver_time_s;
      o->slot.scan.ptr = scan; o->slot.scan.stride = scan_stride; o->slot.scan.n = scan_n;
      SolverSummary S;
      for (int r = 0; r < rounds; ++r) {
        double x[7] = {o->abs_pose[4], o->abs_pose[5], o->abs_pose[6], o->abs_pose[0], o->abs_pose[1], o->abs_pose[2], o->abs_pose[3]};
        int64_t nm = 0;
        if (scan_n > 0) {
          const std::array<double, 7> lp = {x[0], x[1], x[2], x[3], x[4], x[5], x[6]};
          associate_slots(c, o->grid, gates, false, std::vector<Slot*>{&o->slot}, std::vector<std::array<double, 7>>{lp}, &nm);
        }
        if (nm > 0) {
          const ItemPlan<EvalItem> plan = plan_items(std::vector<const Slot*>{&o->slot}, c->eval_slots);
          upload_items(c, 1, plan, o->d_items, o->d_start, o->d_partials);
          const EvalTarget tgt{o->d_items.p, (int)plan.items.size(), o->d_start.p, o->d_partials.p, ep};
          solve_core(c, 1, x, nullptr, nullptr, nullptr, -1, nullptr, sopt, &tgt, S);
        } else {
          // no residual uses the pose: Ceres drops the parameter blocks and Minimize returns at once (solver.cc:410-418)
          S = SolverSummary();
          S.termination = TERM_CONVERGENCE;
          S.message = "Function tolerance reached. No non-constant parameter blocks found.";
        }
        o->abs_pose[4] = x[0]; o->abs_pose[5] = x[1]; o->abs_pose[6] = x[2];
        o->abs_pose[0] = x[3]; o->abs_pose[1] = x[4]; o->abs_pose[2] = x[5]; o->abs_pose[3] = x[6];
        if (o->abs_pose[0] < 0) for (int k = 0; k < 4; ++k) o->abs_pose[k] = -o->abs_pose[k];      // unifyQuaternion (:532-542)
        R.round_n_match[r] = nm;
        R.round_iterations[r] = (int)S.iterations.size();
        R.round_successful[r] = S.num_successful_steps;
        R.round_termination[r] = S.termination;
        for (int k = 0; k < 3; ++k) R.round_pose[r][k] = o->abs_pose[4 + k];
        for (int k = 0; k < 4; ++k) R.round_pose[r][3 + k] = o->abs_pose[k];
      }
      R.n_rounds = rounds;
      fill_summary(S, 6, &R.summary, nullptr, 0, nullptr, 0);
      if (odom_keyframe_rule(o->abs_pose + 4, o->abs_pose, o->trans_last_kf, o->quat_last_kf, o->n_poses, o->kf_num)) {
        o->kf = true;
        for (int k = 0; k < 3; ++k) o->trans_last_kf[k] = o->abs_pose[4 + k];
        for (int k = 0; k < 4; ++k) o->quat_last_kf[k] = o->abs_pose[k];
      } else o->kf = false;
    }
    // savePoses: the pose and surf_last_ds of this sweep
    double prev[7];
    for (int k = 0; k < 7; ++k) { prev[k] = o->last_pose[k]; o->last_pose[k] = o->abs_pose[k]; }
    o->n_poses += 1;
    o->last_ds_stride = scan_stride; o->last_ds_n = scan_n;
    if (scan_n > 0) {
      o->last_ds.reserve((size_t)scan_n * scan_stride);
      GLIO_CUDA_TRY(cudaMemcpyAsync(o->last_ds.p, scan, (size_t)scan_n * scan_stride * sizeof(float), cudaMemcpyDeviceToDevice, c->st));
    }
    odom_relative(prev, o->abs_pose, o->rel_pose);                              // computeRelative
    if (o->kf) {
      o->kf_num = o->n_poses;
      publish = true;
      deskew = o->opt.deskew != 0;
      trans[0] = o->rel_pose[4]; trans[1] = o->rel_pose[5]; trans[2] = o->rel_pose[6];
    }
    R.keyframe = o->kf ? 1 : 0;
  }
  if (publish) {
    odom_publish_run(surf, so ? n_surf : 0, full, fo ? n_full : 0, so, fo, trans, deskew, c->st, c->lc);
    if (out_mem != GLIO_DEVICE) {
      if (so) GLIO_CUDA_TRY(cudaMemcpyAsync(surf_out, so, (size_t)n_surf * sizeof(float4), cudaMemcpyDeviceToHost, c->st));
      if (fo) GLIO_CUDA_TRY(cudaMemcpyAsync(full_out, fo, (size_t)n_full * sizeof(float4), cudaMemcpyDeviceToHost, c->st));
    }
  }
  GLIO_CUDA_TRY(cudaStreamSynchronize(c->st));
  for (int k = 0; k < 3; ++k) { R.pose[k] = o->abs_pose[4 + k]; R.rel_pose[k] = o->rel_pose[4 + k]; }
  for (int k = 0; k < 4; ++k) { R.pose[3 + k] = o->abs_pose[k]; R.rel_pose[3 + k] = o->rel_pose[k]; }
  if (rep) *rep = R;
}

}  // namespace

extern "C" {

void glio_odom_default_options(glio_odom_options* o) {
  if (!o) return;
  memset(o, 0, sizeof(*o));
  o->max_num_iter = 12; o->scan_match_cnt = 1; o->deskew = 0; o->max_solver_time_s = 0.015;   // GLIO/config/config_urban_hk.yaml:19-21
}

int glio_odom_create(glio_ctx* c, const glio_odom_options* options, glio_odom** out) {
  if (!c || !out) return GLIO_ERR_ARG;
  *out = nullptr;
  return guarded(c, [&] {
    glio_odom_options opt; if (options) opt = *options; else glio_odom_default_options(&opt);
    GLIO_REQUIRE(opt.max_num_iter >= 0 && opt.scan_match_cnt >= 1 && opt.scan_match_cnt <= GLIO_ODOM_MAX_ROUNDS && opt.max_solver_time_s >= 0.0,
                 GLIO_ERR_ARG, "glio_odom_create: need max_num_iter >= 0, 1 <= scan_match_cnt <= 8, max_solver_time_s >= 0");
    std::unique_ptr<glio_odom> o(new glio_odom());
    o->ctx = c; o->opt = opt;
    o->reset_state();
    c->odoms.push_back(o.get());
    *out = o.release();
  });
}

void glio_odom_destroy(glio_odom* o) {
  if (!o) return;
  glio_ctx* c = o->ctx;
  DeviceGuard dev; dev.use(c->device);
  cudaStreamSynchronize(c->st);          // nothing queued may still use the buffers `delete o` frees
  c->odoms.erase(std::remove(c->odoms.begin(), c->odoms.end(), o), c->odoms.end());
  delete o;
}

int glio_odom_reset(glio_odom* o) {
  if (!o) return GLIO_ERR_ARG;
  return guarded(o->ctx, [&] { GLIO_CUDA_TRY(cudaStreamSynchronize(o->ctx->st)); o->reset_state(); });
}

int glio_odom_step(glio_odom* o, const float* surf, int64_t n_surf, int surf_mem, const float* full, int64_t n_full, int full_mem,
                   float* surf_out, float* full_out, int out_mem, glio_odom_report* rep) {
  if (!o) return GLIO_ERR_ARG;
  glio_ctx* c = o->ctx;
  return guarded(c, [&] {
    // every argument is checked before anything is enqueued or any state changes
    const int64_t kMax = (int64_t)1 << 30;
    GLIO_REQUIRE(n_surf >= 0 && n_surf < kMax && (surf || n_surf == 0), GLIO_ERR_ARG, "glio_odom_step: bad surf cloud");
    GLIO_REQUIRE(n_full >= 0 && n_full < kMax && (full || n_full == 0), GLIO_ERR_ARG, "glio_odom_step: bad full cloud");
    GLIO_REQUIRE((surf_mem == GLIO_HOST || surf_mem == GLIO_DEVICE) && (full_mem == GLIO_HOST || full_mem == GLIO_DEVICE) &&
                 (out_mem == GLIO_HOST || out_mem == GLIO_DEVICE), GLIO_ERR_ARG, "glio_odom_step: mem must be GLIO_HOST or GLIO_DEVICE");
    auto dev_ok = [c](const void* p) { return on_ctx_device(c, p) && ((uintptr_t)p & 15) == 0; };
    GLIO_REQUIRE(surf_mem != GLIO_DEVICE || n_surf == 0 || dev_ok(surf), GLIO_ERR_ARG,
                 "glio_odom_step: a GLIO_DEVICE surf cloud must be 16-byte aligned memory of the context's GPU");
    GLIO_REQUIRE(full_mem != GLIO_DEVICE || n_full == 0 || dev_ok(full), GLIO_ERR_ARG,
                 "glio_odom_step: a GLIO_DEVICE full cloud must be 16-byte aligned memory of the context's GPU");
    GLIO_REQUIRE(out_mem != GLIO_DEVICE || ((!surf_out || n_surf == 0 || dev_ok(surf_out)) && (!full_out || n_full == 0 || dev_ok(full_out))),
                 GLIO_ERR_ARG, "glio_odom_step: device outputs must be 16-byte aligned memory of the context's GPU (float4 stores)");
    // the surf cloud is kept for the whole step (map of sweep 2, scan filter, pass-through): always an owned device copy
    o->in_surf.reserve((size_t)std::max<int64_t>(n_surf, 1));
    if (n_surf) GLIO_CUDA_TRY(cudaMemcpyAsync(o->in_surf.p, surf, (size_t)n_surf * sizeof(float4),
                                              surf_mem == GLIO_DEVICE ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice, c->st));
    const float4* d_full = reinterpret_cast<const float4*>(full);
    if (n_full && full_mem != GLIO_DEVICE) {
      o->in_full.reserve((size_t)n_full);
      GLIO_CUDA_TRY(cudaMemcpyAsync(o->in_full.p, full, (size_t)n_full * sizeof(float4), cudaMemcpyHostToDevice, c->st));
      d_full = o->in_full.p;
    }
    odom_step(o, o->in_surf.p, n_surf, d_full, n_full, surf_out, full_out, out_mem, rep);
  });
}

int glio_odom_get_clouds(glio_odom* o, int64_t map_capacity, float* map_xyz, int64_t* n_map, int64_t scan_capacity, float* scan_xyz, int64_t* n_scan) {
  if (!o) return GLIO_ERR_ARG;
  glio_ctx* c = o->ctx;
  return guarded(c, [&] {
    const int64_t nm = o->map_pts ? o->map_n : 0, ns = o->last_ds_n;
    if (n_map) *n_map = nm;
    if (n_scan) *n_scan = ns;
    GLIO_REQUIRE((!map_xyz || map_capacity >= nm) && (!scan_xyz || scan_capacity >= ns), GLIO_ERR_ARG, "glio_odom_get_clouds: capacity too small");
    auto fetch = [&](const float* d, int stride, int64_t n, float* xyz) {
      if (!xyz || n <= 0) return;
      std::vector<float> h((size_t)n * stride);
      GLIO_CUDA_TRY(cudaMemcpyAsync(h.data(), d, h.size() * sizeof(float), cudaMemcpyDeviceToHost, c->st));
      GLIO_CUDA_TRY(cudaStreamSynchronize(c->st));
      for (int64_t i = 0; i < n; ++i) for (int k = 0; k < 3; ++k) xyz[3 * i + k] = h[(size_t)i * stride + k];
    };
    fetch(o->map_pts, o->map_stride, nm, map_xyz);
    fetch(o->last_ds.p, o->last_ds_stride, ns, scan_xyz);
  });
}

}  // extern "C"

// ------------------------------------------------------------------------------------------------------------
// loop-closure registration (SURVEY 8 f-7): detectLoopClosure / performLoopClosure, GLIO/src/Estimator.cpp:5101-5273
// ------------------------------------------------------------------------------------------------------------
struct glio_loop {
  glio_ctx* ctx = nullptr;
  glio_loop_options opt{};
  double q_bl[4], t_bl[3];
  struct Keyframe {
    DevBuf<float> xyz;                  // surf_frames[k], packed x,y,z (lidar frame)
    int64_t n = 0;
    double pose[7];                     // pose_info_keyframe[k]: t, q
    double time = 0.0;
    float pos[3];                       // pose_keyframe[k]
  };
  std::vector<std::unique_ptr<Keyframe>> kfs;
  double time_last_loop = 0.0;
  LocalMap latest, his;                 // latest_key_frames / his_key_frames and ds_filter_his_frames
  const float* lat_pts = nullptr; int lat_stride = 3; int64_t lat_n = 0;
  const float* his_pts = nullptr; int his_stride = 3; int64_t his_n = 0;
  IcpWork icp;
};

namespace {

// the concatenation of the given keyframes moved to the world frame, filtered: returns the filtered size, *n_raw the concatenated one
int64_t loop_cloud(glio_loop* L, LocalMap& lm, const std::vector<int>& ids, int64_t* n_raw, const float** pts, int* stride) {
  glio_ctx* c = L->ctx;
  while (!lm.frames.empty()) lm.pop_front();
  for (int k : ids) {
    const glio_loop::Keyframe& kf = *L->kfs[k];
    double t[3], q[4];
    loop_world_of_cloud(kf.pose, L->q_bl, L->t_bl, t, q);
    lm.push(false, kf.xyz.p, 3, kf.n, t, q, c->st, c->lc);               // *cloud += *transformCloud(surf_frames[k], q_tmp, t_tmp)
  }
  *n_raw = lm.n_points();
  bool filtered = false;
  return lm.build(L->opt.leaf, pts, stride, &filtered, c->st, c->lc);     // ds_filter_his_frames.filter
}

void fill_icp_result(const IcpState& h, int64_t n_src, int64_t n_tgt, int syncs, int64_t launches, glio_icp_result* r) {
  memset(r, 0, sizeof(*r));
  r->converged = h.converged; r->state = h.state; r->iterations = h.nr_iter; r->host_syncs = syncs;
  r->n_source = n_src; r->n_target = n_tgt; r->n_corr = h.n_corr; r->launches = launches;
  for (int k = 0; k < 16; ++k) r->final_transformation[k] = h.final_T[k];
  r->fitness = h.fitness;
}

void loop_step(glio_loop* L, const float sel[3], double time_new_odom, glio_loop_report* rep) {
  glio_ctx* c = L->ctx;
  glio_loop_report R;
  memset(&R, 0, sizeof(R));
  R.closest_his_idx = -1; R.latest_frame_idx = -1;
  R.icp.fitness = DBL_MAX;
  const int K = (int)L->kfs.size();
  if (K > 0) {                                                               // performLoopClosure: pose_keyframe->points.empty()
    // kd_tree_his_key_poses->radiusSearch(select_pose, lc_search_radius, ...): FLANN's float L2_Simple distance, kept when below
    // float(radius^2), sorted by (distance, index)
    const float r2 = (float)(L->opt.lc_search_radius * L->opt.lc_search_radius);
    std::vector<std::pair<float, int>> hits;
    for (int k = 0; k < K; ++k) {
      const float* p = L->kfs[k]->pos;
      const float d0 = sel[0] - p[0], d1 = sel[1] - p[1], d2 = sel[2] - p[2];
      float d = 0.f; d = d + d0 * d0; d = d + d1 * d1; d = d + d2 * d2;
      if (d < r2) hits.emplace_back(d, k);
    }
    std::sort(hits.begin(), hits.end());
    R.n_candidates = (int64_t)hits.size();
    for (auto& h : hits)
      if (std::abs(L->kfs[h.second]->time - time_new_odom) > L->opt.lc_time_thres) { R.closest_his_idx = h.second; break; }
    if (R.closest_his_idx >= 0 && !(std::abs(L->time_last_loop - time_new_odom) < 0.2)) {
      R.detected = 1;
      const int latest = K - L->opt.slide_window_width;
      R.latest_frame_idx = latest;
      std::vector<int> ids;
      for (int j = 0; j < 6; ++j) if (latest - j >= 0) ids.push_back(latest - j);
      L->lat_n = loop_cloud(L, L->latest, ids, &R.n_latest, &L->lat_pts, &L->lat_stride);
      ids.clear();
      for (int j = -L->opt.lc_map_width; j <= L->opt.lc_map_width; ++j) {
        const int k = R.closest_his_idx + j;
        if (k < 0 || k > latest) continue;
        ids.push_back(k);
      }
      L->his_n = loop_cloud(L, L->his, ids, &R.n_his, &L->his_pts, &L->his_stride);
      R.n_latest_ds = L->lat_n; R.n_his_ds = L->his_n;
      // pcl::IterativeClosestPoint: source latest_key_frames_ds, target his_key_frames_ds, identity guess; then getFitnessScore
      const int64_t l0 = c->lc.n;
      IcpState h; int syncs = 0;
      icp_run(L->icp, L->lat_pts, L->lat_stride, L->lat_n, L->his_pts, L->his_stride, L->his_n, L->opt.icp, 0, c->pts_per_cell, c->st, c->lc, &h, &syncs);
      fill_icp_result(h, L->lat_n, L->his_n, syncs, c->lc.n - l0, &R.icp);
      if (h.converged && !(h.fitness > (double)L->opt.lc_icp_thres)) {
        R.accepted = 1;
        loop_pose_from(h.final_T, L->kfs[latest]->pose, R.pose_from);
        for (int k = 0; k < 7; ++k) R.pose_to[k] = L->kfs[R.closest_his_idx]->pose[k];
        R.noise_score = h.fitness;
        L->time_last_loop = L->kfs[latest]->time;
      }
    }
  }
  R.time_last_loop = L->time_last_loop;
  if (rep) *rep = R;
}

bool dev_ptr_ok(const glio_ctx* c, const void* p, uintptr_t align) { return on_ctx_device(c, p) && ((uintptr_t)p & (align - 1)) == 0; }

}  // namespace

extern "C" {

void glio_icp_default_options(glio_icp_options* o) {
  if (!o) return;
  memset(o, 0, sizeof(*o));
  o->max_iterations = 100; o->max_correspondence_distance = 30.0; o->transformation_epsilon = 1e-6; o->euclidean_fitness_epsilon = 1e-6;
}

static void check_icp_options(const glio_icp_options& o) {
  GLIO_REQUIRE(o.max_iterations >= 1 && o.max_iterations <= 100000 && o.max_correspondence_distance > 0.0 &&
               std::isfinite(o.max_correspondence_distance) && o.transformation_epsilon >= 0.0 && o.euclidean_fitness_epsilon >= 0.0,
               GLIO_ERR_ARG, "icp options: need 1 <= max_iterations <= 100000, a finite positive correspondence distance, epsilons >= 0");
}

int glio_icp_align(glio_ctx* c, const float* src, int64_t n_src, int src_stride, int src_mem, const float* tgt, int64_t n_tgt, int tgt_stride,
                   int tgt_mem, const glio_icp_options* options, float* aligned_xyz, glio_icp_result* res, glio_icp_iteration* iter_log,
                   int iter_cap, int32_t* corr_query, int32_t* corr_match, float* corr_dist, int64_t corr_cap) {
  if (!c) return GLIO_ERR_ARG;
  return guarded(c, [&] {
    glio_icp_options o; if (options) o = *options; else glio_icp_default_options(&o);
    check_icp_options(o);
    const int64_t kMax = (int64_t)1 << 30;
    GLIO_REQUIRE(n_src >= 0 && n_src < kMax && (src || n_src == 0) && n_tgt >= 0 && n_tgt < kMax && (tgt || n_tgt == 0), GLIO_ERR_ARG,
                 "glio_icp_align: bad cloud pointer or size");
    GLIO_REQUIRE(src_stride >= 3 && src_stride <= 64 && tgt_stride >= 3 && tgt_stride <= 64, GLIO_ERR_ARG, "glio_icp_align: stride_floats must be in [3,64]");
    GLIO_REQUIRE((src_mem == GLIO_HOST || src_mem == GLIO_DEVICE) && (tgt_mem == GLIO_HOST || tgt_mem == GLIO_DEVICE), GLIO_ERR_ARG,
                 "glio_icp_align: mem must be GLIO_HOST or GLIO_DEVICE");
    GLIO_REQUIRE((src_mem != GLIO_DEVICE || n_src == 0 || dev_ptr_ok(c, src, 4)) && (tgt_mem != GLIO_DEVICE || n_tgt == 0 || dev_ptr_ok(c, tgt, 4)),
                 GLIO_ERR_ARG, "glio_icp_align: a GLIO_DEVICE cloud must be 4-byte aligned memory of the context's GPU");
    GLIO_REQUIRE(iter_cap >= 0 && (iter_log || iter_cap == 0) && corr_cap >= 0, GLIO_ERR_ARG, "glio_icp_align: bad log capacities");
    const float* ds = src; const float* dt = tgt;
    if (n_src && src_mem != GLIO_DEVICE) ds = stage_points(c, c->icp_src, src, n_src, src_stride, src_mem);
    if (n_tgt && tgt_mem != GLIO_DEVICE) dt = stage_points(c, c->icp_tgt, tgt, n_tgt, tgt_stride, tgt_mem);
    const int64_t l0 = c->lc.n;
    IcpState h; int syncs = 0;
    icp_run(c->icp, ds, src_stride, n_src, dt, tgt_stride, n_tgt, o, iter_cap, c->pts_per_cell, c->st, c->lc, &h, &syncs);
    if (res) fill_icp_result(h, n_src, n_tgt, syncs, c->lc.n - l0, res);
    if (aligned_xyz && n_src > 0) {
      std::vector<float4> a((size_t)n_src);
      GLIO_CUDA_TRY(cudaMemcpyAsync(a.data(), c->icp.fit.p, (size_t)n_src * sizeof(float4), cudaMemcpyDeviceToHost, c->st));
      GLIO_CUDA_TRY(cudaStreamSynchronize(c->st));
      unpack_float4(a.data(), n_src, aligned_xyz);
    }
    const int nlog = std::min(iter_cap, h.nr_iter);
    if (iter_log && nlog > 0) {
      GLIO_CUDA_TRY(cudaMemcpyAsync(iter_log, c->icp.log.p, (size_t)nlog * sizeof(glio_icp_iteration), cudaMemcpyDeviceToHost, c->st));
      GLIO_CUDA_TRY(cudaStreamSynchronize(c->st));
    }
    const int64_t nc = std::min<int64_t>(corr_cap, h.n_corr);
    if (nc > 0 && n_src > 0 && n_tgt > 0) {
      if (corr_query) GLIO_CUDA_TRY(cudaMemcpyAsync(corr_query, c->icp.cq.p, (size_t)nc * sizeof(int32_t), cudaMemcpyDeviceToHost, c->st));
      if (corr_match) GLIO_CUDA_TRY(cudaMemcpyAsync(corr_match, c->icp.cm.p, (size_t)nc * sizeof(int32_t), cudaMemcpyDeviceToHost, c->st));
      if (corr_dist) GLIO_CUDA_TRY(cudaMemcpyAsync(corr_dist, c->icp.cd.p, (size_t)nc * sizeof(float), cudaMemcpyDeviceToHost, c->st));
      GLIO_CUDA_TRY(cudaStreamSynchronize(c->st));
    }
  });
}

void glio_loop_default_options(glio_loop_options* o) {
  if (!o) return;
  memset(o, 0, sizeof(*o));
  o->lc_search_radius = 25.0; o->lc_time_thres = 30.0; o->lc_map_width = 25; o->lc_icp_thres = 0.2f;   // config_urban_hk.yaml:80-83
  o->slide_window_width = 5; o->leaf = 0.4f;
  o->q_lb[0] = 1.0; o->t_lb[2] = 0.28;                                                                  // :90-97
  glio_icp_default_options(&o->icp);
}

int glio_loop_create(glio_ctx* c, const glio_loop_options* options, glio_loop** out) {
  if (!c || !out) return GLIO_ERR_ARG;
  *out = nullptr;
  return guarded(c, [&] {
    glio_loop_options opt; if (options) opt = *options; else glio_loop_default_options(&opt);
    check_icp_options(opt.icp);
    GLIO_REQUIRE(opt.lc_search_radius > 0.0 && std::isfinite(opt.lc_search_radius) && opt.lc_time_thres >= 0.0 && opt.lc_map_width >= 0 &&
                 opt.lc_map_width <= 100000 && opt.slide_window_width >= 1 && opt.leaf > 0.f && std::isfinite(opt.lc_icp_thres),
                 GLIO_ERR_ARG, "glio_loop_create: need lc_search_radius > 0, lc_time_thres >= 0, lc_map_width >= 0, slide_window_width >= 1, leaf > 0");
    const double n2 = opt.q_lb[0] * opt.q_lb[0] + opt.q_lb[1] * opt.q_lb[1] + opt.q_lb[2] * opt.q_lb[2] + opt.q_lb[3] * opt.q_lb[3];
    GLIO_REQUIRE(n2 > 0.0 && std::isfinite(n2), GLIO_ERR_ARG, "glio_loop_create: q_lb must be a non-zero finite quaternion");
    std::unique_ptr<glio_loop> L(new glio_loop());
    L->ctx = c; L->opt = opt;
    loop_extrinsic_bl(opt.q_lb, opt.t_lb, L->q_bl, L->t_bl);
    c->loops.push_back(L.get());
    *out = L.release();
  });
}

void glio_loop_destroy(glio_loop* L) {
  if (!L) return;
  glio_ctx* c = L->ctx;
  DeviceGuard dev; dev.use(c->device);
  cudaStreamSynchronize(c->st);          // nothing queued may still use the buffers `delete L` frees
  c->loops.erase(std::remove(c->loops.begin(), c->loops.end(), L), c->loops.end());
  delete L;
}

int glio_loop_reset(glio_loop* L) {
  if (!L) return GLIO_ERR_ARG;
  return guarded(L->ctx, [&] {
    GLIO_CUDA_TRY(cudaStreamSynchronize(L->ctx->st));
    L->kfs.clear();
    L->time_last_loop = 0.0;
    L->lat_pts = L->his_pts = nullptr; L->lat_n = L->his_n = 0;
  });
}

int glio_loop_add_keyframe(glio_loop* L, const float* cloud, int64_t n, int stride, int mem, const double pose[7], double time, int32_t* index) {
  if (!L) return GLIO_ERR_ARG;
  glio_ctx* c = L->ctx;
  return guarded(c, [&] {
    GLIO_REQUIRE(n >= 0 && n < ((int64_t)1 << 30) && (cloud || n == 0), GLIO_ERR_ARG, "glio_loop_add_keyframe: bad cloud pointer or size");
    GLIO_REQUIRE(stride >= 3 && stride <= 64, GLIO_ERR_ARG, "glio_loop_add_keyframe: stride_floats must be in [3,64]");
    GLIO_REQUIRE(mem == GLIO_HOST || mem == GLIO_DEVICE, GLIO_ERR_ARG, "glio_loop_add_keyframe: mem must be GLIO_HOST or GLIO_DEVICE");
    GLIO_REQUIRE(mem != GLIO_DEVICE || n == 0 || dev_ptr_ok(c, cloud, 4), GLIO_ERR_ARG,
                 "glio_loop_add_keyframe: a GLIO_DEVICE cloud must be 4-byte aligned memory of the context's GPU");
    GLIO_REQUIRE(pose != nullptr && std::isfinite(time), GLIO_ERR_ARG, "glio_loop_add_keyframe: null pose or non-finite time");
    for (int k = 0; k < 7; ++k) GLIO_REQUIRE(std::isfinite(pose[k]), GLIO_ERR_ARG, "glio_loop_add_keyframe: non-finite pose");
    GLIO_REQUIRE(L->kfs.size() < (size_t)0x7fffffff, GLIO_ERR_ARG, "glio_loop_add_keyframe: too many keyframes");
    std::unique_ptr<glio_loop::Keyframe> kf(new glio_loop::Keyframe());
    kf->n = n;
    if (n > 0) {
      kf->xyz.reserve((size_t)n * 3);
      // x,y,z of every point packed on the way in (one pitched copy, host or device source)
      GLIO_CUDA_TRY(cudaMemcpy2DAsync(kf->xyz.p, 3 * sizeof(float), cloud, (size_t)stride * sizeof(float), 3 * sizeof(float), (size_t)n,
                                      mem == GLIO_DEVICE ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice, c->st));
      if (mem != GLIO_DEVICE) GLIO_CUDA_TRY(cudaStreamSynchronize(c->st));    // the caller may reuse its host buffer on return
    }
    for (int k = 0; k < 7; ++k) kf->pose[k] = pose[k];
    kf->time = time;
    for (int k = 0; k < 3; ++k) kf->pos[k] = (float)pose[k];
    L->kfs.push_back(std::move(kf));
    if (index) *index = (int32_t)(L->kfs.size() - 1);
  });
}

int glio_loop_set_poses(glio_loop* L, int first, int count, const double* poses) {
  if (!L) return GLIO_ERR_ARG;
  return guarded(L->ctx, [&] {
    GLIO_REQUIRE(first >= 0 && count >= 0 && (int64_t)first + count <= (int64_t)L->kfs.size() && (poses || count == 0), GLIO_ERR_ARG,
                 "glio_loop_set_poses: keyframe range out of bounds");
    for (int64_t i = 0; i < 7 * (int64_t)count; ++i) GLIO_REQUIRE(std::isfinite(poses[i]), GLIO_ERR_ARG, "glio_loop_set_poses: non-finite pose");
    for (int i = 0; i < count; ++i) {
      glio_loop::Keyframe& kf = *L->kfs[first + i];
      for (int k = 0; k < 7; ++k) kf.pose[k] = poses[7 * i + k];
      for (int k = 0; k < 3; ++k) kf.pos[k] = (float)kf.pose[k];
    }
  });
}

int glio_loop_size(glio_loop* L, int* n_keyframes) {
  if (!L) return GLIO_ERR_ARG;
  if (n_keyframes) *n_keyframes = (int)L->kfs.size();
  return GLIO_OK;
}

int glio_loop_step(glio_loop* L, const float select_xyz[3], double time_new_odom, glio_loop_report* rep) {
  if (!L) return GLIO_ERR_ARG;
  return guarded(L->ctx, [&] {
    GLIO_REQUIRE(select_xyz != nullptr && std::isfinite(select_xyz[0]) && std::isfinite(select_xyz[1]) && std::isfinite(select_xyz[2]) &&
                 std::isfinite(time_new_odom), GLIO_ERR_ARG, "glio_loop_step: select_xyz and time_new_odom must be finite");
    loop_step(L, select_xyz, time_new_odom, rep);
  });
}

int glio_loop_get_clouds(glio_loop* L, int64_t lat_cap, float* lat_xyz, int64_t* n_lat, int64_t his_cap, float* his_xyz, int64_t* n_his) {
  if (!L) return GLIO_ERR_ARG;
  glio_ctx* c = L->ctx;
  return guarded(c, [&] {
    const int64_t nl = L->lat_pts ? L->lat_n : 0, nh = L->his_pts ? L->his_n : 0;
    if (n_lat) *n_lat = nl;
    if (n_his) *n_his = nh;
    GLIO_REQUIRE((!lat_xyz || lat_cap >= nl) && (!his_xyz || his_cap >= nh), GLIO_ERR_ARG, "glio_loop_get_clouds: capacity too small");
    auto fetch = [&](const float* d, int stride, int64_t n, float* xyz) {
      if (!xyz || n <= 0) return;
      std::vector<float> h((size_t)n * stride);
      GLIO_CUDA_TRY(cudaMemcpyAsync(h.data(), d, h.size() * sizeof(float), cudaMemcpyDeviceToHost, c->st));
      GLIO_CUDA_TRY(cudaStreamSynchronize(c->st));
      for (int64_t i = 0; i < n; ++i) for (int k = 0; k < 3; ++k) xyz[3 * i + k] = h[(size_t)i * stride + k];
    };
    fetch(L->lat_pts, L->lat_stride, nl, lat_xyz);
    fetch(L->his_pts, L->his_stride, nh, his_xyz);
  });
}

}  // extern "C"

// ------------------------------------------------------------------------------------------------------------
// pcl::VoxelGrid of any cloud and save_pcd's global map (SURVEY 8 f-8): downSampleCloud's ds_filter_surf (Estimator.cpp:3628-3630)
// and the export at :5324-5349, on the sort-based filter of grid.cu
// ------------------------------------------------------------------------------------------------------------
namespace {

void check_vs_output(glio_ctx* c, const char* who, int64_t capacity, const float* xyz, int out_mem, const int64_t* n_out) {
  GLIO_REQUIRE(n_out != nullptr && capacity >= 0 && (xyz || capacity == 0), GLIO_ERR_ARG, std::string(who) + ": bad output arguments");
  GLIO_REQUIRE(out_mem == GLIO_HOST || out_mem == GLIO_DEVICE, GLIO_ERR_ARG, std::string(who) + ": out_mem must be GLIO_HOST or GLIO_DEVICE");
  GLIO_REQUIRE(out_mem != GLIO_DEVICE || capacity == 0 || dev_ptr_ok(c, xyz, 4), GLIO_ERR_ARG,
               std::string(who) + ": a GLIO_DEVICE output must be 4-byte aligned memory of the context's GPU");
}

// the filter's result (c->vsort.out_xyz, m points) to the caller; nothing is written when it does not fit
void deliver_vs_output(glio_ctx* c, const char* who, int64_t m, bool filtered, int64_t capacity, float* xyz, int out_mem, int64_t* n_out,
                       int32_t* filt) {
  *n_out = m;
  if (filt) *filt = filtered ? 1 : 0;
  GLIO_REQUIRE(m <= capacity, GLIO_ERR_ARG, std::string(who) + ": capacity is smaller than the number of output points");
  if (m == 0) return;
  GLIO_CUDA_TRY(cudaMemcpyAsync(xyz, c->vsort.out_xyz.p, (size_t)m * 3 * sizeof(float),
                                out_mem == GLIO_DEVICE ? cudaMemcpyDeviceToDevice : cudaMemcpyDeviceToHost, c->st));
  GLIO_CUDA_TRY(cudaStreamSynchronize(c->st));
}

}  // namespace

extern "C" {

int glio_voxel_filter(glio_ctx* c, const float* xyz, int64_t n, int stride, int in_mem, float leaf, int64_t capacity, float* out_xyz,
                      int out_mem, int64_t* n_out, int32_t* filtered) {
  if (!c) return GLIO_ERR_ARG;
  return guarded(c, [&] {
    const char* who = "glio_voxel_filter";
    GLIO_REQUIRE(n >= 0 && n < ((int64_t)1 << 31) && (xyz || n == 0), GLIO_ERR_ARG, "glio_voxel_filter: bad cloud pointer or size");
    GLIO_REQUIRE(stride >= 3 && stride <= 64, GLIO_ERR_ARG, "glio_voxel_filter: stride_floats must be in [3,64]");
    GLIO_REQUIRE(in_mem == GLIO_HOST || in_mem == GLIO_DEVICE, GLIO_ERR_ARG, "glio_voxel_filter: in_mem must be GLIO_HOST or GLIO_DEVICE");
    GLIO_REQUIRE(in_mem != GLIO_DEVICE || n == 0 || dev_ptr_ok(c, xyz, 4), GLIO_ERR_ARG,
                 "glio_voxel_filter: a GLIO_DEVICE cloud must be 4-byte aligned memory of the context's GPU");
    GLIO_REQUIRE(leaf > 0.f && std::isfinite(leaf), GLIO_ERR_ARG, "glio_voxel_filter: leaf must be positive and finite");
    check_vs_output(c, who, capacity, out_xyz, out_mem, n_out);
    if (n == 0) { deliver_vs_output(c, who, 0, true, capacity, out_xyz, out_mem, n_out, filtered); return; }
    const float* d = in_mem == GLIO_DEVICE ? xyz : stage_points(c, c->vs_stage, xyz, n, stride, in_mem);
    bool f = false;
    const int64_t m = voxel_sort_run(c->vsort, d, stride, n, leaf, &f, c->st, c->lc);
    deliver_vs_output(c, who, m, f, capacity, out_xyz, out_mem, n_out, filtered);
  });
}

int glio_loop_global_map(glio_loop* L, int interval, float leaf, int64_t capacity, float* xyz, int out_mem, int64_t* n_map, int64_t* n_raw,
                         int32_t* filtered) {
  if (!L) return GLIO_ERR_ARG;
  glio_ctx* c = L->ctx;
  return guarded(c, [&] {
    const char* who = "glio_loop_global_map";
    GLIO_REQUIRE(interval >= 1, GLIO_ERR_ARG, "glio_loop_global_map: interval must be >= 1");
    GLIO_REQUIRE(leaf > 0.f && std::isfinite(leaf), GLIO_ERR_ARG, "glio_loop_global_map: leaf must be positive and finite");
    check_vs_output(c, who, capacity, xyz, out_mem, n_map);
    // keyframes 0, interval, 2 interval, ... (:5339), in that order, each after the previous one in the concatenation
    std::vector<GlobalMapSeg> segs;
    int64_t N = 0, n_max = 0;
    for (size_t i = 0; i < L->kfs.size(); i += (size_t)interval) {
      const glio_loop::Keyframe& kf = *L->kfs[i];
      if (kf.n == 0) continue;
      GlobalMapSeg g;
      g.xyz = kf.xyz.p; g.n = kf.n; g.off = N;
      for (int k = 0; k < 3; ++k) g.t[k] = kf.pose[k];
      for (int k = 0; k < 4; ++k) g.q[k] = kf.pose[3 + k];
      segs.push_back(g);
      N += kf.n; n_max = std::max(n_max, kf.n);
    }
    if (n_raw) *n_raw = N;
    if (N == 0) { deliver_vs_output(c, who, 0, true, capacity, xyz, out_mem, n_map, filtered); return; }
    GLIO_REQUIRE(N < ((int64_t)1 << 31), GLIO_ERR_ARG, "glio_loop_global_map: the concatenated map has 2^31 points or more");
    c->gm_segs.reserve(segs.size()); c->gm_cat.reserve((size_t)N);
    GLIO_CUDA_TRY(cudaMemcpyAsync(c->gm_segs.p, segs.data(), segs.size() * sizeof(GlobalMapSeg), cudaMemcpyHostToDevice, c->st));
    loop_global_map_cloud(c->gm_segs.p, (int)segs.size(), n_max, L->t_bl, L->q_bl, c->gm_cat.p, c->st, c->lc);
    bool f = false;
    const int64_t m = voxel_sort_run(c->vsort, reinterpret_cast<const float*>(c->gm_cat.p), 4, N, leaf, &f, c->st, c->lc);   // ds_filter_global_map
    deliver_vs_output(c, who, m, f, capacity, xyz, out_mem, n_map, filtered);
  });
}

}  // extern "C"
