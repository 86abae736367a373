// shim_solve.h — implementation of ceres::Solve / Problem::Evaluate for the glio_b200 Ceres-API shim (see ceres.h).
#ifndef GLIO_SHIM_CERES_SHIM_SOLVE_H_
#define GLIO_SHIM_CERES_SHIM_SOLVE_H_

#include <chrono>

namespace ceres {
namespace shim_internal {

struct ActiveBlock { double* user; int size, local, amb_off, tan_off; LocalParameterization* param; };

struct Program {
  std::vector<ActiveBlock> active;
  std::map<double*, int> index;           // user pointer -> active index
  int n_amb = 0, n_tan = 0;
};

// Ceres' Corrector (ceres.tgz::internal/ceres/corrector.cc) for a residual block with nr rows
struct Corr {
  double sqrt_rho1 = 1, residual_scaling = 1, alpha_sq_norm = 0;
  Corr(double sq_norm, const double rho[3]) {
    sqrt_rho1 = std::sqrt(rho[1]);
    if (sq_norm == 0.0 || rho[2] <= 0.0) { residual_scaling = sqrt_rho1; alpha_sq_norm = 0.0; return; }
    const double D = 1.0 + 2.0 * sq_norm * rho[2] / rho[1];
    const double alpha = 1.0 - std::sqrt(D);
    residual_scaling = sqrt_rho1 / (1 - alpha);
    alpha_sq_norm = alpha / sq_norm;
  }
  void jac(int nr, int nc, const double* r, double* J) const {
    if (alpha_sq_norm == 0.0) { for (int i = 0; i < nr * nc; ++i) J[i] *= sqrt_rho1; return; }
    for (int c = 0; c < nc; ++c) {
      double rtj = 0; for (int k = 0; k < nr; ++k) rtj += J[k * nc + c] * r[k];
      for (int k = 0; k < nr; ++k) J[k * nc + c] = sqrt_rho1 * (J[k * nc + c] - alpha_sq_norm * r[k] * rtj);
    }
  }
};

inline bool is_f32(double v) { return (double)(float)v == v; }

}  // namespace shim_internal

inline void Solve(const Solver::Options& options, Problem* problem, Solver::Summary* summary) {
  using namespace shim_internal;
  const auto t_start = std::chrono::steady_clock::now();
  Solver::Summary& S = *summary;
  S = Solver::Summary();
  // ---- reduced program (Program::RemoveFixedBlocks, ceres.tgz::internal/ceres/program.cc:296-366) ----
  std::set<double*> used;
  for (auto& rb : problem->residual_blocks_) for (double* p : rb->params) used.insert(p);
  Program P;
  for (double* u : problem->order_) {
    const Problem::Block& b = problem->blocks_.at(u);
    if (b.constant || !used.count(u)) continue;
    ActiveBlock a; a.user = u; a.size = b.size; a.param = b.param; a.local = b.param ? b.param->LocalSize() : b.size;
    a.amb_off = P.n_amb; a.tan_off = P.n_tan; P.n_amb += a.size; P.n_tan += a.local;
    P.index[u] = (int)P.active.size(); P.active.push_back(a);
  }
  S.num_parameter_blocks = (int)P.active.size(); S.num_parameters = P.n_amb; S.num_effective_parameters = P.n_tan;
  S.num_residual_blocks = problem->NumResidualBlocks(); S.num_residuals = problem->NumResiduals();
  const int n = P.n_tan;
  if (n == 0) { S.termination_type = CONVERGENCE; S.message = "no free parameters"; S.initial_cost = S.final_cost = 0; return; }

  // ---- split residual blocks: device-evaluable unary factors (plane, edge, incre) vs binary plane factors vs host ----
  // one slot per keyframe (t, q): its plane matches (LidarPlaneNormFactor, LidarPlaneNormIncreFactor) go to K2, its edges
  // (LidarEdgeFactor) to K2e
  struct Slot { double* t; double* q; std::vector<float> cp, nsd, w, ecp, epa, epb; std::vector<double> es; };
  std::vector<Slot> slots;
  std::map<std::pair<double*, double*>, int> slot_of;
  std::vector<const Problem::Residual*> host_blocks;
  struct BPair { int kc, ko; std::vector<float> cp; std::vector<double> nc; std::vector<float> w; };
  std::vector<BPair> bpairs;                                     // in creation order == glio_batch_pair_list order
  std::map<std::pair<int, int>, int> bpair_of;
  std::vector<std::pair<double*, double*>> bkfs;                 // keyframes (t, q blocks) touched by binary factors
  std::map<std::pair<double*, double*>, int> bkf_of;
  glio_ctx* ctx = problem->ctx_;
  glio_params gp;
  if (ctx && glio_get_params(ctx, &gp) != GLIO_OK) ctx = nullptr;
  auto slot_at = [&](double* t, double* q) -> Slot& {
    auto key = std::make_pair(t, q);
    auto it = slot_of.find(key);
    if (it != slot_of.end()) return slots[it->second];
    slot_of[key] = (int)slots.size(); slots.push_back(Slot{t, q, {}, {}, {}, {}, {}, {}, {}});
    return slots.back();
  };
  // the kernels apply the context's Huber(huber_delta), or no loss when huber_delta <= 0
  auto loss_ok = [&](const LossFunction* loss) {
    const HuberLoss* hl = dynamic_cast<const HuberLoss*>(loss);
    return (loss == nullptr && gp.huber_delta <= 0) || (hl && hl->a() == gp.huber_delta);
  };
  auto quat_ok = [&](double* q) {
    return P.index.count(q) && problem->blocks_.at(q).size == 4 && dynamic_cast<QuaternionParameterization*>(problem->blocks_.at(q).param) != nullptr;
  };
  auto ext_ok = [&](const double* q_lb, const double* t_lb) {
    bool ok = true;
    for (int k = 0; k < 4; ++k) ok = ok && q_lb[k] == gp.q_lb[k];
    for (int k = 0; k < 3; ++k) ok = ok && t_lb[k] == gp.t_lb[k];
    return ok;
  };
  auto trans_ok = [&](double* t) { return P.index.count(t) && problem->blocks_.at(t).size == 3 && problem->blocks_.at(t).param == nullptr; };
  // the plane routes' keyframe (t, q): unlike trans_ok, t may have a local parameterization
  auto tq_ok = [&](double* t, double* q) { return P.index.count(t) && problem->blocks_.at(t).size == 3 && quat_ok(q); };
  // the batch keyframe table's index of (t, q), appended if new
  auto kf_index = [&](double* t, double* q) {
    auto key = std::make_pair(t, q);
    auto it = bkf_of.find(key);
    if (it != bkf_of.end()) return it->second;
    const int k = (int)bkfs.size(); bkf_of[key] = k; bkfs.push_back(key); return k;
  };
  auto f32_3 = [](const double* v) { return is_f32(v[0]) && is_f32(v[1]) && is_f32(v[2]); };
  auto add_plane = [](Slot& sl, const glio::FactorDesc& d, double w) {
    for (int k = 0; k < 3; ++k) sl.cp.push_back((float)d.cp[k]);
    for (int k = 0; k < 3; ++k) sl.nsd.push_back((float)d.n[k]);
    sl.nsd.push_back((float)d.d); sl.w.push_back((float)w);
  };
  int n_edge_dev = 0;
  // pose-factor candidates: routed after the loop, once every keyframe (t, q) pairing of the problem is known
  struct PoseCand { const Problem::Residual* rb; glio::FactorDesc d; };
  std::vector<PoseCand> pose_cands;
  // DD-pseudorange candidates: routed after the pose factors, on the same keyframe table.  Each candidate's satellites and
  // weight go into the arrays glio_batch_set_dd_psr_factors takes; those of candidates left on the host stay there unused.
  struct DdCand { const Problem::Residual* rb; glio_dd_psr_factor f; };
  std::vector<DdCand> dd_cands;
  std::vector<glio_dd_psr_sat> dd_sats;
  std::vector<double> dd_W;
  std::unique_ptr<glio::DdPsrDesc> dd_desc(new glio::DdPsrDesc());
  // ImuFactor candidates: routed after the DD factors, on the same table, with their descriptions (i, j set there)
  struct ImuCand { const Problem::Residual* rb; glio_imu_factor f; };
  std::vector<ImuCand> imu_cands;
  auto sb_ok = [&](double* sb) { return P.index.count(sb) && problem->blocks_.at(sb).size == 9 && problem->blocks_.at(sb).param == nullptr; };
  for (auto& rbp : problem->residual_blocks_) {
    const Problem::Residual* rb = rbp.get();
    glio::FactorDesc d;
    bool dev = false;
    const bool described = ctx && rb->cost->GlioDescribe(&d);
    if (!described) d.kind = glio::FACTOR_NONE;
    if (described && d.kind == glio::FACTOR_PLANE_UNARY && rb->params.size() == 2) {
      double* t = rb->params[0]; double* q = rb->params[1];
      // unit_score contexts evaluate every match with score = lidar_const (front-end factor): only blocks with exactly that score qualify
      const double w = gp.unit_score ? 1.0 : d.score / gp.lidar_const;
      const bool repr = (gp.unit_score ? d.score == gp.lidar_const : (is_f32(w) && gp.lidar_const * (double)(float)w == d.score)) && f32_3(d.cp) &&
                        f32_3(d.n) && is_f32(d.d);
      if (loss_ok(rb->loss) && tq_ok(t, q) && ext_ok(d.q_lb, d.t_lb) && repr) {
        add_plane(slot_at(t, q), d, w);
        dev = true;
      }
    }
    // LidarEdgeFactor (LidarKeyframeFactor.h:12-70): blocks (t, q), t without a local parameterization; K2e stores the weight s
    // as a float, so it has to be one as well
    if (described && d.kind == glio::FACTOR_EDGE_UNARY && rb->params.size() == 2) {
      double* t = rb->params[0]; double* q = rb->params[1];
      const bool repr = f32_3(d.cp) && f32_3(d.pa) && f32_3(d.pb) && is_f32(d.score);
      if (loss_ok(rb->loss) && trans_ok(t) && quat_ok(q) && ext_ok(d.q_lb, d.t_lb) && repr) {
        Slot& sl = slot_at(t, q);
        for (int k = 0; k < 3; ++k) { sl.ecp.push_back((float)d.cp[k]); sl.epa.push_back((float)d.pa[k]); sl.epb.push_back((float)d.pb[k]); }
        sl.es.push_back(d.score);
        ++n_edge_dev;
        dev = true;
      }
    }
    // LidarPlaneNormIncreFactor (LidarKeyframeFactor.h:222-257): blocks in the order (q, t), no score and no extrinsic -- K2 computes
    // exactly that residual in a front-end context (unit_score = 1, lidar_const = 1, identity extrinsic)
    if (described && d.kind == glio::FACTOR_PLANE_INCRE && rb->params.size() == 2) {
      double* q = rb->params[0]; double* t = rb->params[1];
      const double ident_q[4] = {1, 0, 0, 0}, zero_t[3] = {0, 0, 0};
      const bool ctx_ok = gp.unit_score && gp.lidar_const == 1.0 && ext_ok(ident_q, zero_t);
      const bool repr = f32_3(d.cp) && f32_3(d.n) && is_f32(d.d);
      if (ctx_ok && loss_ok(rb->loss) && trans_ok(t) && quat_ok(q) && repr) {
        add_plane(slot_at(t, q), d, 1.0);
        dev = true;
      }
    }
    // BinaryLidarPlaneNormFactor (LidarKeyframeFactor.h:124-164): four blocks (t_cur, q_cur, t_oth, q_oth), no loss
    // (Estimator.cpp:2768); grouped by keyframe pair and evaluated by K2b
    if (!dev && ctx && d.kind == glio::FACTOR_PLANE_BINARY && rb->params.size() == 4 && rb->loss == nullptr && gp.batch_score != 0.0) {
      double* tc = rb->params[0]; double* qc = rb->params[1]; double* to = rb->params[2]; double* qo = rb->params[3];
      const double w = d.score / gp.batch_score;
      const bool repr = is_f32(w) && gp.batch_score * (double)(float)w == d.score && is_f32(d.cp[0]) && is_f32(d.cp[1]) && is_f32(d.cp[2]);
      if (tq_ok(tc, qc) && tq_ok(to, qo) && !(tc == to && qc == qo) && repr) {
        const int kc = kf_index(tc, qc), ko = kf_index(to, qo);
        auto pkey = std::make_pair(kc, ko);
        auto pit = bpair_of.find(pkey);
        int pi;
        if (pit == bpair_of.end()) { pi = (int)bpairs.size(); bpair_of[pkey] = pi; bpairs.push_back(BPair{kc, ko, {}, {}, {}}); } else pi = pit->second;
        BPair& bp = bpairs[pi];
        for (int k = 0; k < 3; ++k) bp.cp.push_back((float)d.cp[k]);
        for (int k = 0; k < 6; ++k) bp.nc.push_back(d.nc[k]);
        bp.w.push_back((float)w);
        dev = true;
      }
    }
    // LidarPoseFactorBatchRelativeAutoDiff (LidarPoseFactor.h:54-95, blocks t_i, q_i, t_j, q_j) and delta_q_factor_auto
    // (LidarKeyframeFactor.h:281-304, blocks q_i, q_j), both added without a loss (Estimator.cpp:2863, :2924): K2p evaluates them
    // when every block is active, each q a QuaternionParameterization and each t a plain 3-vector.  A candidate stays in
    // host_blocks until the keyframe table below takes it.
    if (!dev && rb->loss == nullptr &&
        ((d.kind == glio::FACTOR_POSE_RELATIVE && rb->params.size() == 4 && trans_ok(rb->params[0]) && quat_ok(rb->params[1]) &&
          trans_ok(rb->params[2]) && quat_ok(rb->params[3])) ||
         (d.kind == glio::FACTOR_POSE_DELTA_Q && rb->params.size() == 2 && quat_ok(rb->params[0]) && quat_ok(rb->params[1]))))
      pose_cands.push_back(PoseCand{rb, d});
    // dd_psr_factor_20 (dd_psr_factor.hpp, added without a loss at Estimator.cpp:1910): K2g computes exactly its residual when the
    // blocks are (t_i, t_j, yaw, anchor) of sizes (3, 3, 1, 3), both t active plain 3-vectors of different keyframes, yaw and
    // anchor constant, and the description within K2g's limits.  A candidate stays in host_blocks until the keyframe table takes it.
    if (!dev && ctx && rb->describer && rb->describer->describe_dd_psr && rb->loss == nullptr && rb->params.size() == 4) {
      const std::vector<int32_t>& sz = rb->cost->parameter_block_sizes();
      double* const* b = rb->params.data();
      const bool shape = sz[0] == 3 && sz[1] == 3 && sz[2] == 1 && sz[3] == 3 && problem->blocks_.at(b[2]).size == 1 &&
                         problem->blocks_.at(b[3]).size == 3 && trans_ok(b[0]) && trans_ok(b[1]) && b[0] != b[1] &&
                         !P.index.count(b[2]) && !P.index.count(b[3]);
      if (shape) *dd_desc = glio::DdPsrDesc();
      if (shape && rb->describer->describe_dd_psr(rb->cost, dd_desc.get()) && dd_desc->n_sat >= 2 && dd_desc->n_sat <= GLIO_DD_PSR_MAX_SAT &&
          dd_desc->master >= 0 && dd_desc->master < dd_desc->n_sat) {
        const glio::DdPsrDesc& dd = *dd_desc;
        glio_dd_psr_factor f;
        f.i = f.j = -1; f.n_sat = dd.n_sat; f.master = dd.master; f.active = 1; f.reserved = 0;
        f.sat_offset = (int64_t)dd_sats.size();
        f.w_offset = dd.w_identity ? -1 : (int64_t)dd_W.size();
        f.ratio = dd.ratio; f.threshold = dd.threshold;
        for (int k = 0; k < 3; ++k) f.station[k] = dd.station[k];
        for (int s_ = 0; s_ < dd.n_sat; ++s_) {
          glio_dd_psr_sat sat;
          for (int k = 0; k < 3; ++k) { sat.sat_user[k] = dd.sat_user[s_][k]; sat.sat_ref[k] = dd.sat_ref[s_][k]; }
          sat.psr_user = dd.psr_user[s_]; sat.psr_ref = dd.psr_ref[s_];
          dd_sats.push_back(sat);
        }
        if (!dd.w_identity) dd_W.insert(dd_W.end(), dd.W, dd.W + (size_t)(dd.n_sat - 1) * (dd.n_sat - 1));
        dd_cands.push_back(DdCand{rb, f});
      }
    }
    // ImuFactor (ImuFactor.h, added without a loss at Estimator.cpp:2993-3001): K2i computes exactly its residual and Jacobian when
    // the blocks are (t_i, q_i, sb_i, t_j, q_j, sb_j) of sizes (3, 4, 9, 3, 4, 9), all active, each t a plain 3-vector, each q a
    // QuaternionParameterization and each sb a plain 9-vector, the two keyframes different, and the description finite (K2i's
    // list takes finite records only).  A candidate stays in host_blocks until the keyframe table takes it.
    if (!dev && ctx && rb->describer && rb->describer->describe_imu && rb->loss == nullptr && rb->params.size() == 6) {
      const std::vector<int32_t>& sz = rb->cost->parameter_block_sizes();
      double* const* b = rb->params.data();
      const bool shape = sz[0] == 3 && sz[1] == 4 && sz[2] == 9 && sz[3] == 3 && sz[4] == 4 && sz[5] == 9 && trans_ok(b[0]) && quat_ok(b[1]) &&
                         sb_ok(b[2]) && trans_ok(b[3]) && quat_ok(b[4]) && sb_ok(b[5]) && !(b[0] == b[3] && b[1] == b[4]);
      glio_imu_factor f;
      std::memset(&f, 0, sizeof(f));
      if (shape && rb->describer->describe_imu(rb->cost, &f)) {
        bool finite = true;
        const double* v = &f.sum_dt;
        for (size_t k = 0; k < (sizeof(f) - offsetof(glio_imu_factor, sum_dt)) / sizeof(double); ++k) finite = finite && std::isfinite(v[k]);
        f.i = f.j = -1; f.active = 1; f.reserved = 0;
        if (finite) imu_cands.push_back(ImuCand{rb, f});
      }
    }
    if (!dev) host_blocks.push_back(rb);
  }
  const int W = (int)slots.size();
  const int KB = (int)bkfs.size(), PB = (int)bpairs.size();

  // ---- pose factors on the batch keyframe table ----
  // Binary-plane and pose blocks that share a (t, q) pair share one keyframe; a q seen only in delta_q blocks is a keyframe of
  // its own without a t (t = NULL: rotation columns only).  A q paired with two t blocks, or a t with two q blocks, has no single
  // keyframe: the pose blocks that touch it stay on the host.  So do blocks whose two sides are one keyframe.
  std::vector<glio_pose_factor> pose_list;
  std::map<double*, std::set<double*>> ts_of_q, qs_of_t;
  std::set<const Problem::Residual*> routed;                     // pose, DD and IMU blocks the keyframe table takes off the host
  {
    auto pairing = [&](double* t, double* q) { ts_of_q[q].insert(t); qs_of_t[t].insert(q); };
    for (const auto& kf : bkfs) pairing(kf.first, kf.second);
    for (const PoseCand& c : pose_cands)
      if (c.d.kind == glio::FACTOR_POSE_RELATIVE) { pairing(c.rb->params[0], c.rb->params[1]); pairing(c.rb->params[2], c.rb->params[3]); }
    for (const ImuCand& c : imu_cands) { pairing(c.rb->params[0], c.rb->params[1]); pairing(c.rb->params[3], c.rb->params[4]); }
    auto q_single = [&](double* q) {
      auto it = ts_of_q.find(q);
      if (it == ts_of_q.end()) return true;
      return it->second.size() == 1 && qs_of_t.at(*it->second.begin()).size() == 1;
    };
    auto kf_of_q = [&](double* q) {
      auto it = ts_of_q.find(q);
      return kf_index(it == ts_of_q.end() ? nullptr : *it->second.begin(), q);
    };
    for (const PoseCand& c : pose_cands) {
      const bool rel = c.d.kind == glio::FACTOR_POSE_RELATIVE;
      double* qi = c.rb->params[rel ? 1 : 0]; double* qj = c.rb->params[rel ? 3 : 1];
      if (qi == qj || !q_single(qi) || !q_single(qj)) continue;
      glio_pose_factor f;
      f.i = kf_of_q(qi); f.j = kf_of_q(qj); f.kind = rel ? GLIO_POSE_RELATIVE : GLIO_POSE_DELTA_Q; f.active = 1;
      for (int k = 0; k < 4; ++k) f.dq[k] = c.d.dq[k];
      for (int k = 0; k < 3; ++k) f.dp[k] = rel ? c.d.dp[k] : 0.0;
      pose_list.push_back(f);
      routed.insert(c.rb);
    }
  }

  // ---- DD pseudorange factors on the same table ----
  // A t paired with one q by the binary-plane or pose blocks (and that q with no other t) is the keyframe (t, q); a t seen in no
  // such pairing is a keyframe of its own without a q (q = NULL: translation columns only, an identity quaternion in the pose
  // array, which K2g does not read).  A t with two q blocks, or whose q has two t blocks, keeps its DD blocks on the host.  K2g
  // takes one R and anchor per list: only the blocks that share the first candidate's constant yaw and anchor blocks (and frame())
  // are routed.
  std::vector<glio_dd_psr_factor> dd_list;
  double dd_R[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1}, dd_anchor[3] = {0, 0, 0};
  {
    auto t_single = [&](double* t) {
      auto it = qs_of_t.find(t);
      return it == qs_of_t.end() || (it->second.size() == 1 && ts_of_q.at(*it->second.begin()).size() == 1);
    };
    auto kf_of_t = [&](double* t) {
      auto it = qs_of_t.find(t);
      return kf_index(t, it == qs_of_t.end() ? nullptr : *it->second.begin());
    };
    const Problem::Residual* first = nullptr;
    for (const DdCand& c : dd_cands) {
      double* const* b = c.rb->params.data();
      if (first && (b[2] != first->params[2] || b[3] != first->params[3] || c.rb->describer->frame != first->describer->frame)) continue;
      if (!t_single(b[0]) || !t_single(b[1])) continue;
      if (!first) {
        first = c.rb;
        c.rb->describer->frame(b[2], b[3], dd_R);
        for (int k = 0; k < 3; ++k) dd_anchor[k] = b[3][k];
      }
      glio_dd_psr_factor f = c.f;
      f.i = kf_of_t(b[0]); f.j = kf_of_t(b[1]);
      dd_list.push_back(f);
      routed.insert(c.rb);
    }
  }

  // ---- IMU factors on the same table ----
  // A keyframe (t, q) whose t pairs with that q alone (and that q with that t alone) takes the IMU blocks whose sb is used by IMU
  // candidates with that keyframe only, while the keyframe is used with that sb only: then K2i's 15 columns per keyframe are
  // [t, delta, sb], and the keyframe's sb columns are its own.  Every other IMU candidate stays on the host.
  std::vector<glio_imu_factor> imu_list;
  std::vector<double*> bkf_sb;                                   // each batch keyframe's sb block (NULL: none)
  {
    std::map<double*, std::set<std::pair<double*, double*>>> kfs_of_sb;
    std::map<std::pair<double*, double*>, std::set<double*>> sbs_of_kf;
    for (const ImuCand& c : imu_cands)
      for (int s = 0; s < 2; ++s) {
        double* const* b = c.rb->params.data() + 3 * s;
        kfs_of_sb[b[2]].insert(std::make_pair(b[0], b[1])); sbs_of_kf[std::make_pair(b[0], b[1])].insert(b[2]);
      }
    auto side_ok = [&](double* const* b) {
      return qs_of_t.at(b[0]).size() == 1 && ts_of_q.at(b[1]).size() == 1 && kfs_of_sb.at(b[2]).size() == 1 && sbs_of_kf.at(std::make_pair(b[0], b[1])).size() == 1;
    };
    for (const ImuCand& c : imu_cands) {
      double* const* b = c.rb->params.data();
      if (!side_ok(b) || !side_ok(b + 3)) continue;
      glio_imu_factor f = c.f;
      f.i = kf_index(b[0], b[1]); f.j = kf_index(b[3], b[4]);
      bkf_sb.resize(bkfs.size(), nullptr);
      bkf_sb[f.i] = b[2]; bkf_sb[f.j] = b[5];
      imu_list.push_back(f);
      routed.insert(c.rb);
    }
  }
  if (!routed.empty())
    host_blocks.erase(std::remove_if(host_blocks.begin(), host_blocks.end(), [&](const Problem::Residual* rb) { return routed.count(rb) != 0; }),
                      host_blocks.end());
  // keyframes of K2b (the first KB), K2p, K2g and K2i; routed pose, DD and IMU blocks
  const int KT = (int)bkfs.size(), NP = (int)pose_list.size(), ND = (int)dd_list.size(), NI = (int)imu_list.size();
  bkf_sb.resize(KT, nullptr);
  auto fail = [&](const char* call) { S.termination_type = FAILURE; S.message = std::string(call) + ": " + glio_last_error(ctx); };
  // the batch evaluations of the present kinds, in the order eval adds them (K2b, K2p, K2g): the glio_eval_* call, its keyframe
  // count, its Hoff pair table (block (a, b): row = a tangent, col = b tangent) and the columns it fills of each keyframe's 6
  struct BatchEval { decltype(&glio_eval_binary) fn; int K; std::vector<int32_t> a, b; int nc; };
  std::vector<BatchEval> batch;
  // a glio_batch_*_pair_list table: its size, then its entries
  auto fetch_pairs = [&](decltype(&glio_batch_pose_pair_list) list, BatchEval& be) {
    int64_t np = 0;
    if (list(ctx, 0, nullptr, nullptr, &np) != GLIO_OK) return false;
    be.a.resize(np); be.b.resize(np);
    return list(ctx, np, be.a.data(), be.b.data(), &np) == GLIO_OK;
  };
  if (PB > 0) {
    if (glio_batch_clear(ctx) != GLIO_OK) return fail("glio_batch_clear");
    batch.push_back(BatchEval{glio_eval_binary, KB, {}, {}, 6});
    for (int p = 0; p < PB; ++p) {
      if (glio_batch_set_pair_matches(ctx, bpairs[p].kc, bpairs[p].ko, bpairs[p].cp.data(), bpairs[p].nc.data(), bpairs[p].w.data(), (int64_t)bpairs[p].w.size()) != GLIO_OK)
        return fail("glio_batch_set_pair_matches");
      batch.back().a.push_back(bpairs[p].kc); batch.back().b.push_back(bpairs[p].ko);
      S.num_device_residual_blocks += (int)bpairs[p].w.size();
    }
  }
  for (int k = 0; k < W; ++k) {
    if (glio_set_matches(ctx, k, slots[k].cp.data(), slots[k].nsd.data(), slots[k].w.data(), (int64_t)slots[k].w.size()) != GLIO_OK)
      return fail("glio_set_matches");
    S.num_device_residual_blocks += (int)slots[k].w.size();
  }
  // edges: every slot's list is replaced (an empty one where the slot has no edge), so lists and selections that an earlier
  // Solve or a direct caller left in the context are never evaluated.  A problem without routed edges makes no edge call at all.
  const bool with_edges = n_edge_dev > 0;
  if (with_edges) {
    for (int k = 0; k < W; ++k) {
      const Slot& sl = slots[k];
      if (glio_set_edges(ctx, k, sl.ecp.data(), sl.epa.data(), sl.epb.data(), sl.es.data(), (int64_t)sl.es.size()) != GLIO_OK)
        return fail("glio_set_edges");
    }
    S.num_device_residual_blocks += n_edge_dev; S.num_device_edge_residual_blocks = n_edge_dev;
  }
  // pose factors: the context's list is replaced after glio_batch_clear (which empties it) and the pair uploads.  A problem
  // without routed pose blocks makes no pose call at all.  glio_eval_binary never adds pose blocks, so glio_batch_use_pose_factors
  // does not change what is computed here.
  if (NP > 0) {
    if (glio_batch_set_pose_factors(ctx, pose_list.data(), NP) != GLIO_OK) return fail("glio_batch_set_pose_factors");
    batch.push_back(BatchEval{glio_eval_pose_factors, KT, {}, {}, 6});
    if (!fetch_pairs(glio_batch_pose_pair_list, batch.back())) return fail("glio_batch_pose_pair_list");
    S.num_device_residual_blocks += NP; S.num_device_pose_residual_blocks = NP;
  }
  // DD factors: the context's list is replaced after the clear, pair and pose uploads.  A problem without routed DD blocks makes
  // no DD call.  glio_eval_binary and glio_eval_pose_factors never add DD blocks, so glio_batch_use_dd_psr_factors does not change
  // what is computed here.  K2g fills only the t columns; restricting it to them keeps its pairs off q columns outside the band.
  if (ND > 0) {
    if (glio_batch_set_dd_psr_factors(ctx, dd_list.data(), ND, dd_sats.data(), (int64_t)dd_sats.size(), dd_W.empty() ? nullptr : dd_W.data(),
                                      (int64_t)dd_W.size(), dd_R, dd_anchor) != GLIO_OK)
      return fail("glio_batch_set_dd_psr_factors");
    batch.push_back(BatchEval{glio_eval_dd_psr_factors, KT, {}, {}, 3});
    if (!fetch_pairs(glio_batch_dd_psr_pair_list, batch.back())) return fail("glio_batch_dd_psr_pair_list");
    S.num_device_residual_blocks += ND; S.num_device_dd_psr_residual_blocks = ND;
  }
  // IMU factors: the context's list is replaced after the clear, pair, pose and DD uploads.  A problem without routed IMU blocks
  // makes no IMU call.  K2i's blocks are 15 x 15 over [t, delta, v, ba, bg]; no other glio_eval_* call adds them, so
  // glio_batch_use_imu_factors does not change what is computed here.
  BatchEval imu{nullptr, KT, {}, {}, 15};
  if (NI > 0) {
    if (glio_batch_set_imu_factors(ctx, imu_list.data(), NI) != GLIO_OK) return fail("glio_batch_set_imu_factors");
    if (!fetch_pairs(glio_batch_imu_pair_list, imu)) return fail("glio_batch_imu_pair_list");
    S.num_device_residual_blocks += NI; S.num_device_imu_residual_blocks = NI;
  }

  // ---- band of J^T J from the block structure ----
  int hb = 0;
  for (auto& rbp : problem->residual_blocks_) {
    int lo = n, hi = -1;
    for (double* p : rbp->params) { auto it = P.index.find(p); if (it == P.index.end()) continue; const ActiveBlock& a = P.active[it->second]; lo = std::min(lo, a.tan_off); hi = std::max(hi, a.tan_off + a.local - 1); }
    if (hi >= 0) hb = std::max(hb, hi - lo);
  }

  // ---- solver setup ----
  std::vector<glio::ParamBlock> blocks;
  for (const ActiveBlock& a : P.active) {
    glio::ParamBlock b{a.amb_off, a.size, a.tan_off, a.local, false, nullptr};
    if (a.param) { LocalParameterization* lp = a.param; b.plus_fn = [lp](const double* x, const double* d, double* o) { lp->Plus(x, d, o); }; }
    blocks.push_back(b);
  }
  glio::SolverOptions so;
  so.max_num_iterations = options.max_num_iterations;
  so.max_solver_time_in_seconds = options.max_solver_time_in_seconds;
  so.dogleg_type = options.dogleg_type == SUBSPACE_DOGLEG ? 1 : 0;
  so.use_nonmonotonic_steps = options.use_nonmonotonic_steps;
  so.max_consecutive_nonmonotonic_steps = options.max_consecutive_nonmonotonic_steps;
  so.initial_trust_region_radius = options.initial_trust_region_radius; so.max_trust_region_radius = options.max_trust_region_radius;
  so.min_trust_region_radius = options.min_trust_region_radius; so.min_relative_decrease = options.min_relative_decrease;
  so.min_lm_diagonal = options.min_lm_diagonal; so.max_lm_diagonal = options.max_lm_diagonal;
  so.max_num_consecutive_invalid_steps = options.max_num_consecutive_invalid_steps; so.jacobi_scaling = options.jacobi_scaling;
  so.function_tolerance = options.function_tolerance; so.gradient_tolerance = options.gradient_tolerance; so.parameter_tolerance = options.parameter_tolerance;
  // LEVENBERG_MARQUARDT is Ceres' default and what the front end's scan matcher runs (LidarOdometry.cpp:521-530); DOGLEG is
  // what the Estimator selects (Estimator.cpp:2427, :3278).  Both are implemented by the host minimizer.
  so.trust_region_strategy = options.trust_region_strategy_type == LEVENBERG_MARQUARDT ? 1 : 0;
  glio::TrustRegionDogleg solver(blocks, so);

  std::vector<double> x(P.n_amb);
  for (const ActiveBlock& a : P.active) std::memcpy(&x[a.amb_off], a.user, sizeof(double) * a.size);
  std::vector<double> poses((size_t)std::max(W, 1) * 7), Hd((size_t)std::max(W, 1) * 36), gd((size_t)std::max(W, 1) * 6), cd(std::max(W, 1));
  std::vector<double> He(with_edges ? Hd.size() : 0), ge(with_edges ? gd.size() : 0), ce(with_edges ? cd.size() : 0);
  size_t max_pairs = 1;
  for (const BatchEval& be : batch) max_pairs = std::max(max_pairs, be.a.size());
  std::vector<double> bposes((size_t)std::max(KT, 1) * 7), bHd((size_t)std::max(KT, 1) * 36), bHo(max_pairs * 36), bg((size_t)std::max(KT, 1) * 6);
  // K2i's inputs and outputs, allocated once per solve: speed-bias states (zeros for a keyframe without an sb, which no IMU factor
  // references), K x 225, P_imu x 225 and K x 15
  std::vector<double> bsb(NI > 0 ? (size_t)KT * 9 : 0), iHd(NI > 0 ? (size_t)KT * 225 : 0), iHo(imu.a.size() * 225), ig(NI > 0 ? (size_t)KT * 15 : 0);
  // tangent column of each unary slot's and each batch keyframe's 6-vector entries (t, then the rotation's delta); -1 for the
  // entries of a keyframe without a t (seen only in delta_q blocks) or without a q (seen only in DD blocks)
  auto cols_of = [&](double* t, double* q, std::vector<int>& col) {
    for (int p = 0; p < 6; ++p) { double* u = p < 3 ? t : q; col.push_back(u ? P.active[P.index[u]].tan_off + p % 3 : -1); }
  };
  std::vector<int> ucol, bcol;
  for (const Slot& sl : slots) cols_of(sl.t, sl.q, ucol);
  for (const auto& kf : bkfs) cols_of(kf.first, kf.second, bcol);
  // K2i's 15 entries per batch keyframe: [t(3), delta(3)] as above, then its sb's v(3), ba(3), bg(3)
  std::vector<int> icol;
  if (NI > 0)
    for (int k = 0; k < KT; ++k) {
      icol.insert(icol.end(), bcol.begin() + 6 * k, bcol.begin() + 6 * k + 6);
      for (int p = 0; p < 9; ++p) icol.push_back(bkf_sb[k] ? P.active[P.index[bkf_sb[k]]].tan_off + p : -1);
    }
  double fixed_cost = 0; bool fixed_done = false;

  glio::EvalFn eval = [&](const double* xa, bool want_jac, double* cost, glio::BandMat* H, double* g) -> bool {
    double ct = 0;
    if (want_jac) { H->reset(n, hb); std::fill(g, g + n, 0.0); }
    // adds K keyframes' Hdiag (K x st^2) and g (K x st), then np Hoff blocks (block i: row = keyframe a[i], col = keyframe b[i],
    // st x st) to the band's lower triangle, over the first nc of each keyframe's st entries (st = 6, or 15 for K2i); entries
    // without a column are skipped
    auto scatter = [&](const int* col, int st, int K, int nc, const double* Hk, const double* gk, int np, const int32_t* a, const int32_t* b,
                       const double* Ho) {
      for (int k = 0; k < K; ++k)
        for (int p = 0; p < nc; ++p) {
          const int ip = col[st * k + p];
          if (ip < 0) continue;
          g[ip] += gk[st * k + p];
          for (int q = 0; q < nc; ++q) { const int iq = col[st * k + q]; if (iq >= 0 && ip >= iq) H->at(ip, iq) += Hk[(size_t)st * st * k + st * p + q]; }
        }
      for (int pr = 0; pr < np; ++pr)
        for (int p = 0; p < nc; ++p) for (int q = 0; q < nc; ++q) {
          const int ip = col[st * a[pr] + p], iq = col[st * b[pr] + q];
          if (ip < 0 || iq < 0) continue;
          const double v = Ho[(size_t)st * st * pr + st * p + q];
          if (ip >= iq) H->at(ip, iq) += v; else H->at(iq, ip) += v;
        }
    };
    // device blocks
    if (W > 0) {
      for (int k = 0; k < W; ++k) {
        const ActiveBlock& at = P.active[P.index[slots[k].t]]; const ActiveBlock& aq = P.active[P.index[slots[k].q]];
        for (int i = 0; i < 3; ++i) poses[7 * k + i] = xa[at.amb_off + i];
        for (int i = 0; i < 4; ++i) poses[7 * k + 3 + i] = xa[aq.amb_off + i];
      }
      if (glio_eval_unary(ctx, W, poses.data(), 0, want_jac ? Hd.data() : nullptr, want_jac ? gd.data() : nullptr, cd.data()) != GLIO_OK) return false;
      if (with_edges) {                      // each keyframe's edge blocks join its plane blocks, as in glio_window_solve
        if (glio_eval_edge(ctx, W, poses.data(), want_jac ? He.data() : nullptr, want_jac ? ge.data() : nullptr, ce.data()) != GLIO_OK) return false;
        for (int k = 0; k < W; ++k) cd[k] += ce[k];
        if (want_jac) {
          for (size_t i = 0; i < (size_t)W * 36; ++i) Hd[i] += He[i];
          for (size_t i = 0; i < (size_t)W * 6; ++i) gd[i] += ge[i];
        }
      }
      for (int k = 0; k < W; ++k) ct += cd[k];
      if (want_jac) scatter(ucol.data(), 6, W, 6, Hd.data(), gd.data(), 0, nullptr, nullptr, nullptr);
    }
    if (!batch.empty() || NI > 0)
      for (int k = 0; k < KT; ++k) {
        for (int i = 0; i < 3; ++i) bposes[7 * k + i] = bkfs[k].first ? xa[P.active[P.index[bkfs[k].first]].amb_off + i] : 0.0;
        if (!bkfs[k].second) { bposes[7 * k + 3] = 1.0; bposes[7 * k + 4] = bposes[7 * k + 5] = bposes[7 * k + 6] = 0.0; continue; }
        const ActiveBlock& aq = P.active[P.index[bkfs[k].second]];
        for (int i = 0; i < 4; ++i) bposes[7 * k + 3 + i] = xa[aq.amb_off + i];
      }
    for (const BatchEval& be : batch) {
      double bc = 0;
      if (be.fn(ctx, be.K, bposes.data(), want_jac ? bHd.data() : nullptr, want_jac ? bHo.data() : nullptr, want_jac ? bg.data() : nullptr, &bc) != GLIO_OK) return false;
      ct += bc;
      if (want_jac) scatter(bcol.data(), 6, be.K, be.nc, bHd.data(), bg.data(), (int)be.a.size(), be.a.data(), be.b.data(), bHo.data());
    }
    // K2i after K2b, K2p and K2g, the order glio_batch_solve adds them in
    if (NI > 0) {
      for (int k = 0; k < KT; ++k)
        for (int i = 0; i < 9; ++i) bsb[9 * k + i] = bkf_sb[k] ? xa[P.active[P.index[bkf_sb[k]]].amb_off + i] : 0.0;
      double ic = 0;
      if (glio_eval_imu_factors(ctx, KT, bposes.data(), bsb.data(), want_jac ? iHd.data() : nullptr, want_jac ? iHo.data() : nullptr,
                                want_jac ? ig.data() : nullptr, &ic) != GLIO_OK)
        return false;
      ct += ic;
      if (want_jac) scatter(icol.data(), 15, KT, 15, iHd.data(), ig.data(), (int)imu.a.size(), imu.a.data(), imu.b.data(), iHo.data());
    }
    // host blocks (ResidualBlock::Evaluate, ceres.tgz::internal/ceres/residual_block.cc:70-197)
    std::vector<const double*> pp; std::vector<double*> jj; std::vector<std::vector<double>> Jamb, Jloc; std::vector<double> r;
    double fc = 0;
    for (const Problem::Residual* rb : host_blocks) {
      const int nb = (int)rb->params.size(), nr = rb->cost->num_residuals();
      const std::vector<int32_t>& sz = rb->cost->parameter_block_sizes();
      pp.assign(nb, nullptr); jj.assign(nb, nullptr); Jamb.resize(nb); Jloc.resize(nb); r.assign(nr, 0.0);
      bool any_active = false;
      for (int b = 0; b < nb; ++b) {
        auto it = P.index.find(rb->params[b]);
        if (it != P.index.end()) { pp[b] = xa + P.active[it->second].amb_off; any_active = true; if (want_jac) { Jamb[b].assign((size_t)nr * sz[b], 0.0); jj[b] = Jamb[b].data(); } }
        else pp[b] = rb->params[b];
      }
      if (!any_active && fixed_done) continue;           // all-constant block: part of the fixed cost, evaluated once
      if (!rb->cost->Evaluate(pp.data(), r.data(), want_jac && any_active ? jj.data() : nullptr)) return false;
      double sq = 0; for (int k = 0; k < nr; ++k) sq += r[k] * r[k];
      double rho[3] = {sq, 1.0, 0.0};
      if (rb->loss) rb->loss->Evaluate(sq, rho);
      if (!any_active) { fc += 0.5 * rho[0]; continue; }
      ct += 0.5 * rho[0];
      if (!want_jac) continue;
      for (int b = 0; b < nb; ++b) {
        if (!jj[b]) continue;
        const ActiveBlock& a = P.active[P.index[rb->params[b]]];
        if (a.param) {
          std::vector<double> Pm((size_t)a.size * a.local);
          a.param->ComputeJacobian(pp[b], Pm.data());
          Jloc[b].assign((size_t)nr * a.local, 0.0);
          for (int k = 0; k < nr; ++k) for (int c = 0; c < a.local; ++c) { double s = 0; for (int m = 0; m < a.size; ++m) s += Jamb[b][(size_t)k * a.size + m] * Pm[(size_t)m * a.local + c]; Jloc[b][(size_t)k * a.local + c] = s; }
        } else Jloc[b] = Jamb[b];
      }
      if (rb->loss) {
        Corr corr(sq, rho);
        for (int b = 0; b < nb; ++b) if (jj[b]) corr.jac(nr, P.active[P.index[rb->params[b]]].local, r.data(), Jloc[b].data());
        for (int k = 0; k < nr; ++k) r[k] *= corr.residual_scaling;
      }
      for (int a_ = 0; a_ < nb; ++a_) {
        if (!jj[a_]) continue;
        const ActiveBlock& A = P.active[P.index[rb->params[a_]]];
        for (int i = 0; i < A.local; ++i) {
          double gi = 0; for (int k = 0; k < nr; ++k) gi += Jloc[a_][(size_t)k * A.local + i] * r[k];
          g[A.tan_off + i] += gi;
        }
        for (int b_ = 0; b_ < nb; ++b_) {
          if (!jj[b_]) continue;
          const ActiveBlock& B = P.active[P.index[rb->params[b_]]];
          for (int i = 0; i < A.local; ++i) for (int j = 0; j < B.local; ++j) {
            const int ri = A.tan_off + i, cj = B.tan_off + j;
            if (ri < cj) continue;
            double h = 0; for (int k = 0; k < nr; ++k) h += Jloc[a_][(size_t)k * A.local + i] * Jloc[b_][(size_t)k * B.local + j];
            H->at(ri, cj) += h;
          }
        }
      }
    }
    if (!fixed_done) { fixed_cost = fc; fixed_done = true; }
    *cost = ct;
    return std::isfinite(ct);
  };

  glio::SolverSummary gs;
  solver.solve(x.data(), eval, &gs);
  for (const ActiveBlock& a : P.active) std::memcpy(a.user, &x[a.amb_off], sizeof(double) * a.size);
  S.termination_type = gs.termination == glio::TERM_CONVERGENCE ? CONVERGENCE : gs.termination == glio::TERM_NO_CONVERGENCE ? NO_CONVERGENCE : FAILURE;
  S.message += gs.message;
  S.fixed_cost = fixed_cost;
  S.initial_cost = gs.initial_cost + fixed_cost; S.final_cost = gs.final_cost + fixed_cost;
  S.num_successful_steps = gs.num_successful_steps; S.num_unsuccessful_steps = gs.num_unsuccessful_steps;
  for (const glio::IterationRecord& r : gs.iterations) {
    IterationSummary it; it.iteration = r.iteration; it.step_is_valid = r.step_is_valid != 0; it.step_is_successful = r.step_is_successful != 0;
    it.cost = r.cost + fixed_cost; it.cost_change = r.cost_change; it.gradient_max_norm = r.gradient_max_norm; it.gradient_norm = r.gradient_norm;
    it.step_norm = r.step_norm; it.relative_decrease = r.relative_decrease; it.trust_region_radius = r.trust_region_radius;
    S.iterations.push_back(it);
  }
  S.total_time_in_seconds = std::chrono::duration<double>(std::chrono::steady_clock::now() - t_start).count();
  if (options.minimizer_progress_to_stdout)
    for (const IterationSummary& it : S.iterations) printf("iter %3d cost %.6e |grad| %.3e radius %.3e %s\n", it.iteration, it.cost, it.gradient_max_norm, it.trust_region_radius, it.step_is_successful ? "" : "(rejected)");
}

inline bool Problem::Evaluate(const EvaluateOptions& eo, double* cost, std::vector<double>* residuals, std::vector<double>* gradient, void*) {
  // host evaluation of every residual block at the current user state (no device routing: this is the slow, exact path
  // the reference never calls; kept for API completeness)
  double ct = 0;
  if (residuals) residuals->clear();
  std::map<double*, int> toff; int nt = 0;
  // every parameter block of the problem owns its columns, constant ones with a zero gradient (Ceres: problem_test.cc:1363-1394)
  for (double* u : order_) { const Block& b = blocks_.at(u); toff[u] = nt; nt += b.param ? b.param->LocalSize() : b.size; }
  if (gradient) gradient->assign(nt, 0.0);
  for (auto& rb : residual_blocks_) {
    const int nb = (int)rb->params.size(), nr = rb->cost->num_residuals();
    const std::vector<int32_t>& sz = rb->cost->parameter_block_sizes();
    std::vector<const double*> pp(rb->params.begin(), rb->params.end());
    std::vector<std::vector<double>> J(nb); std::vector<double*> jj(nb, nullptr); std::vector<double> r(nr);
    if (gradient) for (int b = 0; b < nb; ++b) if (toff.count(rb->params[b]) && !blocks_.at(rb->params[b]).constant) { J[b].assign((size_t)nr * sz[b], 0.0); jj[b] = J[b].data(); }
    if (!rb->cost->Evaluate(pp.data(), r.data(), gradient ? jj.data() : nullptr)) return false;
    double sq = 0; for (double v : r) sq += v * v;
    double rho[3] = {sq, 1.0, 0.0};
    if (rb->loss && eo.apply_loss_function) rb->loss->Evaluate(sq, rho);
    ct += 0.5 * rho[0];
    if (residuals) { shim_internal::Corr c(sq, rho); for (double v : r) residuals->push_back(v * c.residual_scaling); }
    if (gradient) for (int b = 0; b < nb; ++b) {
      if (!jj[b]) continue;
      const Block& blk = blocks_.at(rb->params[b]);
      const int loc = blk.param ? blk.param->LocalSize() : blk.size;
      std::vector<double> Pm;
      if (blk.param) { Pm.resize((size_t)blk.size * loc); blk.param->ComputeJacobian(rb->params[b], Pm.data()); }
      for (int c = 0; c < loc; ++c) {
        double s = 0;
        for (int k = 0; k < nr; ++k) {
          double jl = 0;
          if (blk.param) for (int m = 0; m < blk.size; ++m) jl += J[b][(size_t)k * blk.size + m] * Pm[(size_t)m * loc + c]; else jl = J[b][(size_t)k * blk.size + c];
          s += jl * r[k] * rho[1];
        }
        (*gradient)[toff[rb->params[b]] + c] += s;
      }
    }
  }
  if (cost) *cost = ct;
  return true;
}

}  // namespace ceres
#endif  // GLIO_SHIM_CERES_SHIM_SOLVE_H_
