// assoc.cu — K1 / K1b: per-point LiDAR surf association on a uniform grid.
//
// Replaces Estimator::findCorrespondingSurfFeatures (GLIO/src/Estimator.cpp:3633-3708) and
// findGlobalCorrespondingSurfFeatures[Add]_Batch (Estimator.cpp:3710-3892):
//   transform -> exact 5-NN (FLANN L2_Simple<float> distances, ties by index) -> gate on the squared 5th
//   distance -> 5x3 column-pivoted Householder LS plane fit (double) -> validity -> weight -> outputs.
// Exactness of the kNN: a box of grid cells around the query is searched and grown face by face (k_knn_box) until
// the 5th best distance is provably inside the searched box, or the box already covers the gate radius (then anything
// unseen fails the gate anyway).
//
// This translation unit is compiled with -fmad=false (see Makefile) in addition to the explicit *_rn
// intrinsics of devmath.cuh: kNN indices and the valid mask must be bit-exact w.r.t. the no-FMA reference.
#include "common.cuh"
#include "devmath.cuh"
#include "knn_common.cuh"

namespace glio {

__device__ __forceinline__ int find_seg(const SegDesc* __restrict__ segs, int nseg, int64_t g) {
  int lo = 0, hi = nseg - 1;
  while (lo < hi) {
    int mid = (lo + hi + 1) >> 1;
    if (segs[mid].offset <= g) lo = mid; else hi = mid - 1;
  }
  return lo;
}

// ---- pass 1: transform queries, histogram them by (clamped) grid cell --------------------------------
__global__ void __launch_bounds__(256) k_transform_hist(GridDesc grid, const SegDesc* __restrict__ segs, int nseg,
                                                        int64_t Qt, float4* __restrict__ pm, uint16_t* __restrict__ segid,
                                                        int* __restrict__ cell_count) {
  const int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= Qt) return;
  const int s = find_seg(segs, nseg, g);
  const SegDesc& sd = segs[s];
  const float* src = sd.src + (g - sd.offset) * sd.stride;
  float p[3] = {src[0], src[1], src[2]};
  PoseD P;
  P.t[0] = sd.t[0]; P.t[1] = sd.t[1]; P.t[2] = sd.t[2];
  P.q[0] = sd.q[0]; P.q[1] = sd.q[1]; P.q[2] = sd.q[2]; P.q[3] = sd.q[3];
  transform_point_f(P, p, p);
  pm[g] = make_float4(p[0], p[1], p[2], 0.f);
  segid[g] = (uint16_t)s;
  atomicAdd(&cell_count[cell_of_clamped(grid, p[0], p[1], p[2])], 1);
}

// ---- pass 2: scatter the queries into cell order (locality: a warp's queries share grid cells) -------
__global__ void __launch_bounds__(256) k_order_scatter(GridDesc grid, int64_t Qt, const float4* __restrict__ pm,
                                                       const int* __restrict__ cell_start, int* __restrict__ fill,
                                                       float4* __restrict__ pmq) {
  const int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= Qt) return;
  const float4 p = pm[g];
  const int c = cell_of_clamped(grid, p.x, p.y, p.z);
  const int pos = cell_start[c] + atomicAdd(&fill[c], 1);
  pmq[pos] = make_float4(p.x, p.y, p.z, __int_as_float((int)g));   // the query itself travels in cell order with its scan index:
                                                                     // K1a and K1b read it coalesced, one scattered store per query
}

// ---------------------------------------------------------------------------------------------------
// K1a (box growth): one query per thread; each (y,z) row of cells is one contiguous range of the sorted map, and the
// queries arrive cell-sorted, so the loads of neighbouring threads hit the same lines.  The searched box of a query
// grows one FACE at a time instead of one ring at a time.  After the start box (3x3x3 cells around the query) a face
// is pushed out by one cell layer only if something nearer than the current 5th distance could still hide behind it:
// the face is not at the grid border, not farther than the gate radius, and closer to the query than the 5th distance.
// A query near one cell wall with a 5th neighbour a little beyond it scans one extra slab of 9 cells instead of the 98
// cells of a full second ring; the top-5 is exact (every unscanned point lies beyond some face, all faces are at least
// the 5th distance away), faces are re-tested with the freshest 5th distance.
// ---------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(128, 6) k_knn_box(SearchArgs a) {
  __shared__ int sbnd[18 * 128];
  const int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= a.Qt) return;
  const GridDesc& g = a.grid;
  const float4 q4 = a.pmq[p];
  const float qx = q4.x, qy = q4.y, qz = q4.z;
  Top5 t; top5_init(t);
  const int cx = cell_coord(qx, g.ox, g.inv_cell), cy = cell_coord(qy, g.oy, g.inv_cell), cz = cell_coord(qz, g.oz, g.inv_cell);
  const float gate_r = sqrtf(a.gate_sq) + g.slack;
  const int rmax = (int)ceilf(gate_r * g.inv_cell) + 1;
  const bool far_out = cx < -rmax || cy < -rmax || cz < -rmax || cx >= g.nx + rmax || cy >= g.ny + rmax || cz >= g.nz + rmax;
  float d4f = __int_as_float(0x7f800000);
  if (!far_out) {
    scan_start_box(g, qx, qy, qz, cx, cy, cz, t, d4f, sbnd + threadIdx.x);
    box_grow(g, qx, qy, qz, gate_r, rmax, cx - 1, cx + 1, cy - 1, cy + 1, cz - 1, cz + 1, t, d4f, sbnd + threadIdx.x);
  }
  store_top5(a, p, t);
}

// ---------------------------------------------------------------------------------------------------
// K1b: gate -> plane fit (fp64 column-pivoted Householder QR) -> validity -> weight -> outputs.
// One thread per query, in sorted order (neighbour gathers of adjacent threads hit the same lines).
// ---------------------------------------------------------------------------------------------------
struct FitArgs {
  int64_t Qt;
  const float4* pm;
  const float4* pmq;          // queries in cell-sorted order, .w = scan index
  const int32_t* knn_idx;
  const float* knn_sqd;
  AssocGates gates;
  const float4* pts_sorted;   // searched cloud, cell-sorted (x,y,z,idx): neighbouring queries gather neighbouring lines
  const int* sorted_pos;      // original index -> position in pts_sorted (4 B per point: stays in L2)
  const float* oth_local;     // pair mode: local-frame points of the searched frame (original order)
  int oth_stride;
  uint8_t* status;
  float4* nsd;
  float* weight;
  double* normal_cent;
  int32_t* idx5;
  float* sqd5;
  double* plane;
};

template <bool PAIR>
__global__ void __launch_bounds__(128, 5) k_plane_fit(FitArgs a) {
  const int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= a.Qt) return;
  const float4 q4 = a.pmq[p];
  const int64_t g = __float_as_int(q4.w);
  int id[5];
#pragma unroll
  for (int j = 0; j < 5; ++j) id[j] = a.knn_idx[(int64_t)j * a.Qt + p];
  const float d4 = a.knn_sqd[4 * a.Qt + p];
  uint8_t st;
  float w = 0.f;
  double n[3] = {0, 0, 0}, d = 0;
  double nl[3] = {0, 0, 0}, cl[3] = {0, 0, 0};
  if (id[4] != 0x7fffffff && (double)d4 < a.gates.max_radius) {           // Estimator.cpp:3651 / :3751
    // the five neighbours are gathered twice (for the fit, and again for the validity test: L1/L2 hits) so that the 15 doubles
    // are not live across the QR: ~30 registers less, one more resident block per SM
    int pos[5];
#pragma unroll
    for (int j = 0; j < 5; ++j) pos[j] = __ldg(&a.sorted_pos[id[j]]);
    double Aw[3][5];
#pragma unroll
    for (int j = 0; j < 5; ++j) {
      const float4 m = __ldg(&a.pts_sorted[pos[j]]);
      Aw[0][j] = (double)m.x; Aw[1][j] = (double)m.y; Aw[2][j] = (double)m.z;
    }
    double x[3];
    plane_solve5(Aw, x);                                                    // :3661
    plane_from_solution(x, n, d);                                           // :3662-3663
    bool ok = true;
#pragma unroll
    for (int j = 0; j < 5; ++j) {                                           // :3667-3674
      const float4 m = __ldg(&a.pts_sorted[pos[j]]);
      const double v = dadd(dadd(dadd(dmul(n[0], (double)m.x), dmul(n[1], (double)m.y)), dmul(n[2], (double)m.z)), d);
      if (fabs(v) > a.gates.dist_thres) ok = false;
    }
    if (ok) {
      w = weight_of(n, d, q4.x, q4.y, q4.z);                                // :3678-3679
      st = ((double)w > a.gates.weight_min) ? GLIO_MATCH_VALID : GLIO_MATCH_FAIL_WEIGHT;  // :3681
    } else st = GLIO_MATCH_FAIL_PLANE;
    if (PAIR && st == GLIO_MATCH_VALID) {
      // local-frame fit on the same five indices (Estimator.cpp:3752-3772)
      double Al[3][5];
      double sx = 0.0, sy = 0.0, sz = 0.0;
#pragma unroll
      for (int j = 0; j < 5; ++j) {
        const float* lp = a.oth_local + (int64_t)id[j] * a.oth_stride;
        Al[0][j] = (double)lp[0]; Al[1][j] = (double)lp[1]; Al[2][j] = (double)lp[2];
        sx = dadd(sx, Al[0][j]); sy = dadd(sy, Al[1][j]); sz = dadd(sz, Al[2][j]);
      }
      cl[0] = sx / 5.0; cl[1] = sy / 5.0; cl[2] = sz / 5.0;
      double xl[3], dl;
      plane_solve5(Al, xl);
      plane_from_solution(xl, nl, dl);
    }
  } else st = GLIO_MATCH_FAIL_RADIUS;

  a.status[g] = st;
  if (!PAIR) {
    float4 o = make_float4(0.f, 0.f, 0.f, 0.f);
    if (st == GLIO_MATCH_VALID) {                                            // :3683-3687 float stores
      o.x = (float)dmul((double)w, n[0]); o.y = (float)dmul((double)w, n[1]);
      o.z = (float)dmul((double)w, n[2]); o.w = (float)dmul((double)w, d);
    }
    a.nsd[g] = o;
  } else {
    double* nc = a.normal_cent + 6 * g;
    const bool v = st == GLIO_MATCH_VALID;
    nc[0] = v ? nl[0] : 0.0; nc[1] = v ? nl[1] : 0.0; nc[2] = v ? nl[2] : 0.0;
    nc[3] = v ? cl[0] : 0.0; nc[4] = v ? cl[1] : 0.0; nc[5] = v ? cl[2] : 0.0;
  }
  a.weight[g] = (st == GLIO_MATCH_VALID || st == GLIO_MATCH_FAIL_WEIGHT) ? w : 0.f;
  if (a.idx5) {
#pragma unroll
    for (int j = 0; j < 5; ++j) {
      a.idx5[5 * g + j] = (id[j] == 0x7fffffff) ? -1 : id[j];
      a.sqd5[5 * g + j] = a.knn_sqd[(int64_t)j * a.Qt + p];
    }
    a.plane[4 * g] = n[0]; a.plane[4 * g + 1] = n[1]; a.plane[4 * g + 2] = n[2]; a.plane[4 * g + 3] = d;
  }
}

// K1 front half, shared by the surf fit (assoc_run) and the line fit (edge_assoc_run): transform the queries, put them in cell
// order and find their exact 5 nearest neighbours within sqrt(gate_sq) of the grid's cloud.  Qt > 0.
static void assoc_search(const GridBuild& gb, const SegDesc* d_segs, int nseg, const AssocWork& w, float gate_sq, DevBuf<int>& cell_count,
                         DevBuf<int>& cell_pos, DevBuf<int>& scan_tmp, cudaStream_t st, LaunchCounter& lc) {
  const GridDesc& grid = gb.desc;
  const int64_t Qt = w.Qt;
  GLIO_REQUIRE(Qt < ((int64_t)1 << 31), GLIO_ERR_ARG, "assoc_run: too many queries in one launch");
  GLIO_REQUIRE(nseg > 0 && nseg < 65536, GLIO_ERR_ARG, "assoc_run: bad segment count");
  const int64_t ncell = (int64_t)grid.nx * grid.ny * grid.nz;
  cell_count.reserve((size_t)ncell + 2);
  cell_pos.reserve((size_t)ncell + 2);
  GLIO_CUDA_TRY(cudaMemsetAsync(cell_count.p, 0, (size_t)(ncell + 1) * sizeof(int), st));
  const unsigned nb = (unsigned)((Qt + 255) / 256);
  lc.begin("k_transform_hist", st); k_transform_hist<<<nb, 256, 0, st>>>(grid, d_segs, nseg, Qt, w.pm, w.seg, cell_count.p); lc.end(st);
  exclusive_scan_i32(cell_count.p, cell_pos.p, ncell + 1, scan_tmp, st, lc);
  GLIO_CUDA_TRY(cudaMemsetAsync(cell_count.p, 0, (size_t)(ncell + 1) * sizeof(int), st));
  lc.begin("k_order_scatter", st); k_order_scatter<<<nb, 256, 0, st>>>(grid, Qt, w.pm, cell_pos.p, cell_count.p, w.pmq); lc.end(st);
  SearchArgs sa;
  sa.grid = grid; sa.Qt = Qt; sa.pm = w.pm; sa.pmq = w.pmq; sa.gate_sq = gate_sq;
  sa.knn_idx = w.knn_idx; sa.knn_sqd = w.knn_sqd; sa.store_all_sqd = w.idx5 != nullptr;
  lc.begin("k_knn_box", st); k_knn_box<<<(unsigned)((Qt + 127) / 128), 128, 0, st>>>(sa); lc.end(st);
}

void assoc_run(const GridBuild& gb, const SegDesc* d_segs, int nseg, const AssocWork& w, const AssocGates& gates,
               const float* oth_local, int oth_stride, DevBuf<int>& cell_count, DevBuf<int>& cell_pos,
               DevBuf<int>& scan_tmp, cudaStream_t st, LaunchCounter& lc) {
  const int64_t Qt = w.Qt;
  if (Qt <= 0) return;
  assoc_search(gb, d_segs, nseg, w, (float)gates.max_radius, cell_count, cell_pos, scan_tmp, st, lc);
  FitArgs fa;
  fa.Qt = Qt; fa.pm = w.pm; fa.pmq = w.pmq; fa.knn_idx = w.knn_idx; fa.knn_sqd = w.knn_sqd; fa.gates = gates;
  fa.pts_sorted = gb.pts.p; fa.sorted_pos = gb.sorted_pos.p; fa.oth_local = oth_local; fa.oth_stride = oth_stride;
  fa.status = w.status; fa.nsd = w.nsd; fa.weight = w.weight; fa.normal_cent = w.normal_cent;
  fa.idx5 = w.idx5; fa.sqd5 = w.sqd5; fa.plane = w.plane;
  const unsigned nk = (unsigned)((Qt + 127) / 128);
  lc.begin(w.normal_cent ? "k_plane_fit_pair" : "k_plane_fit", st);
  if (w.normal_cent) k_plane_fit<true><<<nk, 128, 0, st>>>(fa);
  else k_plane_fit<false><<<nk, 128, 0, st>>>(fa);
  lc.end(st);
  GLIO_CUDA_TRY(cudaGetLastError());
}

// ---- stream compaction of the valid matches, per segment, in scan order ------------------------------
__global__ void __launch_bounds__(256) k_flags(const uint8_t* __restrict__ status, int64_t Qt, int* __restrict__ flags) {
  const int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (g < Qt) flags[g] = status[g] == GLIO_MATCH_VALID ? 1 : 0;
  if (g == Qt) flags[g] = 0;
}

__global__ void __launch_bounds__(256) k_compact(const SegDesc* __restrict__ segs, int64_t Qt, const uint16_t* __restrict__ segid,
                                                 const uint8_t* __restrict__ status, const int* __restrict__ pos,
                                                 const float4* __restrict__ nsd, const float* __restrict__ weight,
                                                 const double* __restrict__ normal_cent, const CompactDst* __restrict__ dst) {
  const int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= Qt) return;
  if (status[g] != GLIO_MATCH_VALID) return;
  const int s = segid[g];
  const SegDesc& sd = segs[s];
  const int lp = pos[g] - pos[sd.offset];
  const int64_t li = g - sd.offset;
  const float* src = sd.src + li * sd.stride;
  const CompactDst d = dst[s];
  d.cpw[lp] = make_float4(src[0], src[1], src[2], weight[g]);
  if (d.nsd) d.nsd[lp] = nsd[g];
  if (d.nc) {
#pragma unroll
    for (int k = 0; k < 6; ++k) d.nc[6 * (int64_t)lp + k] = normal_cent[6 * g + k];
  }
  d.src[lp] = (int32_t)li;
}

__global__ void k_seg_counts(const SegDesc* __restrict__ segs, int nseg, const int* __restrict__ pos, int* __restrict__ counts) {
  const int s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s < nseg) counts[s] = pos[segs[s].offset + segs[s].count] - pos[segs[s].offset];
}

void compact_count(const AssocWork& w, const SegDesc* d_segs, int nseg, int* d_flags, int* d_pos, DevBuf<int>& scan_tmp,
                   int* d_counts, cudaStream_t st, LaunchCounter& lc) {
  const int64_t Qt = w.Qt;
  const unsigned nb = (unsigned)((Qt + 1 + 255) / 256);
  lc.begin("k_flags", st); k_flags<<<nb, 256, 0, st>>>(w.status, Qt, d_flags); lc.end(st);
  exclusive_scan_i32(d_flags, d_pos, Qt + 1, scan_tmp, st, lc);
  lc.begin("k_seg_counts", st); k_seg_counts<<<(nseg + 127) / 128, 128, 0, st>>>(d_segs, nseg, d_pos, d_counts); lc.end(st);
  GLIO_CUDA_TRY(cudaGetLastError());
}

void compact_scatter(const AssocWork& w, const SegDesc* d_segs, int nseg, const int* d_pos, const void* d_dst, cudaStream_t st,
                     LaunchCounter& lc) {
  const int64_t Qt = w.Qt;
  const unsigned nb = (unsigned)((Qt + 255) / 256);
  lc.begin("k_compact", st); k_compact<<<nb, 256, 0, st>>>(d_segs, Qt, w.seg, w.status, d_pos, w.nsd, w.weight, w.normal_cent, (const CompactDst*)d_dst); lc.end(st);
  GLIO_CUDA_TRY(cudaGetLastError());
}

void compact_run(const AssocWork& w, const SegDesc* d_segs, int nseg, int* d_flags, int* d_pos, DevBuf<int>& scan_tmp,
                 const void* d_dst /*CompactDst[nseg]*/, int* d_counts, cudaStream_t st, LaunchCounter& lc) {
  compact_count(w, d_segs, nseg, d_flags, d_pos, scan_tmp, d_counts, st, lc);
  compact_scatter(w, d_segs, nseg, d_pos, d_dst, st, lc);
}

// ---------------------------------------------------------------------------------------------------
// K1e: scan-to-map EDGE association (glio_window_associate_edges).  The reference has no edge association; the line form
// (curr_point, last_point_a, last_point_b, s) of LidarEdgeFactor is built here by the arithmetic include/glio_b200.h specifies,
// and tests/edge_reference.py restates it in Python doubles.  Every operation is an explicit round-to-nearest intrinsic and the
// file is compiled -fmad=false, so both agree bit for bit.  Queries, neighbours and the gate on the 5th squared distance come from
// the same K1 front half (assoc_search) as the surf path.
// ---------------------------------------------------------------------------------------------------
constexpr int EDGE_JACOBI_MAX_SWEEPS = 32;

__device__ __forceinline__ double ddiv_rn(double a, double b) { return __ddiv_rn(a, b); }

// One rotation of the cyclic Jacobi method zeroing a[p][q] of the symmetric 3x3 matrix a (both triangles kept), accumulated
// into the columns of v.  An off-diagonal element that no longer changes either diagonal element in double (|a_ii| + 100|a_pq|
// == |a_ii| for i = p and q) is set to zero without a rotation.
//   theta = (a_qq - a_pp) / (2 a_pq),  t = sgn(theta) / (|theta| + sqrt(theta^2 + 1))  (sgn(0) = +1),
//   c = 1 / sqrt(t^2 + 1),  s = t c,  a_pp -= t a_pq,  a_qq += t a_pq,  a_pq = 0,
//   r != p, q:  a_rp = c a_rp - s a_rq,  a_rq = s a_rp + c a_rq;   rows i of v:  v_ip = c v_ip - s v_iq,  v_iq = s v_ip + c v_iq
__device__ __forceinline__ void jacobi_rotate(double (&a)[3][3], double (&v)[3][3], const int p, const int q) {
  const double apq = a[p][q];
  if (apq == 0.0) return;
  const double g = dmul(100.0, fabs(apq));
  if (dadd(fabs(a[p][p]), g) == fabs(a[p][p]) && dadd(fabs(a[q][q]), g) == fabs(a[q][q])) { a[p][q] = 0.0; a[q][p] = 0.0; return; }
  const double theta = ddiv_rn(dsub(a[q][q], a[p][p]), dmul(2.0, apq));
  double t = ddiv_rn(1.0, dadd(fabs(theta), __dsqrt_rn(dadd(dmul(theta, theta), 1.0))));
  if (theta < 0.0) t = -t;
  const double c = ddiv_rn(1.0, __dsqrt_rn(dadd(dmul(t, t), 1.0)));
  const double s = dmul(t, c);
  const double tapq = dmul(t, apq);
  a[p][p] = dsub(a[p][p], tapq);
  a[q][q] = dadd(a[q][q], tapq);
  a[p][q] = 0.0; a[q][p] = 0.0;
  const int r = 3 - p - q;
  const double arp = a[r][p], arq = a[r][q];
  a[r][p] = a[p][r] = dsub(dmul(c, arp), dmul(s, arq));
  a[r][q] = a[q][r] = dadd(dmul(s, arp), dmul(c, arq));
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    const double vip = v[i][p], viq = v[i][q];
    v[i][p] = dsub(dmul(c, vip), dmul(s, viq));
    v[i][q] = dadd(dmul(s, vip), dmul(c, viq));
  }
}

// Eigen-decomposition of the symmetric 3x3 a: sweeps of the rotations (0,1), (0,2), (1,2) until all three off-diagonal
// elements are zero, at most EDGE_JACOBI_MAX_SWEEPS sweeps.  lam[0..2]: the diagonal sorted ascending, ties by index (a stable
// sort); dir: the column of v belonging to lam[2], signed so that its largest-magnitude component (lowest index on ties) is positive.
__device__ __forceinline__ void jacobi_eig3(double (&a)[3][3], double lam[3], double dir[3]) {
  double v[3][3] = {{1.0, 0.0, 0.0}, {0.0, 1.0, 0.0}, {0.0, 0.0, 1.0}};
#pragma unroll 1
  for (int sweep = 0; sweep < EDGE_JACOBI_MAX_SWEEPS; ++sweep) {
    if (a[0][1] == 0.0 && a[0][2] == 0.0 && a[1][2] == 0.0) break;
    jacobi_rotate(a, v, 0, 1);
    jacobi_rotate(a, v, 0, 2);
    jacobi_rotate(a, v, 1, 2);
  }
  // three compare-exchanges of adjacent (value, index) pairs, strict: a stable ascending sort (kept in registers)
  double l0 = a[0][0], l1 = a[1][1], l2 = a[2][2];
  int o0 = 0, o1 = 1, o2 = 2;
  if (l0 > l1) { const double t = l0; l0 = l1; l1 = t; const int i = o0; o0 = o1; o1 = i; }
  if (l1 > l2) { const double t = l1; l1 = l2; l2 = t; const int i = o1; o1 = o2; o2 = i; }
  if (l0 > l1) { const double t = l0; l0 = l1; l1 = t; const int i = o0; o0 = o1; o1 = i; }
  lam[0] = l0; lam[1] = l1; lam[2] = l2;
  dir[0] = o2 == 0 ? v[0][0] : (o2 == 1 ? v[0][1] : v[0][2]);
  dir[1] = o2 == 0 ? v[1][0] : (o2 == 1 ? v[1][1] : v[1][2]);
  dir[2] = o2 == 0 ? v[2][0] : (o2 == 1 ? v[2][1] : v[2][2]);
  double big = dir[0];
  if (fabs(dir[1]) > fabs(big)) big = dir[1];
  if (fabs(dir[2]) > fabs(big)) big = dir[2];
  if (big < 0.0) { dir[0] = -dir[0]; dir[1] = -dir[1]; dir[2] = -dir[2]; }
}

// steps 4-5 of the line fit: centroid c (summed nearest first, / 5.0) and the undivided scatter matrix A (both triangles) of the
// five points x[coordinate][neighbour].  The same operations in the same order as k_line_fit's inline copy, which is kept as it
// is so that its generated code does not change.
__device__ __forceinline__ void centroid_scatter5(const double (&x)[3][5], double c[3], double (&A)[3][3]) {
#pragma unroll
  for (int i = 0; i < 3; ++i) c[i] = ddiv_rn(dadd(dadd(dadd(dadd(x[i][0], x[i][1]), x[i][2]), x[i][3]), x[i][4]), 5.0);
#pragma unroll
  for (int i = 0; i < 3; ++i)
#pragma unroll
    for (int k = 0; k < 3; ++k) A[i][k] = 0.0;
#pragma unroll
  for (int j = 0; j < 5; ++j) {
    const double dx = dsub(x[0][j], c[0]), dy = dsub(x[1][j], c[1]), dz = dsub(x[2][j], c[2]);
    A[0][0] = dadd(A[0][0], dmul(dx, dx)); A[0][1] = dadd(A[0][1], dmul(dx, dy)); A[0][2] = dadd(A[0][2], dmul(dx, dz));
    A[1][1] = dadd(A[1][1], dmul(dy, dy)); A[1][2] = dadd(A[1][2], dmul(dy, dz)); A[2][2] = dadd(A[2][2], dmul(dz, dz));
  }
  A[1][0] = A[0][1]; A[2][0] = A[0][2]; A[2][1] = A[1][2];
}

struct LineFitArgs {
  int64_t Qt;
  const float4* pmq;          // queries in cell-sorted order, .w = scan index
  const int32_t* knn_idx;
  const float* knn_sqd;
  const float4* pts_sorted;   // the corner map, cell-sorted (x,y,z,idx)
  const int* sorted_pos;      // original index -> position in pts_sorted
  double max_sqdist, min_ratio, half_length;
  uint8_t* status;
  float4* pa;                 // per query (scan order): float(c + h v), float(c - h v)
  float4* pb;
  // debug (nullable)
  int32_t* idx5;
  float* sqd5;
  double* eig;                // 3 per query, ascending
};

// One thread per query, in sorted order.  Gate on the squared 5th distance -> centroid -> scatter matrix -> Jacobi -> line gate.
__global__ void __launch_bounds__(128) k_line_fit(LineFitArgs a) {
  const int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= a.Qt) return;
  const int64_t g = __float_as_int(a.pmq[p].w);
  int id[5];
#pragma unroll
  for (int j = 0; j < 5; ++j) id[j] = a.knn_idx[(int64_t)j * a.Qt + p];
  const float d4 = a.knn_sqd[4 * a.Qt + p];
  uint8_t st = GLIO_EDGE_FAIL_RADIUS;
  double lam[3] = {0.0, 0.0, 0.0};
  float4 oa = make_float4(0.f, 0.f, 0.f, 0.f), ob = oa;
  if (id[4] != 0x7fffffff && (double)d4 < a.max_sqdist) {
    double x[3][5];
#pragma unroll
    for (int j = 0; j < 5; ++j) {
      const float4 m = __ldg(&a.pts_sorted[__ldg(&a.sorted_pos[id[j]])]);
      x[0][j] = (double)m.x; x[1][j] = (double)m.y; x[2][j] = (double)m.z;
    }
    double c[3];
#pragma unroll
    for (int i = 0; i < 3; ++i) c[i] = ddiv_rn(dadd(dadd(dadd(dadd(x[i][0], x[i][1]), x[i][2]), x[i][3]), x[i][4]), 5.0);
    double A[3][3] = {{0.0, 0.0, 0.0}, {0.0, 0.0, 0.0}, {0.0, 0.0, 0.0}};
#pragma unroll
    for (int j = 0; j < 5; ++j) {
      const double dx = dsub(x[0][j], c[0]), dy = dsub(x[1][j], c[1]), dz = dsub(x[2][j], c[2]);
      A[0][0] = dadd(A[0][0], dmul(dx, dx)); A[0][1] = dadd(A[0][1], dmul(dx, dy)); A[0][2] = dadd(A[0][2], dmul(dx, dz));
      A[1][1] = dadd(A[1][1], dmul(dy, dy)); A[1][2] = dadd(A[1][2], dmul(dy, dz)); A[2][2] = dadd(A[2][2], dmul(dz, dz));
    }
    A[1][0] = A[0][1]; A[2][0] = A[0][2]; A[2][1] = A[1][2];
    double v[3];
    jacobi_eig3(A, lam, v);
    if (lam[2] > dmul(a.min_ratio, lam[1])) {
      st = GLIO_EDGE_VALID;
      const double h = a.half_length;
      oa = make_float4((float)dadd(c[0], dmul(h, v[0])), (float)dadd(c[1], dmul(h, v[1])), (float)dadd(c[2], dmul(h, v[2])), 0.f);
      ob = make_float4((float)dsub(c[0], dmul(h, v[0])), (float)dsub(c[1], dmul(h, v[1])), (float)dsub(c[2], dmul(h, v[2])), 0.f);
    } else st = GLIO_EDGE_FAIL_LINE;
  }
  a.status[g] = st;
  a.pa[g] = oa; a.pb[g] = ob;
  if (a.idx5) {
#pragma unroll
    for (int j = 0; j < 5; ++j) {
      a.idx5[5 * g + j] = (id[j] == 0x7fffffff) ? -1 : id[j];
      a.sqd5[5 * g + j] = a.knn_sqd[(int64_t)j * a.Qt + p];
    }
    a.eig[3 * g] = lam[0]; a.eig[3 * g + 1] = lam[1]; a.eig[3 * g + 2] = lam[2];
  }
}

// K1be, pair mode (glio_batch_associate_edges_pairs): the same gates on the world cloud of the searched frame; a valid query's line
// is then refitted (steps 4-6 again) on the same five indices in the searched frame's local coordinates as stored, as the pair plane
// fit refits its plane (Estimator.cpp:3752-3772), and pa / pb are that local line.  Debug views are not written.
__global__ void __launch_bounds__(128) k_line_fit_pair(LineFitArgs a, const float* __restrict__ oth_local, int oth_stride) {
  const int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= a.Qt) return;
  const int64_t g = __float_as_int(a.pmq[p].w);
  int id[5];
#pragma unroll
  for (int j = 0; j < 5; ++j) id[j] = a.knn_idx[(int64_t)j * a.Qt + p];
  const float d4 = a.knn_sqd[4 * a.Qt + p];
  uint8_t st = GLIO_EDGE_FAIL_RADIUS;
  float4 oa = make_float4(0.f, 0.f, 0.f, 0.f), ob = oa;
  if (id[4] != 0x7fffffff && (double)d4 < a.max_sqdist) {
    double x[3][5];
#pragma unroll
    for (int j = 0; j < 5; ++j) {
      const float4 m = __ldg(&a.pts_sorted[__ldg(&a.sorted_pos[id[j]])]);
      x[0][j] = (double)m.x; x[1][j] = (double)m.y; x[2][j] = (double)m.z;
    }
    double c[3], A[3][3], lam[3], v[3];
    centroid_scatter5(x, c, A);
    jacobi_eig3(A, lam, v);
    if (lam[2] > dmul(a.min_ratio, lam[1])) {
      st = GLIO_EDGE_VALID;
#pragma unroll
      for (int j = 0; j < 5; ++j) {
        const float* lp = oth_local + (int64_t)id[j] * oth_stride;
        x[0][j] = (double)lp[0]; x[1][j] = (double)lp[1]; x[2][j] = (double)lp[2];
      }
      centroid_scatter5(x, c, A);
      jacobi_eig3(A, lam, v);
      const double h = a.half_length;
      oa = make_float4((float)dadd(c[0], dmul(h, v[0])), (float)dadd(c[1], dmul(h, v[1])), (float)dadd(c[2], dmul(h, v[2])), 0.f);
      ob = make_float4((float)dsub(c[0], dmul(h, v[0])), (float)dsub(c[1], dmul(h, v[1])), (float)dsub(c[2], dmul(h, v[2])), 0.f);
    } else st = GLIO_EDGE_FAIL_LINE;
  }
  a.status[g] = st;
  a.pa[g] = oa; a.pb[g] = ob;
}

void edge_assoc_run(const GridBuild& gb, const SegDesc* d_segs, int nseg, const AssocWork& w, const EdgeFitParams& ep, float4* pa, float4* pb,
                    double* eig, const float* oth_local, int oth_stride, DevBuf<int>& cell_count, DevBuf<int>& cell_pos,
                    DevBuf<int>& scan_tmp, cudaStream_t st, LaunchCounter& lc) {
  const int64_t Qt = w.Qt;
  if (Qt <= 0) return;
  assoc_search(gb, d_segs, nseg, w, (float)ep.max_sqdist, cell_count, cell_pos, scan_tmp, st, lc);
  LineFitArgs la;
  la.Qt = Qt; la.pmq = w.pmq; la.knn_idx = w.knn_idx; la.knn_sqd = w.knn_sqd;
  la.pts_sorted = gb.pts.p; la.sorted_pos = gb.sorted_pos.p;
  la.max_sqdist = ep.max_sqdist; la.min_ratio = ep.min_ratio; la.half_length = ep.half_length;
  la.status = w.status; la.pa = pa; la.pb = pb; la.idx5 = w.idx5; la.sqd5 = w.sqd5; la.eig = eig;
  const unsigned nk = (unsigned)((Qt + 127) / 128);
  if (oth_local) { lc.begin("k_line_fit_pair", st); k_line_fit_pair<<<nk, 128, 0, st>>>(la, oth_local, oth_stride); lc.end(st); }
  else { lc.begin("k_line_fit", st); k_line_fit<<<nk, 128, 0, st>>>(la); lc.end(st); }
  GLIO_CUDA_TRY(cudaGetLastError());
}

// the valid edge records of every segment into its slot's buffers, in scan order (positions from compact_count)
__global__ void __launch_bounds__(256) k_compact_edge(const SegDesc* __restrict__ segs, int64_t Qt, const uint16_t* __restrict__ segid,
                                                      const uint8_t* __restrict__ status, const int* __restrict__ pos,
                                                      const float4* __restrict__ pa, const float4* __restrict__ pb, float score,
                                                      const EdgeDst* __restrict__ dst) {
  const int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= Qt) return;
  if (status[g] != GLIO_EDGE_VALID) return;
  const int s = segid[g];
  const SegDesc& sd = segs[s];
  const int lp = pos[g] - pos[sd.offset];
  const int64_t li = g - sd.offset;
  const float* src = sd.src + li * sd.stride;
  const EdgeDst d = dst[s];
  d.cps[lp] = make_float4(src[0], src[1], src[2], score);
  d.pa[lp] = pa[g];
  d.pb[lp] = pb[g];
  d.src[lp] = (int32_t)li;
}

void compact_edge_scatter(const AssocWork& w, const SegDesc* d_segs, const int* d_pos, const float4* pa, const float4* pb, float score,
                          const EdgeDst* d_dst, cudaStream_t st, LaunchCounter& lc) {
  const int64_t Qt = w.Qt;
  const unsigned nb = (unsigned)((Qt + 255) / 256);
  lc.begin("k_compact_edge", st); k_compact_edge<<<nb, 256, 0, st>>>(d_segs, Qt, w.seg, w.status, d_pos, pa, pb, score, d_dst); lc.end(st);
  GLIO_CUDA_TRY(cudaGetLastError());
}

// gather (feature selection as an input index list)
__global__ void __launch_bounds__(256) k_gather_sel(const int32_t* __restrict__ keep, int64_t n, int64_t n_match,
                                                    const float4* __restrict__ cpw, const float4* __restrict__ nsd,
                                                    const double* __restrict__ nc, float4* __restrict__ o_cpw,
                                                    float4* __restrict__ o_nsd, double* __restrict__ o_nc, int* __restrict__ bad) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int k = keep[i];
  if (k < 0 || k >= n_match) { atomicAdd(bad, 1); return; }
  o_cpw[i] = cpw[k];
  if (nsd) o_nsd[i] = nsd[k];
  if (nc) {
#pragma unroll
    for (int c = 0; c < 6; ++c) o_nc[6 * i + c] = nc[6 * (int64_t)k + c];
  }
}

void gather_selection(const int32_t* d_keep, int64_t n, int64_t n_match, const float4* cpw, const float4* nsd, const double* nc,
                      float4* o_cpw, float4* o_nsd, double* o_nc, int* d_bad, cudaStream_t st, LaunchCounter& lc) {
  if (n <= 0) return;
  lc.begin("k_gather_sel", st); k_gather_sel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(d_keep, n, n_match, cpw, nsd, nc, o_cpw, o_nsd, o_nc, d_bad); lc.end(st);
  GLIO_CUDA_TRY(cudaGetLastError());
}

}  // namespace glio
