// grid.cu — K0: uniform-grid build over a point cloud (replaces pcl::KdTreeFLANN::setInputCloud,
// GLIO/src/Estimator.cpp:2056,3729-3731,3821-3823) + the shared exclusive-scan primitive.
//
// Layout: points are counting-sorted by cell id ((cz*ny + cy)*nx + cx, x fastest) into float4
// (x, y, z, bitcast(original index)).  HBM traffic: read 4*stride*n, write 16 n + the cell table.
#include "common.cuh"
#include "devmath.cuh"

namespace glio {

// ------------------------------------------------------------------------------------------------
// exclusive scan (int32), 3-phase: per-block scan of 4096 items + scan of block sums (recursive) + add.
// ------------------------------------------------------------------------------------------------
constexpr int SCAN_T = 1024;
constexpr int SCAN_IPT = 4;
constexpr int SCAN_B = SCAN_T * SCAN_IPT;

__global__ void __launch_bounds__(SCAN_T) k_scan_block(const int* __restrict__ in, int* __restrict__ out,
                                                        int* __restrict__ block_sums, int64_t n) {
  __shared__ int warp_sums[32];
  const int64_t base = (int64_t)blockIdx.x * SCAN_B + (int64_t)threadIdx.x * SCAN_IPT;
  int v[SCAN_IPT];
  int tsum = 0;
#pragma unroll
  for (int k = 0; k < SCAN_IPT; ++k) {
    v[k] = (base + k < n) ? in[base + k] : 0;
    tsum += v[k];
  }
  // inclusive warp scan of thread sums
  int x = tsum;
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    int y = __shfl_up_sync(0xffffffffu, x, o);
    if (lane >= o) x += y;
  }
  if (lane == 31) warp_sums[wid] = x;
  __syncthreads();
  if (wid == 0) {
    int w = warp_sums[lane];
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      int y = __shfl_up_sync(0xffffffffu, w, o);
      if (lane >= o) w += y;
    }
    warp_sums[lane] = w;
  }
  __syncthreads();
  int excl = x - tsum + (wid > 0 ? warp_sums[wid - 1] : 0);
#pragma unroll
  for (int k = 0; k < SCAN_IPT; ++k) {
    if (base + k < n) out[base + k] = excl;
    excl += v[k];
  }
  if (threadIdx.x == SCAN_T - 1 && block_sums) block_sums[blockIdx.x] = excl;
}

__global__ void __launch_bounds__(SCAN_T) k_scan_add(int* __restrict__ out, const int* __restrict__ block_offs, int64_t n) {
  const int add = block_offs[blockIdx.x];
  const int64_t base = (int64_t)blockIdx.x * SCAN_B + (int64_t)threadIdx.x * SCAN_IPT;
#pragma unroll
  for (int k = 0; k < SCAN_IPT; ++k)
    if (base + k < n) out[base + k] += add;
}

// second half of a two-launch scan: every block sums the block totals in front of it by itself (nb <= 4096 totals: one
// coalesced read + a block reduction) instead of waiting for a third launch to scan them
__global__ void __launch_bounds__(SCAN_T) k_scan_add2(int* __restrict__ out, const int* __restrict__ block_sums, int64_t n) {
  __shared__ int warp_sums[32];
  int part = 0;
  for (int i = threadIdx.x; i < (int)blockIdx.x; i += SCAN_T) part += block_sums[i];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) part += __shfl_xor_sync(0xffffffffu, part, o);
  if ((threadIdx.x & 31) == 0) warp_sums[threadIdx.x >> 5] = part;
  __syncthreads();
  int add = 0;
#pragma unroll
  for (int w = 0; w < SCAN_T / 32; ++w) add += warp_sums[w];
  if (blockIdx.x == 0) return;
  const int64_t base = (int64_t)blockIdx.x * SCAN_B + (int64_t)threadIdx.x * SCAN_IPT;
#pragma unroll
  for (int k = 0; k < SCAN_IPT; ++k)
    if (base + k < n) out[base + k] += add;
}

static void scan_rec(const int* in, int* out, int64_t n, int* tmp, int64_t tmp_cap, cudaStream_t st, LaunchCounter& lc) {
  const int64_t nb = (n + SCAN_B - 1) / SCAN_B;
  if (nb <= 1) {
    lc.begin("k_scan_block", st); k_scan_block<<<1, SCAN_T, 0, st>>>(in, out, nullptr, n); lc.end(st);
    return;
  }
  GLIO_REQUIRE(nb <= tmp_cap, GLIO_ERR_STATE, "scan scratch too small");
  lc.begin("k_scan_block", st); k_scan_block<<<(unsigned)nb, SCAN_T, 0, st>>>(in, out, tmp, n); lc.end(st);
  if (nb <= 4096) {
    lc.begin("k_scan_add", st); k_scan_add2<<<(unsigned)nb, SCAN_T, 0, st>>>(out, tmp, n); lc.end(st);
    return;
  }
  scan_rec(tmp, tmp, nb, tmp + nb, tmp_cap - nb, st, lc);
  lc.begin("k_scan_add", st); k_scan_add<<<(unsigned)nb, SCAN_T, 0, st>>>(out, tmp, n); lc.end(st);
}

void exclusive_scan_i32(const int* in, int* out, int64_t n, DevBuf<int>& tmp, cudaStream_t st, LaunchCounter& lc) {
  if (n <= 0) return;
  int64_t need = 0;
  for (int64_t m = (n + SCAN_B - 1) / SCAN_B; m > 1; m = (m + SCAN_B - 1) / SCAN_B) need += m;
  need += 8;
  tmp.reserve((size_t)need);
  scan_rec(in, out, n, tmp.p, (int64_t)tmp.cap, st, lc);
  GLIO_CUDA_TRY(cudaGetLastError());
}

// ------------------------------------------------------------------------------------------------
// grid build kernels
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ int float_to_ordered(float f) {
  int i = __float_as_int(f);
  return i ^ ((i >> 31) & 0x7fffffff);
}
__host__ __device__ __forceinline__ float ordered_to_float_h(int i) {
  int j = i ^ ((i >> 31) & 0x7fffffff);
#ifdef __CUDA_ARCH__
  return __int_as_float(j);
#else
  float f; memcpy(&f, &j, 4); return f;
#endif
}

// load (and optionally transform: world = float(q*double(p)+t), Estimator.cpp:1517-1545) points into float4 + index,
// and reduce the bounding box.
__global__ void __launch_bounds__(256) k_load_bounds(const float* __restrict__ xyz, int stride, int64_t n, PoseD pose, int has_pose,
                                                     float4* __restrict__ out, int* __restrict__ bounds /*6 ordered ints*/) {
  float mn[3] = {3.0e38f, 3.0e38f, 3.0e38f}, mx[3] = {-3.0e38f, -3.0e38f, -3.0e38f};
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    float p[3] = {xyz[i * stride], xyz[i * stride + 1], xyz[i * stride + 2]};
    if (has_pose) transform_point_f(pose, p, p);
    out[i] = make_float4(p[0], p[1], p[2], __int_as_float((int)i));
#pragma unroll
    for (int d = 0; d < 3; ++d) { mn[d] = fminf(mn[d], p[d]); mx[d] = fmaxf(mx[d], p[d]); }
  }
#pragma unroll
  for (int d = 0; d < 3; ++d) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      mn[d] = fminf(mn[d], __shfl_xor_sync(0xffffffffu, mn[d], o));
      mx[d] = fmaxf(mx[d], __shfl_xor_sync(0xffffffffu, mx[d], o));
    }
  }
  // one set of global atomics per block (8 warps -> shared memory -> thread 0), not per warp
  __shared__ float smn[8][3], smx[8][3];
  const int wid = threadIdx.x >> 5;
  if ((threadIdx.x & 31) == 0) {
#pragma unroll
    for (int d = 0; d < 3; ++d) { smn[wid][d] = mn[d]; smx[wid][d] = mx[d]; }
  }
  __syncthreads();
  if (threadIdx.x < 3) {
    const int d = threadIdx.x;
    float a = smn[0][d], b = smx[0][d];
    for (int w = 1; w < (int)(blockDim.x >> 5); ++w) { a = fminf(a, smn[w][d]); b = fmaxf(b, smx[w][d]); }
    atomicMin(&bounds[d], float_to_ordered(a));
    atomicMax(&bounds[3 + d], float_to_ordered(b));
  }
}

__global__ void k_init_bounds(int* bounds) {
  if (threadIdx.x < 3) bounds[threadIdx.x] = 0x7fffffff;
  else if (threadIdx.x < 6) bounds[threadIdx.x] = (int)0x80000000;
}

__global__ void __launch_bounds__(256) k_cell_hist(const float4* __restrict__ pts, int64_t n, GridDesc g, int* __restrict__ count) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    float4 p = pts[i];
    atomicAdd(&count[cell_of_clamped(g, p.x, p.y, p.z)], 1);
  }
}

__global__ void __launch_bounds__(256) k_cell_scatter(const float4* __restrict__ pts, int64_t n, GridDesc g,
                                                      const int* __restrict__ cell_start, int* __restrict__ fill,
                                                      float4* __restrict__ sorted, int* __restrict__ sorted_pos) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    float4 p = pts[i];
    int c = cell_of_clamped(g, p.x, p.y, p.z);
    int pos = cell_start[c] + atomicAdd(&fill[c], 1);
    sorted[pos] = p;
    sorted_pos[i] = pos;          // original index -> position in the cell-sorted copy (K1b gathers neighbours from there)
  }
}

// The face tests (box_face_open, axis_gap, nn_face_open) compute a face as ox + (float)k * cell and a point's cell as
// floor((x - ox) * inv_cell), each rounded in float.  The two roundings can disagree near a face: a point up to a few
// spacings of the float grid (ulp) nearer than the computed face can be counted beyond it.  The face distances are
// therefore shrunk by this slack: the 2 mm of old while every face and cell corner of the grid stays below 2^12 m in
// magnitude, 8 ulp(M) above (M: the largest |ox|, |ox + n*cell| over the axes), which covers the worst disagreement of
// tests/test_knn_margins.py with room to spare.  Queries add no term: the face distance b = face - q is rounded
// relative to b, which the 0.999 factor covers.
static float face_slack(const GridDesc& g) {
  const float o[3] = {g.ox, g.oy, g.oz};
  const int n[3] = {g.nx, g.ny, g.nz};
  float M = 0.f;
  for (int d = 0; d < 3; ++d) M = std::max(M, std::max(std::fabs(o[d]), std::fabs(o[d] + (float)n[d] * g.cell)));
  const float ulp = std::nextafter(M, INFINITY) - M;
  return std::max(2e-3f, 8.f * ulp);
}

void grid_build(GridBuild& gb, const float* d_xyz, int stride, int64_t n, const double* t, const double* q,
                float cell_size_hint, float pts_per_cell, cudaStream_t st, LaunchCounter& lc) {
  GLIO_REQUIRE(n > 0 && n < (int64_t)1 << 31, GLIO_ERR_ARG, "grid_build: point count out of range");
  gb.tmp4.reserve((size_t)n);
  gb.pts.reserve((size_t)n);
  gb.sorted_pos.reserve((size_t)n);
  gb.bounds.reserve(8);
  PoseD pose{};
  int has_pose = 0;
  if (t && q) { has_pose = 1; for (int k = 0; k < 3; ++k) pose.t[k] = t[k]; for (int k = 0; k < 4; ++k) pose.q[k] = q[k]; }
  int* d_bounds = (int*)gb.bounds.p;
  lc.begin("k_init_bounds", st); k_init_bounds<<<1, 32, 0, st>>>(d_bounds); lc.end(st);
  const int nb = (int)std::min<int64_t>((n + 255) / 256, kNumSMs * 8);
  lc.begin("k_load_bounds", st); k_load_bounds<<<nb, 256, 0, st>>>(d_xyz, stride, n, pose, has_pose, gb.tmp4.p, d_bounds); lc.end(st);
  int hb[6];
  GLIO_CUDA_TRY(cudaMemcpyAsync(hb, d_bounds, sizeof(hb), cudaMemcpyDeviceToHost, st));
  GLIO_CUDA_TRY(cudaStreamSynchronize(st));
  float mn[3], mx[3];
  for (int d = 0; d < 3; ++d) { mn[d] = ordered_to_float_h(hb[d]); mx[d] = ordered_to_float_h(hb[3 + d]); }
  for (int d = 0; d < 3; ++d)
    GLIO_REQUIRE(std::isfinite(mn[d]) && std::isfinite(mx[d]), GLIO_ERR_ARG, "grid_build: non-finite point coordinates");
  // cell size: caller hint, else from the bounding-box surface area (LiDAR clouds are surfaces): about
  // pts_per_cell points per occupied cell.
  float L[3] = {mx[0] - mn[0] + 1e-3f, mx[1] - mn[1] + 1e-3f, mx[2] - mn[2] + 1e-3f};
  float cell = cell_size_hint;
  if (!(cell > 0)) {
    double area = 2.0 * ((double)L[0] * L[1] + (double)L[1] * L[2] + (double)L[0] * L[2]);
    cell = (float)std::sqrt(pts_per_cell * area / (double)n);
    if (cell < 0.05f) cell = 0.05f;
    if (cell > 4.0f) cell = 4.0f;
  }
  const double max_cells = 48.0e6;
  for (;;) {
    double nc = std::ceil(L[0] / cell + 1) * std::ceil(L[1] / cell + 1) * std::ceil(L[2] / cell + 1);
    if (nc <= max_cells) break;
    cell *= 1.26f;
  }
  GridDesc& g = gb.desc;
  g.cell = cell; g.inv_cell = 1.0f / cell;
  g.ox = mn[0] - 0.5f * cell; g.oy = mn[1] - 0.5f * cell; g.oz = mn[2] - 0.5f * cell;
  g.nx = (int)std::floor((mx[0] - g.ox) / cell) + 2;
  g.ny = (int)std::floor((mx[1] - g.oy) / cell) + 2;
  g.nz = (int)std::floor((mx[2] - g.oz) / cell) + 2;
  g.npts = n;
  g.slack = face_slack(g);
  const int64_t ncell = (int64_t)g.nx * g.ny * g.nz;
  gb.cell_start.reserve((size_t)ncell + 2);
  gb.fill.reserve((size_t)ncell + 2);
  GLIO_CUDA_TRY(cudaMemsetAsync(gb.fill.p, 0, (size_t)(ncell + 1) * sizeof(int), st));
  lc.begin("k_cell_hist", st); k_cell_hist<<<nb, 256, 0, st>>>(gb.tmp4.p, n, g, gb.fill.p); lc.end(st);
  exclusive_scan_i32(gb.fill.p, gb.cell_start.p, ncell + 1, gb.scan_tmp, st, lc);
  GLIO_CUDA_TRY(cudaMemsetAsync(gb.fill.p, 0, (size_t)(ncell + 1) * sizeof(int), st));
  lc.begin("k_cell_scatter", st); k_cell_scatter<<<nb, 256, 0, st>>>(gb.tmp4.p, n, g, gb.cell_start.p, gb.fill.p, gb.pts.p, gb.sorted_pos.p); lc.end(st);
  GLIO_CUDA_TRY(cudaGetLastError());
  g.cell_start = gb.cell_start.p;
  g.pts = gb.pts.p;
}

// =====================================================================================================================
// Local map maintenance on the device (SURVEY 8 f-1): keyframe clouds moved to the world frame when they are pushed
// (transformCloud, Estimator.cpp:1517-1545), concatenated, then pcl::VoxelGrid down-sampling as GLIO configures it
// (ds_filter_surf_map, leaf 0.4 m, Estimator.cpp:854, 3617-3618).  The voxel filter is a counting sort by PCL's voxel
// index (float min/max, min_b = floor(min*inv_leaf), idx = ijk0 + ijk1*div0 + ijk2*div0*div1) followed by a per-voxel float
// sum in INPUT order and a float division by the count; output in ascending voxel index (PCL's output order).
// PCL sums the points of a voxel in whatever order std::sort leaves them; summing in input order is the deterministic
// member of that family (the stable order).
// =====================================================================================================================
__global__ void __launch_bounds__(256) k_lm_transform(const float* __restrict__ xyz, int stride, int64_t n, PoseD pose, float4* __restrict__ out) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    float p[3] = {xyz[i * stride], xyz[i * stride + 1], xyz[i * stride + 2]};
    transform_point_f(pose, p, p);
    out[i] = make_float4(p[0], p[1], p[2], 0.f);
  }
}

void localmap_transform(const float* d_xyz, int stride, int64_t n, const double* t, const double* q, float4* d_out, cudaStream_t st, LaunchCounter& lc) {
  PoseD pose;
  for (int k = 0; k < 3; ++k) pose.t[k] = t[k];
  for (int k = 0; k < 4; ++k) pose.q[k] = q[k];
  const int nb = (int)std::min<int64_t>((n + 255) / 256, kNumSMs * 8);
  lc.begin("k_lm_transform", st); k_lm_transform<<<nb, 256, 0, st>>>(d_xyz, stride, n, pose, d_out); lc.end(st);
  GLIO_CUDA_TRY(cudaGetLastError());
}

struct VoxelDesc { float inv; int min_b[3]; int div0, div01; };
__device__ __forceinline__ int voxel_of(const VoxelDesc& v, float x, float y, float z) {
  const int i0 = (int)__fsub_rn(floorf(__fmul_rn(x, v.inv)), (float)v.min_b[0]);
  const int i1 = (int)__fsub_rn(floorf(__fmul_rn(y, v.inv)), (float)v.min_b[1]);
  const int i2 = (int)__fsub_rn(floorf(__fmul_rn(z, v.inv)), (float)v.min_b[2]);
  return i0 + i1 * v.div0 + i2 * v.div01;
}
__global__ void __launch_bounds__(256) k_vox_hist(const float4* __restrict__ pts, int64_t n, VoxelDesc v, int* __restrict__ count) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const float4 p = pts[i];
    atomicAdd(&count[voxel_of(v, p.x, p.y, p.z)], 1);
  }
}
__global__ void __launch_bounds__(256) k_vox_scatter(const float4* __restrict__ pts, int64_t n, VoxelDesc v, const int* __restrict__ start,
                                                     int* __restrict__ fill, int* __restrict__ order) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const float4 p = pts[i];
    const int c = voxel_of(v, p.x, p.y, p.z);
    order[start[c] + atomicAdd(&fill[c], 1)] = (int)i;
  }
}
// Order the point indices of every voxel ascending (= input order): the atomic scatter leaves them in arrival order.
// One warp per voxel: bitonic sort of 32*K keys held K per lane (shuffles for partner distances < 32, register swaps
// above); voxels with more than 256 points fall back to counting ranks.
template <int K>
__device__ __forceinline__ void warp_bitonic_sort(int (&v)[K], int lane) {
  constexpr int N = 32 * K;
#pragma unroll
  for (int k = 2; k <= N; k <<= 1) {
#pragma unroll
    for (int j = k >> 1; j > 0; j >>= 1) {
      if (j >= 32) {
        const int jr = j >> 5;
#pragma unroll
        for (int r = 0; r < K; ++r) {
          const int pr = r ^ jr;
          if (pr > r) {
            const bool asc = (((r << 5) + lane) & k) == 0;
            const int a = v[r], b = v[pr];
            const bool sw = asc ? (a > b) : (a < b);
            v[r] = sw ? b : a; v[pr] = sw ? a : b;
          }
        }
      } else {
#pragma unroll
        for (int r = 0; r < K; ++r) {
          const bool asc = (((r << 5) + lane) & k) == 0;
          const int o = __shfl_xor_sync(0xffffffffu, v[r], j);
          const bool lower = (lane & j) == 0;
          v[r] = (lower == asc) ? min(v[r], o) : max(v[r], o);
        }
      }
    }
  }
}

template <int K>
__device__ __forceinline__ void sort_segment(const int* __restrict__ order, int* __restrict__ sorted, int s, int n, int lane) {
  int v[K];
#pragma unroll
  for (int r = 0; r < K; ++r) { const int i = (r << 5) + lane; v[r] = i < n ? order[s + i] : 0x7fffffff; }
  warp_bitonic_sort<K>(v, lane);
#pragma unroll
  for (int r = 0; r < K; ++r) { const int i = (r << 5) + lane; if (i < n) sorted[s + i] = v[r]; }
}

__global__ void __launch_bounds__(256) k_vox_sort(const int* __restrict__ start, int64_t nvox, const int* __restrict__ order, int* __restrict__ sorted) {
  const int lane = threadIdx.x & 31;
  const int64_t nwarps = (int64_t)gridDim.x * (blockDim.x >> 5);
  for (int64_t c0 = ((int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5)) * 32; c0 < nvox; c0 += nwarps * 32) {
    // the 32 lanes look at 32 consecutive voxels, then the warp serves the non-empty ones in turn
    const int64_t c = c0 + lane;
    int s = 0, n = 0;
    if (c < nvox) { s = start[c]; n = start[c + 1] - s; }
    unsigned m = __ballot_sync(0xffffffffu, n > 0);
    while (m) {
      const int l = __ffs(m) - 1; m &= m - 1;
      const int ss = __shfl_sync(0xffffffffu, s, l), nn = __shfl_sync(0xffffffffu, n, l);
      if (nn == 1) { if (lane == 0) sorted[ss] = order[ss]; }
      else if (nn <= 32) sort_segment<1>(order, sorted, ss, nn, lane);
      else if (nn <= 64) sort_segment<2>(order, sorted, ss, nn, lane);
      else if (nn <= 128) sort_segment<4>(order, sorted, ss, nn, lane);
      else if (nn <= 256) sort_segment<8>(order, sorted, ss, nn, lane);
      else {
        for (int i = lane; i < nn; i += 32) {
          const int key = order[ss + i];
          int r = 0;
          for (int k = 0; k < nn; ++k) r += order[ss + k] < key ? 1 : 0;
          sorted[ss + r] = key;
        }
      }
    }
  }
}
__global__ void __launch_bounds__(256) k_vox_flags(const int* __restrict__ start, int64_t nvox, int* __restrict__ flags) {
  const int64_t c = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (c < nvox) flags[c] = start[c + 1] > start[c] ? 1 : 0;
  if (c == nvox) flags[c] = 0;
}
__global__ void __launch_bounds__(256) k_vox_centroid(const float4* __restrict__ pts, const int* __restrict__ start, const int* __restrict__ sorted,
                                                      const int* __restrict__ opos, int64_t nvox, float* __restrict__ out_xyz, int* __restrict__ out_vox) {
  const int64_t c = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= nvox) return;
  const int s = start[c], e = start[c + 1];
  if (e <= s) return;
  float sx = 0.f, sy = 0.f, sz = 0.f;
  for (int k = s; k < e; ++k) { const float4 p = pts[sorted[k]]; sx = __fadd_rn(sx, p.x); sy = __fadd_rn(sy, p.y); sz = __fadd_rn(sz, p.z); }
  const float cnt = (float)(e - s);
  const int o = opos[c];
  out_xyz[3 * (size_t)o] = __fdiv_rn(sx, cnt); out_xyz[3 * (size_t)o + 1] = __fdiv_rn(sy, cnt); out_xyz[3 * (size_t)o + 2] = __fdiv_rn(sz, cnt);
  if (out_vox) out_vox[o] = (int)c;
}

// Set-up shared by the dense and the sort-based filter: the points (stride floats apart) copied as float4 (x, y, z, index) into
// tmp4 while their float min / max is reduced (getMinMax3D), read back to the host (one synchronisation).
static void voxel_bounds(const float* d_xyz, int stride, int64_t n, float4* tmp4, int* d_bounds, float mn[3], float mx[3], cudaStream_t st,
                         LaunchCounter& lc) {
  lc.begin("k_init_bounds", st); k_init_bounds<<<1, 32, 0, st>>>(d_bounds); lc.end(st);
  const int nb = (int)std::min<int64_t>((n + 255) / 256, kNumSMs * 8);
  PoseD none{};
  lc.begin("k_load_bounds", st); k_load_bounds<<<nb, 256, 0, st>>>(d_xyz, stride, n, none, 0, tmp4, d_bounds); lc.end(st);
  int hb[6];
  GLIO_CUDA_TRY(cudaMemcpyAsync(hb, d_bounds, sizeof(hb), cudaMemcpyDeviceToHost, st));
  GLIO_CUDA_TRY(cudaStreamSynchronize(st));
  for (int d = 0; d < 3; ++d) { mn[d] = ordered_to_float_h(hb[d]); mx[d] = ordered_to_float_h(hb[3 + d]); }
  for (int d = 0; d < 3; ++d) GLIO_REQUIRE(std::isfinite(mn[d]) && std::isfinite(mx[d]), GLIO_ERR_ARG, "voxel_filter: non-finite point coordinates");
}

// PCL's leaf-size check and voxel layout (VoxelGrid::applyFilter): false when PCL passes the input through unchanged.  div01 is
// div0 * div1 wrapped to 32 bits, as PCL's int arithmetic leaves it.
static bool voxel_layout(const float mn[3], const float mx[3], float leaf, VoxelDesc& v, int div[3]) {
  const float inv = 1.0f / leaf;                               // setLeafSize: Array4f::Ones() / leaf
  const int64_t dx = (int64_t)((mx[0] - mn[0]) * inv) + 1, dy = (int64_t)((mx[1] - mn[1]) * inv) + 1, dz = (int64_t)((mx[2] - mn[2]) * inv) + 1;
  if (dx * dy * dz > (int64_t)0x7fffffff) return false;        // PCL: "leaf size too small", input passed through
  v.inv = inv;
  for (int d = 0; d < 3; ++d) { v.min_b[d] = (int)std::floor(mn[d] * inv); div[d] = (int)std::floor(mx[d] * inv) - v.min_b[d] + 1; }
  v.div0 = div[0]; v.div01 = (int)((uint32_t)div[0] * (uint32_t)div[1]);
  return true;
}

int64_t voxel_filter_run(VoxelWork& w, const float4* d_in, int64_t n, float leaf, cudaStream_t st, LaunchCounter& lc) {
  GLIO_REQUIRE(n > 0 && n < ((int64_t)1 << 31), GLIO_ERR_ARG, "voxel_filter: bad point count");
  GLIO_REQUIRE(leaf > 0.f, GLIO_ERR_ARG, "voxel_filter: leaf size must be positive");
  w.tmp4.reserve((size_t)n); w.bounds.reserve(8);
  const int nb = (int)std::min<int64_t>((n + 255) / 256, kNumSMs * 8);
  float mn[3], mx[3];
  voxel_bounds(reinterpret_cast<const float*>(d_in), 4, n, w.tmp4.p, w.bounds.p, mn, mx, st, lc);
  VoxelDesc v;
  int div[3];
  if (!voxel_layout(mn, mx, leaf, v, div)) return -1;
  const int64_t nvox = (int64_t)div[0] * div[1] * div[2];
  GLIO_REQUIRE(nvox <= (int64_t)256 * 1024 * 1024, GLIO_ERR_ARG, "voxel_filter: more than 2^28 voxels in the bounding box (dense voxel table)");
  w.count.reserve((size_t)nvox + 2); w.start.reserve((size_t)nvox + 2); w.opos.reserve((size_t)nvox + 2);
  w.order.reserve((size_t)n); w.sorted.reserve((size_t)n); w.out_xyz.reserve((size_t)n * 3); w.out_vox.reserve((size_t)n);
  GLIO_CUDA_TRY(cudaMemsetAsync(w.count.p, 0, (size_t)(nvox + 1) * sizeof(int), st));
  lc.begin("k_vox_hist", st); k_vox_hist<<<nb, 256, 0, st>>>(w.tmp4.p, n, v, w.count.p); lc.end(st);
  exclusive_scan_i32(w.count.p, w.start.p, nvox + 1, w.scan_tmp, st, lc);
  GLIO_CUDA_TRY(cudaMemsetAsync(w.count.p, 0, (size_t)(nvox + 1) * sizeof(int), st));
  lc.begin("k_vox_scatter", st); k_vox_scatter<<<nb, 256, 0, st>>>(w.tmp4.p, n, v, w.start.p, w.count.p, w.order.p); lc.end(st);
  lc.begin("k_vox_sort", st); k_vox_sort<<<kNumSMs * 8, 256, 0, st>>>(w.start.p, nvox, w.order.p, w.sorted.p); lc.end(st);
  const unsigned nbv = (unsigned)((nvox + 1 + 255) / 256);
  lc.begin("k_vox_flags", st); k_vox_flags<<<nbv, 256, 0, st>>>(w.start.p, nvox, w.count.p); lc.end(st);
  exclusive_scan_i32(w.count.p, w.opos.p, nvox + 1, w.scan_tmp, st, lc);
  lc.begin("k_vox_centroid", st); k_vox_centroid<<<nbv, 256, 0, st>>>(w.tmp4.p, w.start.p, w.sorted.p, w.opos.p, nvox, w.out_xyz.p, w.out_vox.p); lc.end(st);
  int m = 0;
  GLIO_CUDA_TRY(cudaMemcpyAsync(&m, w.opos.p + nvox, sizeof(int), cudaMemcpyDeviceToHost, st));
  GLIO_CUDA_TRY(cudaStreamSynchronize(st));
  GLIO_CUDA_TRY(cudaGetLastError());
  return (int64_t)m;
}

// =====================================================================================================================
// Sort-based pcl::VoxelGrid (glio_voxel_filter, glio_loop_global_map): the same keys, order and sums as the dense filter above,
// but its cost follows the number of points instead of the bounding box.  One 32-bit key per point (PCL's voxel index, int
// arithmetic wrapped to 32 bits and compared unsigned, as PCL's cloud_point_index_idx does), a stable LSD radix sort of
// (key, point index) over the key bits the box needs, segment heads, their exclusive scan, one centroid per segment summed in
// input order.  Kernels: k_vs_key, per pass k_vs_hist + k_scan_block / k_scan_add + k_vs_scatter, then k_vs_heads,
// k_scan_block / k_scan_add, k_vs_centroid; k_vs_pack instead of all of these when PCL passes the input through.
// =====================================================================================================================
constexpr int VS_T = 256;                 // threads of the radix kernels
constexpr int VS_R = 8;                   // rounds of VS_T keys per block: a block sorts a tile of 2048 consecutive keys
constexpr int VS_TILE = VS_T * VS_R;
constexpr int VS_DIGIT = 8;               // key bits per pass

__device__ __forceinline__ unsigned voxel_key(const VoxelDesc& v, float x, float y, float z) {
  const int i0 = (int)__fsub_rn(floorf(__fmul_rn(x, v.inv)), (float)v.min_b[0]);
  const int i1 = (int)__fsub_rn(floorf(__fmul_rn(y, v.inv)), (float)v.min_b[1]);
  const int i2 = (int)__fsub_rn(floorf(__fmul_rn(z, v.inv)), (float)v.min_b[2]);
  return (unsigned)i0 + (unsigned)i1 * (unsigned)v.div0 + (unsigned)i2 * (unsigned)v.div01;
}

__global__ void __launch_bounds__(256) k_vs_key(const float4* __restrict__ pts, int64_t n, VoxelDesc v, unsigned* __restrict__ keys,
                                                int* __restrict__ vals, int* __restrict__ bad) {
  bool finite = true;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const float4 p = pts[i];
    finite = finite && isfinite(p.x) && isfinite(p.y) && isfinite(p.z);
    keys[i] = voxel_key(v, p.x, p.y, p.z);
    vals[i] = (int)i;
  }
  if (!finite) atomicOr(bad, 1);
}

// digit counts of one block's tile, stored digit-major (hist[d * gridDim.x + block]) so that one exclusive scan gives every
// (digit, block) its first output position
__global__ void __launch_bounds__(VS_T) k_vs_hist(const unsigned* __restrict__ keys, int64_t n, int shift, int nbits, int* __restrict__ hist) {
  __shared__ int h[1 << VS_DIGIT];
  const unsigned mask = (1u << nbits) - 1u;
  h[threadIdx.x] = 0;
  __syncthreads();
  const int64_t base = (int64_t)blockIdx.x * VS_TILE;
#pragma unroll
  for (int r = 0; r < VS_R; ++r) {
    const int64_t i = base + r * VS_T + threadIdx.x;
    if (i < n) atomicAdd(&h[(keys[i] >> shift) & mask], 1);
  }
  __syncthreads();
  if (threadIdx.x <= mask) hist[(int64_t)threadIdx.x * gridDim.x + blockIdx.x] = h[threadIdx.x];
}

// Stable scatter of one block's tile: the tile is taken VS_T keys at a time in input order; inside a warp the lanes with the same
// digit rank themselves by lane (match_any), the warps of a round follow each other in warp order, and the rounds in tile order.
__global__ void __launch_bounds__(VS_T) k_vs_scatter(const unsigned* __restrict__ kin, const int* __restrict__ vin, int64_t n, int shift,
                                                     int nbits, const int* __restrict__ offs, unsigned* __restrict__ kout,
                                                     int* __restrict__ vout) {
  constexpr int NW = VS_T / 32;
  __shared__ int run[1 << VS_DIGIT];          // next output position of each digit
  __shared__ int wc[NW][1 << VS_DIGIT];       // this round's per-warp digit counts, then each warp's first position
  const unsigned mask = (1u << nbits) - 1u;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const unsigned lt = (1u << lane) - 1u;
  run[threadIdx.x] = threadIdx.x <= mask ? offs[(int64_t)threadIdx.x * gridDim.x + blockIdx.x] : 0;
  const int64_t base = (int64_t)blockIdx.x * VS_TILE;
  for (int r = 0; r < VS_R; ++r) {
#pragma unroll
    for (int w = 0; w < NW; ++w) wc[w][threadIdx.x] = 0;
    __syncthreads();
    const int64_t i = base + r * VS_T + threadIdx.x;
    const bool valid = i < n;
    const unsigned key = valid ? kin[i] : 0u;
    const int val = valid ? vin[i] : 0;
    const unsigned d = valid ? (key >> shift) & mask : 0xffffffffu;      // invalid lanes never match a digit
    const unsigned peers = __match_any_sync(0xffffffffu, d);
    const int rank = __popc(peers & lt);
    if (valid && rank == 0) wc[warp][d] = __popc(peers);
    __syncthreads();
    if (threadIdx.x <= mask) {
      int s = run[threadIdx.x];
#pragma unroll
      for (int w = 0; w < NW; ++w) { const int c = wc[w][threadIdx.x]; wc[w][threadIdx.x] = s; s += c; }
      run[threadIdx.x] = s;
    }
    __syncthreads();
    if (valid) {
      const int o = wc[warp][d] + rank;
      kout[o] = key; vout[o] = val;
    }
    __syncthreads();
  }
}

__global__ void __launch_bounds__(256) k_vs_heads(const unsigned* __restrict__ keys, int64_t n, int* __restrict__ flags) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i <= n; i += (int64_t)gridDim.x * blockDim.x)
    flags[i] = (i < n && (i == 0 || keys[i] != keys[i - 1])) ? 1 : 0;
}

// one thread per segment (its head): float sums in input order (the sort is stable), divided by the float count
__global__ void __launch_bounds__(256) k_vs_centroid(const float4* __restrict__ pts, const unsigned* __restrict__ keys, const int* __restrict__ vals,
                                                     const int* __restrict__ flags, const int* __restrict__ pos, int64_t n, float* __restrict__ out_xyz) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    if (!flags[i]) continue;
    const unsigned k = keys[i];
    float sx = 0.f, sy = 0.f, sz = 0.f;
    int64_t j = i;
    do {
      const float4 p = pts[vals[j]];
      sx = __fadd_rn(sx, p.x); sy = __fadd_rn(sy, p.y); sz = __fadd_rn(sz, p.z);
      ++j;
    } while (j < n && keys[j] == k);
    const float cnt = (float)(j - i);
    const size_t o = 3 * (size_t)pos[i];
    out_xyz[o] = __fdiv_rn(sx, cnt); out_xyz[o + 1] = __fdiv_rn(sy, cnt); out_xyz[o + 2] = __fdiv_rn(sz, cnt);
  }
}

// PCL's pass-through: the input x,y,z as they are
__global__ void __launch_bounds__(256) k_vs_pack(const float4* __restrict__ pts, int64_t n, float* __restrict__ out_xyz, int* __restrict__ bad) {
  bool finite = true;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const float4 p = pts[i];
    finite = finite && isfinite(p.x) && isfinite(p.y) && isfinite(p.z);
    out_xyz[3 * i] = p.x; out_xyz[3 * i + 1] = p.y; out_xyz[3 * i + 2] = p.z;
  }
  if (!finite) atomicOr(bad, 1);
}

static int voxel_key_bits(const int div[3]) {
  const int64_t nvox = (int64_t)div[0] * div[1] * div[2];
  if (nvox > ((int64_t)1 << 32)) return 32;                    // the keys wrap: every bit can differ
  int b = 0;
  for (int64_t m = nvox - 1; m > 0; m >>= 1) ++b;              // keys are in [0, nvox)
  return b;
}

int64_t voxel_sort_run(VoxelSortWork& w, const float* d_xyz, int stride, int64_t n, float leaf, bool* filtered, cudaStream_t st, LaunchCounter& lc) {
  GLIO_REQUIRE(n > 0 && n < ((int64_t)1 << 31), GLIO_ERR_ARG, "voxel_filter: bad point count");
  GLIO_REQUIRE(leaf > 0.f && std::isfinite(leaf), GLIO_ERR_ARG, "voxel_filter: leaf size must be positive and finite");
  w.tmp4.reserve((size_t)n); w.bounds.reserve(8); w.bad.reserve(1); w.out_xyz.reserve((size_t)n * 3);
  float mn[3], mx[3];
  voxel_bounds(d_xyz, stride, n, w.tmp4.p, w.bounds.p, mn, mx, st, lc);
  // every point NaN: fminf / fmaxf skipped them all and the bounds are still the initial ones
  GLIO_REQUIRE(mn[0] <= mx[0] && mn[1] <= mx[1] && mn[2] <= mx[2], GLIO_ERR_ARG, "voxel_filter: non-finite point coordinates");
  GLIO_CUDA_TRY(cudaMemsetAsync(w.bad.p, 0, sizeof(int), st));
  const int nb = (int)std::min<int64_t>((n + 255) / 256, kNumSMs * 8);
  VoxelDesc v;
  int div[3];
  int m = 0;
  *filtered = voxel_layout(mn, mx, leaf, v, div);
  if (!*filtered) {
    lc.begin("k_vs_pack", st); k_vs_pack<<<nb, 256, 0, st>>>(w.tmp4.p, n, w.out_xyz.p, w.bad.p); lc.end(st);
    m = (int)n;
  } else {
    w.key0.reserve((size_t)n); w.key1.reserve((size_t)n); w.val0.reserve((size_t)n); w.val1.reserve((size_t)n);
    w.flags.reserve((size_t)n + 1); w.pos.reserve((size_t)n + 1);
    lc.begin("k_vs_key", st); k_vs_key<<<nb, 256, 0, st>>>(w.tmp4.p, n, v, w.key0.p, w.val0.p, w.bad.p); lc.end(st);
    const int bits = voxel_key_bits(div);
    const int64_t tiles = (n + VS_TILE - 1) / VS_TILE;
    w.hist.reserve((size_t)tiles << VS_DIGIT);
    unsigned *ka = w.key0.p, *kb = w.key1.p;
    int *va = w.val0.p, *vb = w.val1.p;
    for (int shift = 0; shift < bits; shift += VS_DIGIT) {
      const int nbits = std::min(VS_DIGIT, bits - shift);
      lc.begin("k_vs_hist", st); k_vs_hist<<<(unsigned)tiles, VS_T, 0, st>>>(ka, n, shift, nbits, w.hist.p); lc.end(st);
      exclusive_scan_i32(w.hist.p, w.hist.p, tiles << nbits, w.scan_tmp, st, lc);     // in place: every thread reads its items first
      lc.begin("k_vs_scatter", st); k_vs_scatter<<<(unsigned)tiles, VS_T, 0, st>>>(ka, va, n, shift, nbits, w.hist.p, kb, vb); lc.end(st);
      std::swap(ka, kb); std::swap(va, vb);
    }
    lc.begin("k_vs_heads", st); k_vs_heads<<<nb, 256, 0, st>>>(ka, n, w.flags.p); lc.end(st);
    exclusive_scan_i32(w.flags.p, w.pos.p, n + 1, w.scan_tmp, st, lc);
    lc.begin("k_vs_centroid", st); k_vs_centroid<<<nb, 256, 0, st>>>(w.tmp4.p, ka, va, w.flags.p, w.pos.p, n, w.out_xyz.p); lc.end(st);
    GLIO_CUDA_TRY(cudaMemcpyAsync(&m, w.pos.p + n, sizeof(int), cudaMemcpyDeviceToHost, st));
  }
  int bad = 0;
  GLIO_CUDA_TRY(cudaMemcpyAsync(&bad, w.bad.p, sizeof(int), cudaMemcpyDeviceToHost, st));
  GLIO_CUDA_TRY(cudaStreamSynchronize(st));
  GLIO_CUDA_TRY(cudaGetLastError());
  GLIO_REQUIRE(!bad, GLIO_ERR_ARG, "voxel_filter: non-finite point coordinates");
  return (int64_t)m;
}

void LocalMap::push(bool at_front, const float* d_xyz, int stride, int64_t n, const double* t, const double* q, cudaStream_t st, LaunchCounter& lc) {
  std::unique_ptr<Frame> f;
  if (!spare.empty()) { f = std::move(spare.back()); spare.pop_back(); }
  else f = std::make_unique<Frame>();
  f->pts.reserve((size_t)n); f->n = n;
  if (n > 0) localmap_transform(d_xyz, stride, n, t, q, f->pts.p, st, lc);
  if (at_front) frames.push_front(std::move(f)); else frames.push_back(std::move(f));
}

void LocalMap::pop_front() {
  spare.push_back(std::move(frames.front()));
  frames.pop_front();
}

void LocalMap::clear() {
  frames.clear();
  spare.clear();
}

int64_t LocalMap::n_points() const {
  int64_t np = 0;
  for (auto& f : frames) np += f->n;
  return np;
}

int64_t LocalMap::build(float leaf, const float** pts, int* stride, bool* filtered, cudaStream_t st, LaunchCounter& lc) {
  const int64_t N = n_points();
  cat.reserve((size_t)N);
  int64_t o = 0;
  for (auto& f : frames) {
    if (f->n) GLIO_CUDA_TRY(cudaMemcpyAsync(cat.p + o, f->pts.p, (size_t)f->n * sizeof(float4), cudaMemcpyDeviceToDevice, st));
    o += f->n;
  }
  const int64_t m = (leaf > 0.f && N > 0) ? voxel_filter_run(vox, cat.p, N, leaf, st, lc) : -1;
  *filtered = m >= 0;
  if (m >= 0) { *pts = vox.out_xyz.p; *stride = 3; return m; }
  *pts = reinterpret_cast<const float*>(cat.p); *stride = 4;
  return N;
}


}  // namespace glio
