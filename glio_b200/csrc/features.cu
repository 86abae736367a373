// features.cu — the front end's feature extraction on the device (SURVEY 8 f-4):
// Preprocessing::cloudHandler, GLIO/src/Preprocessing.cpp:529-655.  Input = `laserCloud`: the scan lines concatenated ring
// after ring (x, y, z, intensity at a caller stride) with scanStartInd / scanEndInd per ring.
//   k_feat_curvature  LOAM curvature of every point: |sum of the ten ring neighbours - 10 p|^2, float, the reference's
//                     left-to-right order (:537-546)
//   k_feat_select     one CTA per ring; the six sectors of a ring in order (their neighbour suppression reaches up to five
//                     points into the next sector, so sectors of a ring are sequential; rings run concurrently, which is
//                     the reference's sequential order only while no ring reads what another writes: a ring marks
//                     picked[] from scan_start - 5 to scan_end + 4 and reads and compacts within [scan_start, scan_end), so
//                     glio_extract_features refuses processed rings whose ranges, ordered by start, are less than 5 points
//                     apart (scan_start[next] < scan_end[prev] + 5); the reference's layout leaves 11): bitonic sort of
//                     the sector by (curvature, index) in shared memory, then the greedy pick of <= 2 sharp + <= 8 more less-sharp edge points from the top and <= 4
//                     flat points from the bottom with the +-5 suppression (:549-643), then the ordered compaction of the
//                     remaining label <= 0 points as "less flat" (:645-650)
//   k_feat_voxel      one CTA per ring: pcl::VoxelGrid (leaf ds_v) of the ring's less-flat points, all in shared memory:
//                     bounds, voxel index, sort by (voxel, position), per-voxel float sums in input order / count (:652-659)
//   k_feat_offsets / k_feat_gather   ring-major concatenation = the reference's push_back order
// std::sort leaves the order of EQUAL curvatures (and of points inside a voxel) to the implementation; ties are broken by
// index here, the deterministic member of that family.
// Compiled with -fmad=false: every float that decides a label or a voxel is rounded as on the reference's baseline x86-64.
#include "common.cuh"
#include "devmath.cuh"

namespace glio {

constexpr int FEAT_T = 256;
constexpr int FEAT_SECT_CAP = 4096;      // points of one sector that fit the shared-memory sort (a ring may have 6 x this)
constexpr int FEAT_RING_CAP = 8192;      // less-flat points of one ring that fit the shared-memory voxel filter

__device__ __forceinline__ float3 feat_pt(const FeatArgs& a, int64_t i) {
  const float* p = a.cloud + i * a.stride;
  return make_float3(p[0], p[1], p[2]);
}

__global__ void __launch_bounds__(256) k_feat_curvature(FeatArgs a) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= a.n) return;
  float c = 0.f;
  if (i >= 5 && i < a.n - 5) {
    float3 s = feat_pt(a, i - 5);
#pragma unroll
    for (int k = -4; k <= -1; ++k) { const float3 p = feat_pt(a, i + k); s.x = fadd(s.x, p.x); s.y = fadd(s.y, p.y); s.z = fadd(s.z, p.z); }
    const float3 p0 = feat_pt(a, i);
    s.x = fsub(s.x, fmul(10.f, p0.x)); s.y = fsub(s.y, fmul(10.f, p0.y)); s.z = fsub(s.z, fmul(10.f, p0.z));
#pragma unroll
    for (int k = 1; k <= 5; ++k) { const float3 p = feat_pt(a, i + k); s.x = fadd(s.x, p.x); s.y = fadd(s.y, p.y); s.z = fadd(s.z, p.z); }
    c = fadd(fadd(fmul(s.x, s.x), fmul(s.y, s.y)), fmul(s.z, s.z));
  }
  a.curv[i] = c;
}

// block-wide bitonic sort of n 64-bit keys in shared memory (n <= cap, cap a power of two)
__device__ __forceinline__ void block_bitonic(unsigned long long* keys, int n) {
  int np2 = 1; while (np2 < n) np2 <<= 1;
  for (int i = n + threadIdx.x; i < np2; i += blockDim.x) keys[i] = ~0ull;
  __syncthreads();
  for (int k = 2; k <= np2; k <<= 1)
    for (int j = k >> 1; j > 0; j >>= 1) {
      for (int i = threadIdx.x; i < np2; i += blockDim.x) {
        const int l = i ^ j;
        if (l > i) {
          const unsigned long long x = keys[i], y = keys[l];
          const bool asc = (i & k) == 0;
          if ((x > y) == asc) { keys[i] = y; keys[l] = x; }
        }
      }
      __syncthreads();
    }
}

__device__ __forceinline__ float feat_d2(const FeatArgs& a, int i, int j) {
  const float3 p = feat_pt(a, i), q = feat_pt(a, j);
  const float dx = fsub(p.x, q.x), dy = fsub(p.y, q.y), dz = fsub(p.z, q.z);
  return fadd(fadd(fmul(dx, dx), fmul(dy, dy)), fmul(dz, dz));
}
__device__ __forceinline__ void feat_suppress(const FeatArgs& a, int ind) {          // :584-603 / :622-641
  for (int l = 1; l <= 5; ++l) { if ((double)feat_d2(a, ind + l, ind + l - 1) > 0.05) break; a.picked[ind + l] = 1; }
  for (int l = -1; l >= -5; --l) { if ((double)feat_d2(a, ind + l, ind + l + 1) > 0.05) break; a.picked[ind + l] = 1; }
}
__device__ __forceinline__ bool feat_near(const FeatArgs& a, int i) {
  const float3 p = feat_pt(a, i);
  return (double)fadd(fadd(fmul(p.x, p.x), fmul(p.y, p.y)), fmul(p.z, p.z)) < 0.25;
}

__global__ void __launch_bounds__(FEAT_T) k_feat_select(FeatArgs a) {
  __shared__ unsigned long long keys[FEAT_SECT_CAP];
  __shared__ int s_warp[FEAT_T / 32];
  __shared__ int s_base;
  const int ring = blockIdx.x;
  int ns = 0, nls = 0, nf = 0, nlf = 0;
  const int st = a.scan_start[ring], en = a.scan_end[ring];
  const bool use = !(en - st < 6 || ring % a.ds_rate != 0);
  if (use) {
    for (int j = 0; j < 6; ++j) {
      const int sp = st + (en - st) * j / 6, ep = st + (en - st) * (j + 1) / 6 - 1;
      const int len = ep - sp + 1;
      if (len > FEAT_SECT_CAP) { if (threadIdx.x == 0) atomicExch(a.err, 1); break; }
      if (len > 0) {
        for (int i = threadIdx.x; i < len; i += blockDim.x) keys[i] = ((unsigned long long)__float_as_uint(a.curv[sp + i]) << 32) | (unsigned)(sp + i);
        __syncthreads();
        block_bitonic(keys, len);
        if (threadIdx.x == 0) {
          int largest = 0;
          for (int k = len - 1; k >= 0; --k) {                                         // :557-605
            const int ind = (int)(keys[k] & 0xffffffffull);
            if (a.picked[ind] == 0 && (double)a.curv[ind] > a.edge_thres) {
              ++largest;
              if (largest <= 2) { a.label[ind] = 2; a.ring_sharp[ring * FEAT_MAX_SHARP + ns++] = ind; a.ring_less_sharp[ring * FEAT_MAX_LESS_SHARP + nls++] = ind; }
              else if (largest <= 10) { a.label[ind] = 1; a.ring_less_sharp[ring * FEAT_MAX_LESS_SHARP + nls++] = ind; }
              else break;
              a.picked[ind] = 1;
              feat_suppress(a, ind);
            }
          }
          int smallest = 0;
          for (int k = 0; k < len; ++k) {                                              // :607-643
            const int ind = (int)(keys[k] & 0xffffffffull);
            if (feat_near(a, ind)) continue;
            if (a.picked[ind] == 0 && (double)a.curv[ind] < a.surf_thres) {
              a.label[ind] = -1; a.ring_flat[ring * FEAT_MAX_FLAT + nf++] = ind;
              ++smallest;
              if (smallest >= 4) break;
              a.picked[ind] = 1;
              feat_suppress(a, ind);
            }
          }
        }
        __syncthreads();
        // less flat: the points of the sector with label <= 0 that are not within 0.5 m, in index order (:645-650)
        for (int base = 0; base < len; base += blockDim.x) {
          const int k = sp + base + threadIdx.x;
          const bool keep = (base + (int)threadIdx.x < len) && !feat_near(a, k) && a.label[k] <= 0;
          const unsigned bal = __ballot_sync(0xffffffffu, keep);
          const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
          if (lane == 0) s_warp[wid] = __popc(bal);
          __syncthreads();
          if (threadIdx.x == 0) { int acc = nlf; for (int w = 0; w < FEAT_T / 32; ++w) { const int c = s_warp[w]; s_warp[w] = acc; acc += c; } s_base = acc; }
          __syncthreads();
          if (keep) a.ring_less_flat[st + s_warp[wid] + __popc(bal & ((1u << lane) - 1u))] = k;
          nlf = s_base;
          __syncthreads();
        }
      }
    }
  }
  if (threadIdx.x == 0) {
    a.counts[0 * a.n_scans + ring] = ns; a.counts[1 * a.n_scans + ring] = nls; a.counts[2 * a.n_scans + ring] = nf; a.counts[3 * a.n_scans + ring] = nlf;
  }
}

// pcl::VoxelGrid<PointXYZI> of one ring's less-flat points (voxel_grid.hpp applyFilter, all fields averaged)
__global__ void __launch_bounds__(FEAT_T) k_feat_voxel(FeatArgs a) {
  extern __shared__ unsigned long long vkeys[];           // FEAT_RING_CAP keys
  __shared__ float s_mn[3][FEAT_T / 32], s_mx[3][FEAT_T / 32];
  __shared__ int s_cnt[FEAT_T / 32];
  __shared__ int s_total;
  const int ring = blockIdx.x;
  const int m = a.counts[3 * a.n_scans + ring];
  const int st = a.scan_start[ring];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  if (m <= 0) { if (threadIdx.x == 0) a.counts[4 * a.n_scans + ring] = 0; return; }
  if (m > FEAT_RING_CAP) { if (threadIdx.x == 0) { atomicExch(a.err, 2); a.counts[4 * a.n_scans + ring] = 0; } return; }
  const int32_t* list = a.ring_less_flat + st;
  // getMinMax3D
  float mn[3] = {3.0e38f, 3.0e38f, 3.0e38f}, mx[3] = {-3.0e38f, -3.0e38f, -3.0e38f};
  for (int i = threadIdx.x; i < m; i += blockDim.x) {
    const float3 p = feat_pt(a, list[i]);
    mn[0] = fminf(mn[0], p.x); mn[1] = fminf(mn[1], p.y); mn[2] = fminf(mn[2], p.z);
    mx[0] = fmaxf(mx[0], p.x); mx[1] = fmaxf(mx[1], p.y); mx[2] = fmaxf(mx[2], p.z);
  }
#pragma unroll
  for (int d = 0; d < 3; ++d) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) { mn[d] = fminf(mn[d], __shfl_xor_sync(0xffffffffu, mn[d], o)); mx[d] = fmaxf(mx[d], __shfl_xor_sync(0xffffffffu, mx[d], o)); }
    if (lane == 0) { s_mn[d][wid] = mn[d]; s_mx[d][wid] = mx[d]; }
  }
  __syncthreads();
#pragma unroll
  for (int d = 0; d < 3; ++d) for (int w = 0; w < FEAT_T / 32; ++w) { mn[d] = fminf(mn[d], s_mn[d][w]); mx[d] = fmaxf(mx[d], s_mx[d][w]); }
  const float inv = __fdiv_rn(1.0f, a.ds_v);
  const long long dx = (long long)fmul(fsub(mx[0], mn[0]), inv) + 1, dy = (long long)fmul(fsub(mx[1], mn[1]), inv) + 1, dz = (long long)fmul(fsub(mx[2], mn[2]), inv) + 1;
  float4* out = a.ring_ds + st;
  if (dx * dy * dz > 0x7fffffffll) {                      // PCL: leaf size too small for the cloud, the input is passed through
    for (int i = threadIdx.x; i < m; i += blockDim.x) { const float* p = a.cloud + (int64_t)list[i] * a.stride; out[i] = make_float4(p[0], p[1], p[2], p[a.ioff]); }
    if (threadIdx.x == 0) a.counts[4 * a.n_scans + ring] = m;
    return;
  }
  int min_b[3], div_b[3];
#pragma unroll
  for (int d = 0; d < 3; ++d) { min_b[d] = (int)floorf(fmul(mn[d], inv)); div_b[d] = (int)floorf(fmul(mx[d], inv)) - min_b[d] + 1; }
  const int mul1 = div_b[0], mul2 = div_b[0] * div_b[1];
  for (int i = threadIdx.x; i < m; i += blockDim.x) {
    const float3 p = feat_pt(a, list[i]);
    const int i0 = (int)fsub(floorf(fmul(p.x, inv)), (float)min_b[0]);
    const int i1 = (int)fsub(floorf(fmul(p.y, inv)), (float)min_b[1]);
    const int i2 = (int)fsub(floorf(fmul(p.z, inv)), (float)min_b[2]);
    vkeys[i] = ((unsigned long long)(unsigned)(i0 + i1 * mul1 + i2 * mul2) << 32) | (unsigned)i;     // ties by position = input order
  }
  __syncthreads();
  block_bitonic(vkeys, m);
  // one thread per voxel head: float sums in input order, divided by the float count; output in ascending voxel index
  int run = 0;
  for (int base = 0; base < m; base += blockDim.x) {
    const int i = base + threadIdx.x;
    const bool head = i < m && (i == 0 || (vkeys[i] >> 32) != (vkeys[i - 1] >> 32));
    const unsigned bal = __ballot_sync(0xffffffffu, head);
    if (lane == 0) s_cnt[wid] = __popc(bal);
    __syncthreads();
    if (threadIdx.x == 0) { int acc = run; for (int w = 0; w < FEAT_T / 32; ++w) { const int c = s_cnt[w]; s_cnt[w] = acc; acc += c; } s_total = acc; }
    __syncthreads();
    if (head) {
      const unsigned vox = (unsigned)(vkeys[i] >> 32);
      float s[4] = {0.f, 0.f, 0.f, 0.f};
      int cnt = 0;
      for (int k = i; k < m && (unsigned)(vkeys[k] >> 32) == vox; ++k) {
        const float* p = a.cloud + (int64_t)list[(int)(vkeys[k] & 0xffffffffull)] * a.stride;
        s[0] = fadd(s[0], p[0]); s[1] = fadd(s[1], p[1]); s[2] = fadd(s[2], p[2]); s[3] = fadd(s[3], p[a.ioff]);
        ++cnt;
      }
      const float c = (float)cnt;
      out[s_cnt[wid] + __popc(bal & ((1u << lane) - 1u))] = make_float4(__fdiv_rn(s[0], c), __fdiv_rn(s[1], c), __fdiv_rn(s[2], c), __fdiv_rn(s[3], c));
    }
    run = s_total;
    __syncthreads();
  }
  if (threadIdx.x == 0) a.counts[4 * a.n_scans + ring] = run;
}

__global__ void k_feat_offsets(FeatArgs a) {
  const int l = threadIdx.x;          // one thread per list (5 lists; n_scans is small)
  if (l >= 5) return;
  int acc = 0;
  for (int r = 0; r < a.n_scans; ++r) { a.offsets[l * (a.n_scans + 1) + r] = acc; acc += a.counts[l * a.n_scans + r]; }
  a.offsets[l * (a.n_scans + 1) + a.n_scans] = acc;
}

__global__ void __launch_bounds__(256) k_feat_gather(FeatArgs a) {
  const int ring = blockIdx.x, S = a.n_scans;
  const int st = a.scan_start[ring];
  const int c0 = a.counts[0 * S + ring], c1 = a.counts[1 * S + ring], c2 = a.counts[2 * S + ring], c3 = a.counts[3 * S + ring], c4 = a.counts[4 * S + ring];
  const int o0 = a.offsets[0 * (S + 1) + ring], o1 = a.offsets[1 * (S + 1) + ring], o2 = a.offsets[2 * (S + 1) + ring], o3 = a.offsets[3 * (S + 1) + ring], o4 = a.offsets[4 * (S + 1) + ring];
  for (int i = threadIdx.x; i < c0; i += blockDim.x) a.out_sharp[o0 + i] = a.ring_sharp[ring * FEAT_MAX_SHARP + i];
  for (int i = threadIdx.x; i < c1; i += blockDim.x) a.out_less_sharp[o1 + i] = a.ring_less_sharp[ring * FEAT_MAX_LESS_SHARP + i];
  for (int i = threadIdx.x; i < c2; i += blockDim.x) a.out_flat[o2 + i] = a.ring_flat[ring * FEAT_MAX_FLAT + i];
  for (int i = threadIdx.x; i < c3; i += blockDim.x) a.out_less_flat[o3 + i] = a.ring_less_flat[st + i];
  for (int i = threadIdx.x; i < c4; i += blockDim.x) a.out_ds[o4 + i] = a.ring_ds[st + i];
}

void features_run(FeatArgs& a, cudaStream_t st, LaunchCounter& lc) {
  // a function attribute belongs to one device's context: set it on every call, so whichever GPU runs this launch has it
  GLIO_CUDA_TRY(cudaFuncSetAttribute(k_feat_voxel, cudaFuncAttributeMaxDynamicSharedMemorySize, FEAT_RING_CAP * 8));
  GLIO_CUDA_TRY(cudaMemsetAsync(a.label, 0, (size_t)a.n, st));
  GLIO_CUDA_TRY(cudaMemsetAsync(a.picked, 0, (size_t)a.n, st));
  GLIO_CUDA_TRY(cudaMemsetAsync(a.err, 0, sizeof(int32_t), st));
  lc.begin("k_feat_curvature", st); k_feat_curvature<<<(unsigned)((a.n + 255) / 256), 256, 0, st>>>(a); lc.end(st);
  lc.begin("k_feat_select", st); k_feat_select<<<a.n_scans, FEAT_T, 0, st>>>(a); lc.end(st);
  lc.begin("k_feat_voxel", st); k_feat_voxel<<<a.n_scans, FEAT_T, FEAT_RING_CAP * 8, st>>>(a); lc.end(st);
  lc.begin("k_feat_offsets", st); k_feat_offsets<<<1, 32, 0, st>>>(a); lc.end(st);
  lc.begin("k_feat_gather", st); k_feat_gather<<<a.n_scans, 256, 0, st>>>(a); lc.end(st);
  GLIO_CUDA_TRY(cudaGetLastError());
}

}  // namespace glio
