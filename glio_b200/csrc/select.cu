// select.cu — the Estimator's random feature selection (Estimator.cpp:3894-4116) as a seeded sampler on the device.
//
// Every selection the reference makes (window featureSelection, batch start/end and incremental) is an ordered uniform sample
// without replacement of k positions out of 0 .. n-2 (DESIGN 2); edge lists are selected by the same rules and draws, in domains
// of their own, and a segment gathers either plane matches or edges.  Draw j of a segment takes
//   r_j = mulhi64(u_j, n-1-j),  u_j = word j % 4 of Philox4x64-10 at counter (j/4 + 1, stream, nonce, 0), key (seed, domain)
// and selects the r_j-th (0-based) value of 0 .. n-2 not chosen yet.  mulhi64 without rejection is uniform up to a relative
// bias below (n-1)/2^64 < 2^-33 for n < 2^31.  Integer arithmetic only: the result is the same bits on every device.
//
//   k_sel_sample  one warp per segment: the lanes generate 32 Philox words at a time; the rank-to-index walk keeps the chosen
//                 values sorted in shared memory (s_0 < s_1 < ...): the r-th free value is r + #{i : s_i - i <= r}, counted
//                 with ballot / popc, and it is inserted at that count.  The warp then writes the keep list (draw order) and
//                 gathers the selected records into the selection buffers the evaluation reads.
#include "common.cuh"

namespace glio {

namespace {

constexpr uint64_t kPhiloxM0 = 0xD2E7470EE14C6C93ull, kPhiloxM1 = 0xCA5A826395121157ull;
constexpr uint64_t kPhiloxW0 = 0x9E3779B97F4A7C15ull, kPhiloxW1 = 0xBB67AE8584CAA73Bull;

// word w (0..3) of philox4x64_R(10, ctr, key) (Random123; numpy.random.Philox)
__device__ __forceinline__ uint64_t philox_word(uint64_t c0, uint64_t c1, uint64_t c2, uint64_t c3, uint64_t k0, uint64_t k1, int w) {
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    if (r) { k0 += kPhiloxW0; k1 += kPhiloxW1; }
    const uint64_t h0 = __umul64hi(kPhiloxM0, c0), l0 = kPhiloxM0 * c0;
    const uint64_t h1 = __umul64hi(kPhiloxM1, c2), l1 = kPhiloxM1 * c2;
    c0 = h1 ^ c1 ^ k0; c1 = l1; c2 = h0 ^ c3 ^ k1; c3 = l0;
  }
  return w == 0 ? c0 : w == 1 ? c1 : w == 2 ? c2 : c3;
}

__global__ void __launch_bounds__(32) k_sel_sample(const SelSeg* __restrict__ segs, uint64_t seed, uint64_t domain, uint64_t nonce) {
  extern __shared__ int32_t s_sorted[];          // the chosen values, ascending (k of the launch's largest segment)
  const SelSeg sg = segs[blockIdx.x];
  const int lane = threadIdx.x;
  const int k = sg.k;
  const uint64_t stream = sg.stream;
  int m = 0;                                     // values chosen so far
  for (int base = 0; base < k; base += 32) {
    const int j = base + lane;
    uint64_t r = 0;
    if (j < k) {
      const uint64_t u = philox_word((uint64_t)(j / 4) + 1, stream, nonce, 0, seed, domain, j & 3);
      r = __umul64hi(u, (uint64_t)(sg.n - 1 - j));
    }
    const int cnt = min(32, k - base);
    for (int t = 0; t < cnt; ++t) {
      const int64_t rj = (int64_t)__shfl_sync(0xffffffffu, (unsigned long long)r, t);
      // pos = #{i < m : s_i - i <= rj}; s_i - i is non-decreasing, so those i are a prefix and the new value goes there
      int pos = 0;
      for (int c = 0; c < m; c += 32) {
        const int i = c + lane;
        const bool le = i < m && (int64_t)s_sorted[i] - i <= rj;
        pos += __popc(__ballot_sync(0xffffffffu, le));
      }
      const int32_t v = (int32_t)(rj + pos);
      // shift s[pos .. m) up by one, from the top chunk down (each chunk is read before its upper neighbour is overwritten)
      for (int c = ((m - pos + 31) / 32 - 1) * 32; c >= 0; c -= 32) {
        const int i = pos + c + lane;
        const int32_t x = i < m ? s_sorted[i] : 0;
        __syncwarp();
        if (i < m) s_sorted[i + 1] = x;
        __syncwarp();
      }
      if (lane == 0) { s_sorted[pos] = v; sg.keep[base + t] = v; }
      __syncwarp();
      ++m;
    }
  }
  __syncwarp();                                  // orders lane 0's keep writes before the other lanes read them
  for (int j = lane; j < k; j += 32) {
    const int64_t src = sg.keep[j];
    sg.o_cpw[j] = sg.cpw[src];
    if (sg.nsd) sg.o_nsd[j] = sg.nsd[src];
    if (sg.nc) {
#pragma unroll
      for (int c = 0; c < 6; ++c) sg.o_nc[6 * (int64_t)j + c] = sg.nc[6 * src + c];
    }
    if (sg.pa) { sg.o_pa[j] = sg.pa[src]; sg.o_pb[j] = sg.pb[src]; }
  }
}

}  // namespace

void select_sample_run(const SelSeg* d_segs, int nseg, int k_max, uint64_t seed, uint64_t domain, uint64_t nonce, cudaStream_t st,
                       LaunchCounter& lc) {
  if (nseg <= 0) return;
  lc.begin("k_sel_sample", st);
  k_sel_sample<<<nseg, 32, (size_t)(k_max + 1) * sizeof(int32_t), st>>>(d_segs, seed, domain, nonce);
  lc.end(st);
  GLIO_CUDA_TRY(cudaGetLastError());
}

}  // namespace glio
