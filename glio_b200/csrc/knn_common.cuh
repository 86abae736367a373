// knn_common.cuh — the pieces of the K1a box search (assoc.cu k_knn_box): the top-5 register list, the search arguments
// and the per-thread scanning helpers.  loop.cu shares the (distance, index) key.
#pragma once
#include "common.cuh"
#include "devmath.cuh"

namespace glio {

// ---- top-5 by (distance, index) -------------------------------------------------------------------
// One 64-bit key per neighbour: (bits of the non-negative float distance) << 32 | index.  Unsigned key order ==
// lexicographic (distance, index) order, so ties are broken by index exactly like a stable sort by (distance, index).
struct Top5 {
  unsigned long long k0, k1, k2, k3, k4;
};
__device__ __forceinline__ unsigned long long make_key(float d, int id) { return ((unsigned long long)__float_as_uint(d) << 32) | (unsigned int)id; }
__device__ __forceinline__ float key_dist(unsigned long long k) { return __uint_as_float((unsigned int)(k >> 32)); }
__device__ __forceinline__ int key_idx(unsigned long long k) { return (int)(unsigned int)(k & 0xffffffffull); }
constexpr unsigned long long KEY_EMPTY = 0x7f8000007fffffffull;   // (+inf, INT_MAX)
__device__ __forceinline__ void top5_init(Top5& t) { t.k0 = t.k1 = t.k2 = t.k3 = t.k4 = KEY_EMPTY; }
// compare-exchange of two keys: one 64-bit compare + select for the smaller key, the larger one by XOR (the plain
// two-select form made ptxas emit a second, mirrored compare: 8 instead of 6 instructions per exchange in the hottest
// block of K1a)
__device__ __forceinline__ void key_cswap(unsigned long long& a, unsigned long long& b) {
  const unsigned long long lo = a < b ? a : b;
  b = a ^ b ^ lo;
  a = lo;
}
#define GLIO_KSWAP(A, B) key_cswap((A), (B));
__device__ __forceinline__ void top5_push(Top5& t, float d, int id) {
  const unsigned long long k = make_key(d, id);
  if (k < t.k4) {
    t.k4 = k;
    GLIO_KSWAP(t.k3, t.k4)
    GLIO_KSWAP(t.k2, t.k3)
    GLIO_KSWAP(t.k1, t.k2)
    GLIO_KSWAP(t.k0, t.k1)
  }
}

struct SearchArgs {
  GridDesc grid;
  int64_t Qt;
  const float4* pm;     // transformed queries, scan order
  const float4* pmq;    // the same in cell-sorted order, .w = bitcast scan index (k_order_scatter)
  float gate_sq;
  int32_t* knn_idx;     // [5][Qt] sorted order
  float* knn_sqd;       // [5][Qt] sorted order; rows 0..3 are written only when store_all_sqd (the gate needs the 5th only)
  bool store_all_sqd;
};

__device__ __forceinline__ void store_top5(const SearchArgs& a, int64_t p, const Top5& t) {
  a.knn_idx[0 * a.Qt + p] = key_idx(t.k0); a.knn_idx[1 * a.Qt + p] = key_idx(t.k1); a.knn_idx[2 * a.Qt + p] = key_idx(t.k2);
  a.knn_idx[3 * a.Qt + p] = key_idx(t.k3); a.knn_idx[4 * a.Qt + p] = key_idx(t.k4);
  a.knn_sqd[4 * a.Qt + p] = key_dist(t.k4);
  if (a.store_all_sqd) {
    a.knn_sqd[0 * a.Qt + p] = key_dist(t.k0); a.knn_sqd[1 * a.Qt + p] = key_dist(t.k1); a.knn_sqd[2 * a.Qt + p] = key_dist(t.k2);
    a.knn_sqd[3 * a.Qt + p] = key_dist(t.k3);
  }
}


// ---- per-thread scanning helpers of the box search
__device__ __forceinline__ void scan_range_keys(const float4* __restrict__ pts, int s, int e, float qx, float qy, float qz, Top5& t, float& d4f) {
  for (int k = s; k < e; ++k) {
    const float4 p = __ldg(&pts[k]);
    const float d = l2_simple(qx, qy, qz, p.x, p.y, p.z);
    if (d <= d4f) {                                  // cheap float test first; ties on distance resolved on the full key
      const unsigned long long key = make_key(d, __float_as_int(p.w));
      if (key < t.k4) { t.k4 = key; GLIO_KSWAP(t.k3, t.k4) GLIO_KSWAP(t.k2, t.k3) GLIO_KSWAP(t.k1, t.k2) GLIO_KSWAP(t.k0, t.k1) d4f = key_dist(t.k4); }
    }
  }
}

// the 3x3x3 start box around the query's cell (cx, cy, cz): fetch the bounds of all nine rows up front (18 independent
// loads in flight instead of nine dependent load -> scan steps), park them in this thread's shared-memory column, then
// scan the query's own row first so the 5th distance tightens early
__device__ __forceinline__ void scan_start_box(const GridDesc& g, float qx, float qy, float qz, int cx, int cy, int cz, Top5& t, float& d4f,
                                               int* __restrict__ sb) {
  const int* __restrict__ cs = g.cell_start;
  const int x0 = max(cx - 1, 0), x1 = min(cx + 1, g.nx - 1);
#pragma unroll
  for (int i = 0; i < 9; ++i) {
    const int z = cz + i / 3 - 1, y = cy + i % 3 - 1;
    int s = 0, e = 0;
    if (z >= 0 && z < g.nz && y >= 0 && y < g.ny && x0 <= x1) { const int row = (z * g.ny + y) * g.nx; s = __ldg(&cs[row + x0]); e = __ldg(&cs[row + x1 + 1]); }
    sb[(2 * i) * 128] = s; sb[(2 * i + 1) * 128] = e;
  }
#pragma unroll 1
  for (int i = 0; i < 9; ++i) {
    const int o = (int)((0x862053714ull >> (4 * i)) & 15ull);     // 4,1,7,3,5,0,2,6,8
    scan_range_keys(g.pts, sb[(2 * o) * 128], sb[(2 * o + 1) * 128], qx, qy, qz, t, d4f);
  }
}

// The slab scan of the growth phase, built for the queries that have to look far (sparse map around them, most
// rows empty): (1) a row whose cells are provably farther than the current 5th distance is skipped without touching memory -
// the same margins as the face test, strict inequality, so nothing that could enter the top-5 (ties included) is skipped;
// (2) the bounds of up to eight surviving rows are fetched together (18 independent loads in flight) and parked in the thread's
// shared-memory column before the rows are scanned: the chain of dependent loads per slab shrinks ~9x.
__device__ __forceinline__ float axis_gap(float q, float lo, float hi, float slack) {
  const float d = fmaxf(lo - q, q - hi);                   // > 0 outside [lo, hi]
  const float m = d * 0.999f - slack;
  return m > 0.f ? m : 0.f;
}
__device__ __forceinline__ void scan_rows_batched(const GridDesc& g, int x0, int x1, int y0, int y1, int z0, int z1, float qx, float qy, float qz, Top5& t, float& d4f,
                                                  int* __restrict__ sb) {
  x0 = max(x0, 0); x1 = min(x1, g.nx - 1); y0 = max(y0, 0); y1 = min(y1, g.ny - 1); z0 = max(z0, 0); z1 = min(z1, g.nz - 1);
  if (x0 > x1 || y0 > y1 || z0 > z1) return;
  const int* __restrict__ cs = g.cell_start;
  const float gx = axis_gap(qx, g.ox + (float)x0 * g.cell, g.ox + (float)(x1 + 1) * g.cell, g.slack);
  const float gx2 = gx * gx;
  const int dx1 = x1 + 1 - x0;
  constexpr int NB = 8;
  int y = y0, z = z0;
  bool more = true;
  while (more) {
    // (a) pick the next rows that survive the distance test: pure arithmetic, their first-cell offsets go to shared memory
    int nb = 0;
#pragma unroll 1
    while (nb < NB && more) {
      const float gy = axis_gap(qy, g.oy + (float)y * g.cell, g.oy + (float)(y + 1) * g.cell, g.slack);
      const float gz = axis_gap(qz, g.oz + (float)z * g.cell, g.oz + (float)(z + 1) * g.cell, g.slack);
      if (!(d4f <= gx2 + gy * gy + gz * gz)) { sb[(2 * nb) * 128] = (z * g.ny + y) * g.nx + x0; ++nb; }
      if (++y > y1) { y = y0; if (++z > z1) more = false; }
    }
    // (b) all their bounds in flight together, then parked next to the offsets
    int bs[NB], be[NB];
#pragma unroll
    for (int i = 0; i < NB; ++i) {
      bs[i] = 0; be[i] = 0;
      if (i < nb) { const int o = sb[(2 * i) * 128]; bs[i] = __ldg(&cs[o]); be[i] = __ldg(&cs[o + dx1]); }
    }
#pragma unroll
    for (int i = 0; i < NB; ++i) { sb[(2 * i) * 128] = bs[i]; sb[(2 * i + 1) * 128] = be[i]; }
    // (c) scan
#pragma unroll 1
    for (int i = 0; i < nb; ++i) scan_range_keys(g.pts, sb[(2 * i) * 128], sb[(2 * i + 1) * 128], qx, qy, qz, t, d4f);
  }
}

// one face test of the box growth: does something nearer than the current 5th distance possibly hide beyond face f?
__device__ __forceinline__ bool box_face_open(const GridDesc& g, int f, float qx, float qy, float qz, float gate_r, int lx, int hx, int ly, int hy, int lz, int hz,
                                              const Top5& t) {
  const int ax = f >> 1;
  const bool up = (f & 1) != 0;
  const int lo = ax == 0 ? lx : (ax == 1 ? ly : lz), hi = ax == 0 ? hx : (ax == 1 ? hy : hz), n = ax == 0 ? g.nx : (ax == 1 ? g.ny : g.nz);
  const float qa = ax == 0 ? qx : (ax == 1 ? qy : qz), oa = ax == 0 ? g.ox : (ax == 1 ? g.oy : g.oz);
  if (up ? (hi >= n - 1) : (lo <= 0)) return false;                   // nothing beyond this face
  const float b = up ? (oa + (float)(hi + 1) * g.cell) - qa : qa - (oa + (float)lo * g.cell);
  const float bs = b * 0.999f - g.slack;                              // GridDesc::slack
  if (bs >= gate_r) return false;                                     // beyond the gate radius
  if (bs > 0.f && key_dist(t.k4) <= bs * bs) return false;            // the 5th distance is inside this face
  return true;
}
// face-by-face growth of the searched box [lx,hx] x [ly,hy] x [lz,hz] until no face is open (see k_knn_box)
__device__ __forceinline__ void box_grow(const GridDesc& g, float qx, float qy, float qz, float gate_r, int rmax, int lx, int hx, int ly, int hy, int lz, int hz,
                                         Top5& t, float& d4f, int* __restrict__ sb) {
  for (int round = 0; round < rmax + 3; ++round) {
    bool any = false;
#pragma unroll 1
    for (int f = 0; f < 6; ++f) {
      if (!box_face_open(g, f, qx, qy, qz, gate_r, lx, hx, ly, hy, lz, hz, t)) continue;
      const int ax = f >> 1;
      const bool up = (f & 1) != 0;
      const int hi = ax == 0 ? hx : (ax == 1 ? hy : hz), lo = ax == 0 ? lx : (ax == 1 ? ly : lz);
      const int nc = up ? hi + 1 : lo - 1;
      int bx0 = lx, bx1 = hx, by0 = ly, by1 = hy, bz0 = lz, bz1 = hz;
      if (ax == 0) { bx0 = bx1 = nc; if (up) hx = nc; else lx = nc; }
      else if (ax == 1) { by0 = by1 = nc; if (up) hy = nc; else ly = nc; }
      else { bz0 = bz1 = nc; if (up) hz = nc; else lz = nc; }
      scan_rows_batched(g, bx0, bx1, by0, by1, bz0, bz1, qx, qy, qz, t, d4f, sb);
      any = true;
    }
    if (!any) break;
  }
}

}  // namespace glio
