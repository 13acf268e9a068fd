// GeoGuessr evaluation metrics of reference evaluation/metrics.py (compute_geoguessr_metrics, :139-202):
//   - a country index over Polygon / MultiPolygon geometries and a locate kernel that gives each label point its
//     country (find_country, :59-72) and tells whether that country contains the prediction (country_accuracy, :74-88);
//   - one fused pass over the samples for haversine_np, the Under_*_km counts, the GeoGuessr score and the geocell
//     top-1 / top-k hits, plus the median km error by exact selection (radix_select.cuh).
//
// Geometry semantics are GEOS's in the plane of (lng, lat) degrees, as shapely evaluates them (DESIGN.md §1):
//   - boundary: the point lies exactly on an edge of a ring; covered: boundary, or an odd ray-crossing count over the
//     shell and holes of some part; contains: covered and not boundary.  The crossing rule is GEOS RayCrossingCounter's,
//     with an exact orientation sign (fp64 filter, then an exact expansion sum).
//   - a label covered by no geometry takes the nearest one by GEOS Distance::pointToSegment, lowest index on ties.
//
// Country index, built on the device: per-part and per-geometry bounding boxes, and per part a set of latitude bands of
// equal height (about EDGES_PER_BAND edges each); every edge is listed in each band its latitude range touches, in edge
// order (count, scan, then a stable warp-per-part scatter).  band_of() is monotone in y, so an edge whose latitude range
// holds y is always listed in band_of(y): the locate kernel scans one band per part instead of the whole ring.
// No float atomics anywhere: every result, and every byte of the index, is deterministic.
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

#include "../../include/pigeon_b200.h"
#include "radix_select.cuh"
#include "tma_host.h"

namespace pg {
namespace {

constexpr int EDGES_PER_BAND = 16;
constexpr int MAX_BANDS_PER_PART = 1 << 16;
constexpr int LOCATE_THREADS = 128;
constexpr int METRIC_THREADS = 256;
constexpr int SELECT_THREADS = 1024;
constexpr int NUM_KM = 10;
__constant__ double KM_THRESHOLDS[NUM_KM] = {1, 5, 10, 25, 50, 100, 200, 750, 1000, 2500};

__host__ __device__ constexpr size_t align256(size_t x) { return (x + 255) & ~size_t(255); }

// Index layout.  T (total bands) is only known on the device, so band arrays take its upper bound V / EDGES_PER_BAND + P.
struct Index {
  double *part_box, *geom_box;  // [P, 4], [G, 4]: xmin, ymin, xmax, ymax
  double* part_band;            // [P, 2]: y0, bands per degree
  int32_t* part_nb;             // [P] bands in the part
  int64_t* part_band_base;      // [P + 1] first band of the part
  int64_t* band_off;            // [Tmax + 1] first entry of each band
  int64_t* band_cur;            // [Tmax] scatter cursors (build only)
  double* meta;                 // [1]: max |coordinate| over all vertices
};

size_t index_layout(int64_t V, int64_t P, int64_t G, char* base, Index* ix) {
  size_t off = 0;
  auto take = [&](size_t bytes) {
    char* p = base ? base + off : nullptr;
    off += align256(bytes);
    return p;
  };
  const int64_t tmax = V / EDGES_PER_BAND + P + 1;
  Index t;
  t.part_box = (double*)take(32 * size_t(P));
  t.geom_box = (double*)take(32 * size_t(G));
  t.part_band = (double*)take(16 * size_t(P));
  t.part_nb = (int32_t*)take(4 * size_t(P));
  t.part_band_base = (int64_t*)take(8 * size_t(P + 1));
  t.band_off = (int64_t*)take(8 * size_t(tmax + 1));
  t.band_cur = (int64_t*)take(8 * size_t(tmax));
  t.meta = (double*)take(16);
  if (ix) *ix = t;
  return off;
}

struct Geo {
  const double* v;  // [V, 2]
  const int64_t *ring_off, *part_ring_off, *geom_part_off;
  int64_t V, R, P, G;
};

__device__ __forceinline__ int band_of(double y, double y0, double per_deg, int nb) {
  const double t = __dmul_rn(__dsub_rn(y, y0), per_deg);  // both roundings are monotone in y
  return t <= 0.0 ? 0 : (t >= double(nb - 1) ? nb - 1 : int(t));
}

// ---------------------------------------------------------------------------------------------------------- build
// One CTA per part: bounding box of its vertices (the part's rings are contiguous), its edge count and band layout.
__global__ void part_kernel(Geo g, Index ix) {
  __shared__ double red[4][32];
  const int64_t p = blockIdx.x;
  const int64_t r0 = g.part_ring_off[p], r1 = g.part_ring_off[p + 1];
  const int64_t v0 = g.ring_off[r0], v1 = g.ring_off[r1];
  double b[4] = {INFINITY, INFINITY, -INFINITY, -INFINITY};
  for (int64_t i = v0 + threadIdx.x; i < v1; i += blockDim.x) {
    const double x = g.v[2 * i], y = g.v[2 * i + 1];
    b[0] = fmin(b[0], x); b[1] = fmin(b[1], y); b[2] = fmax(b[2], x); b[3] = fmax(b[3], y);
  }
  for (int o = 16; o > 0; o >>= 1) {
    b[0] = fmin(b[0], __shfl_xor_sync(0xffffffffu, b[0], o));
    b[1] = fmin(b[1], __shfl_xor_sync(0xffffffffu, b[1], o));
    b[2] = fmax(b[2], __shfl_xor_sync(0xffffffffu, b[2], o));
    b[3] = fmax(b[3], __shfl_xor_sync(0xffffffffu, b[3], o));
  }
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
  if (lane == 0) for (int c = 0; c < 4; ++c) red[c][warp] = b[c];
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int w = 1; w < nw; ++w) {
      b[0] = fmin(b[0], red[0][w]); b[1] = fmin(b[1], red[1][w]); b[2] = fmax(b[2], red[2][w]); b[3] = fmax(b[3], red[3][w]);
    }
    for (int c = 0; c < 4; ++c) ix.part_box[4 * p + c] = b[c];
    const int64_t edges = (v1 - v0) - (r1 - r0);
    int64_t nb = (edges + EDGES_PER_BAND - 1) / EDGES_PER_BAND;
    nb = nb < 1 ? 1 : (nb > MAX_BANDS_PER_PART ? MAX_BANDS_PER_PART : nb);
    const double h = __dsub_rn(b[3], b[1]);
    ix.part_nb[p] = int32_t(h > 0.0 ? nb : 1);
    ix.part_band[2 * p] = b[1];
    ix.part_band[2 * p + 1] = h > 0.0 ? __ddiv_rn(double(nb), h) : 0.0;
  }
}

// One CTA: geometry boxes, the exclusive scan of bands per part, the largest |coordinate| and zeroed band counts.
__global__ void layout_kernel(Geo g, Index ix) {
  const int tid = threadIdx.x;
  double mx = 0.0;
  for (int64_t q = tid; q < g.G; q += blockDim.x) {
    double b[4] = {INFINITY, INFINITY, -INFINITY, -INFINITY};
    for (int64_t p = g.geom_part_off[q]; p < g.geom_part_off[q + 1]; ++p) {
      b[0] = fmin(b[0], ix.part_box[4 * p]); b[1] = fmin(b[1], ix.part_box[4 * p + 1]);
      b[2] = fmax(b[2], ix.part_box[4 * p + 2]); b[3] = fmax(b[3], ix.part_box[4 * p + 3]);
    }
    for (int c = 0; c < 4; ++c) { ix.geom_box[4 * q + c] = b[c]; mx = fmax(mx, fabs(b[c])); }
  }
  __shared__ double s_mx[1024];
  s_mx[tid] = mx;
  __syncthreads();
  if (tid == 0) {
    for (int t = 1; t < blockDim.x; ++t) mx = fmax(mx, s_mx[t]);
    ix.meta[0] = mx;
    int64_t acc = 0;
    for (int64_t p = 0; p < g.P; ++p) { ix.part_band_base[p] = acc; acc += ix.part_nb[p]; }
    ix.part_band_base[g.P] = acc;
  }
  __syncthreads();
  const int64_t T = ix.part_band_base[g.P];
  for (int64_t t = tid; t <= T; t += blockDim.x) ix.band_off[t] = 0;
}

__device__ __forceinline__ int64_t upper_index(const int64_t* off, int64_t n, int64_t i) {
  int64_t lo = 0, hi = n;  // largest r with off[r] <= i
  while (hi - lo > 1) {
    const int64_t mid = (lo + hi) >> 1;
    if (off[mid] <= i) lo = mid; else hi = mid;
  }
  return lo;
}

// Bands [b0, b1] of the part that edge (i, i + 1) touches.
__device__ __forceinline__ void edge_bands(const Geo& g, const Index& ix, int64_t p, int64_t i, int* b0, int* b1) {
  const double ya = g.v[2 * i + 1], yb = g.v[2 * i + 3];
  const double y0 = ix.part_band[2 * p], per = ix.part_band[2 * p + 1];
  const int nb = ix.part_nb[p];
  *b0 = band_of(fmin(ya, yb), y0, per, nb);
  *b1 = band_of(fmax(ya, yb), y0, per, nb);
}

// One thread per vertex that starts an edge: count its entries per band (integer atomics: exact).
__global__ void count_kernel(Geo g, Index ix) {
  const int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= g.V) return;
  const int64_t r = upper_index(g.ring_off, g.R + 1, i);
  if (i + 1 >= g.ring_off[r + 1]) return;  // the closing vertex starts no edge
  const int64_t p = upper_index(g.part_ring_off, g.P + 1, r);
  int b0, b1;
  edge_bands(g, ix, p, i, &b0, &b1);
  const int64_t base = ix.part_band_base[p];
  for (int b = b0; b <= b1; ++b) atomicAdd(reinterpret_cast<unsigned long long*>(&ix.band_off[base + b + 1]), 1ull);
}

// One CTA: inclusive scan of the counts into band offsets, and the entry total.
__global__ void scan_kernel(Geo g, Index ix, int64_t* num_entries_out) {
  __shared__ int64_t s[1024];
  const int64_t T = ix.part_band_base[g.P];
  int64_t carry = 0;
  for (int64_t c0 = 1; c0 <= T; c0 += blockDim.x) {
    const int64_t t = c0 + threadIdx.x;
    int64_t v = t <= T ? ix.band_off[t] : 0;
    s[threadIdx.x] = v;
    __syncthreads();
    for (int o = 1; o < blockDim.x; o <<= 1) {
      const int64_t y = threadIdx.x >= o ? s[threadIdx.x - o] : 0;
      __syncthreads();
      s[threadIdx.x] += y;
      __syncthreads();
    }
    if (t <= T) { ix.band_off[t] = carry + s[threadIdx.x]; ix.band_cur[t - 1] = carry + s[threadIdx.x] - v; }
    carry += s[blockDim.x - 1];
    __syncthreads();
  }
  if (threadIdx.x == 0 && num_entries_out) *num_entries_out = carry;
}

// One warp per part, edges in order, 32 at a time: for each band an edge touches, lanes that write the same band rank
// themselves by lane (match_any), so each band lists its edges in edge order whatever the scheduling.
__global__ void fill_kernel(Geo g, Index ix, int32_t* __restrict__ entries) {
  const int64_t p = (int64_t(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (p >= g.P) return;
  const int64_t r0 = g.part_ring_off[p], r1 = g.part_ring_off[p + 1];
  const int64_t v0 = g.ring_off[r0], v1 = g.ring_off[r1];
  const int64_t base = ix.part_band_base[p];
  int64_t r = r0;
  for (int64_t c = v0; c < v1; c += 32) {
    const int64_t i = c + lane;
    bool edge = false;
    int b0 = 0, b1 = -1;
    if (i < v1) {
      while (g.ring_off[r + 1] <= i) ++r;
      edge = i + 1 < g.ring_off[r + 1];
      if (edge) edge_bands(g, ix, p, i, &b0, &b1);
    }
    int span = b1 - b0 + 1, max_span = span;
    for (int o = 16; o > 0; o >>= 1) max_span = max(max_span, __shfl_xor_sync(0xffffffffu, max_span, o));
    for (int t = 0; t < max_span; ++t) {
      const int key = t < span ? b0 + t : -1;
      const unsigned peers = __match_any_sync(0xffffffffu, key);
      if (key >= 0) {
        const int64_t cur = ix.band_cur[base + key];
        entries[cur + __popc(peers & ((1u << lane) - 1))] = int32_t(i);
        __syncwarp(peers);
        if (lane == 31 - __clz(peers)) ix.band_cur[base + key] = cur + __popc(peers);
      }
      __syncwarp();
    }
  }
}

// ---------------------------------------------------------------------------------------------------------- locate
__device__ __forceinline__ void two_sum(double a, double b, double* s, double* e) {
  const double x = __dadd_rn(a, b), bv = __dsub_rn(x, a), av = __dsub_rn(x, bv);
  *s = x;
  *e = __dadd_rn(__dsub_rn(a, av), __dsub_rn(b, bv));
}
__device__ __forceinline__ void two_diff(double a, double b, double* s, double* e) { two_sum(a, -b, s, e); }
__device__ __forceinline__ void two_prod(double a, double b, double* p, double* e) {
  *p = __dmul_rn(a, b);
  *e = __fma_rn(a, b, -*p);
}

// Sign of the exact (a - c) x (b - c), i.e. of GEOS Orientation::index(a, b, c): Shewchuk's orient2d filter, then the
// exact sum of the 16 product terms as a nonoverlapping expansion (Grow-Expansion with zero elimination).  Exact for
// all finite inputs whose products do not underflow (|terms| above 2^-969).
__device__ __noinline__ int orient_exact(double ax, double ay, double bx, double by, double cx, double cy) {
  double acx, acx_e, acy, acy_e, bcx, bcx_e, bcy, bcy_e;
  two_diff(ax, cx, &acx, &acx_e); two_diff(ay, cy, &acy, &acy_e);
  two_diff(bx, cx, &bcx, &bcx_e); two_diff(by, cy, &bcy, &bcy_e);
  const double l[2] = {acx, acx_e}, lr[2] = {bcy, bcy_e}, r[2] = {acy, acy_e}, rr[2] = {bcx, bcx_e};
  double terms[16];
  int n = 0;
  for (int u = 0; u < 2; ++u)
    for (int w = 0; w < 2; ++w) {
      two_prod(l[u], lr[w], &terms[n], &terms[n + 1]);
      two_prod(r[u], rr[w], &terms[n + 2], &terms[n + 3]);
      terms[n + 2] = -terms[n + 2];
      terms[n + 3] = -terms[n + 3];
      n += 4;
    }
  double e[17];
  int m = 0;
  for (int t = 0; t < 16; ++t) {
    double q = terms[t];
    int k = 0;
    for (int j = 0; j < m; ++j) {
      double s, h;
      two_sum(q, e[j], &s, &h);
      q = s;
      if (h != 0.0) e[k++] = h;
    }
    if (q != 0.0) e[k++] = q;
    m = k;
  }
  return m == 0 ? 0 : (e[m - 1] > 0.0 ? 1 : -1);
}

__device__ __forceinline__ int orient(double ax, double ay, double bx, double by, double cx, double cy) {
  const double detleft = __dmul_rn(__dsub_rn(ax, cx), __dsub_rn(by, cy));
  const double detright = __dmul_rn(__dsub_rn(ay, cy), __dsub_rn(bx, cx));
  const double det = __dsub_rn(detleft, detright);
  double detsum;
  if (detleft > 0.0) {
    if (detright <= 0.0) return det > 0.0 ? 1 : (det < 0.0 ? -1 : 0);
    detsum = __dadd_rn(detleft, detright);
  } else if (detleft < 0.0) {
    if (detright >= 0.0) return det > 0.0 ? 1 : (det < 0.0 ? -1 : 0);
    detsum = __dsub_rn(-detleft, detright);
  } else {
    return det > 0.0 ? 1 : (det < 0.0 ? -1 : 0);
  }
  const double errbound = __dmul_rn(3.3306690738754716e-16, detsum);  // (3 + 16 eps) eps, eps = 2^-53
  if (det >= errbound || -det >= errbound) return det > 0.0 ? 1 : -1;
  return orient_exact(ax, ay, bx, by, cx, cy);
}

// GEOS RayCrossingCounter::countSegment for edge p1 -> p2 and point (x, y).
__device__ __forceinline__ void count_segment(double x1, double y1, double x2, double y2, double x, double y,
                                              int* crossings, bool* on_boundary) {
  if (x1 < x && x2 < x) return;
  if (x == x2 && y == y2) { *on_boundary = true; return; }
  if (y1 == y && y2 == y) {
    const double mn = fmin(x1, x2), mx = fmax(x1, x2);
    if (x >= mn && x <= mx) *on_boundary = true;
    return;
  }
  if ((y1 > y && y2 <= y) || (y2 > y && y1 <= y)) {
    int o = orient(x1, y1, x2, y2, x, y);
    if (o == 0) { *on_boundary = true; return; }
    if (y2 < y1) o = -o;
    if (o > 0) ++*crossings;
  }
}

__device__ __forceinline__ bool in_box(const double* b, double x, double y) {
  return x >= b[0] && x <= b[2] && y >= b[1] && y <= b[3];
}

// Location of (x, y) against geometry q: returns covered; *boundary is set when it lies on an edge of any ring.
__device__ bool locate_in(const Geo& g, const Index& ix, const int32_t* __restrict__ entries, int64_t q, double x,
                          double y, bool* boundary) {
  bool inside = false, bnd = false;
  if (in_box(ix.geom_box + 4 * q, x, y)) {
    for (int64_t p = g.geom_part_off[q]; p < g.geom_part_off[q + 1] && !bnd; ++p) {
      if (!in_box(ix.part_box + 4 * p, x, y)) continue;
      const int64_t band = ix.part_band_base[p] + band_of(y, ix.part_band[2 * p], ix.part_band[2 * p + 1], ix.part_nb[p]);
      int crossings = 0;
      for (int64_t e = ix.band_off[band]; e < ix.band_off[band + 1] && !bnd; ++e) {
        const int64_t i = entries[e];
        count_segment(g.v[2 * i], g.v[2 * i + 1], g.v[2 * i + 2], g.v[2 * i + 3], x, y, &crossings, &bnd);
      }
      inside |= (crossings & 1) != 0;
    }
  }
  *boundary = bnd;
  return bnd || inside;
}

__device__ __forceinline__ double point_dist(double px, double py, double ax, double ay) {
  const double dx = __dsub_rn(px, ax), dy = __dsub_rn(py, ay);
  return __dsqrt_rn(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)));
}

// GEOS Distance::pointToSegment, same operation order, no contraction.
__device__ __forceinline__ double point_to_segment(double px, double py, double ax, double ay, double bx, double by) {
  if (ax == bx && ay == by) return point_dist(px, py, ax, ay);
  const double dx = __dsub_rn(bx, ax), dy = __dsub_rn(by, ay);
  const double len2 = __dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy));
  const double r = __ddiv_rn(__dadd_rn(__dmul_rn(__dsub_rn(px, ax), dx), __dmul_rn(__dsub_rn(py, ay), dy)), len2);
  if (r <= 0.0) return point_dist(px, py, ax, ay);
  if (r >= 1.0) return point_dist(px, py, bx, by);
  const double s = __ddiv_rn(__dsub_rn(__dmul_rn(__dsub_rn(ay, py), dx), __dmul_rn(__dsub_rn(ax, px), dy)), len2);
  return __dmul_rn(fabs(s), __dsqrt_rn(len2));
}

// Euclidean distance from (x, y) to a box (0 inside).
__device__ __forceinline__ double box_dist(const double* b, double x, double y) {
  const double dx = fmax(fmax(b[0] - x, x - b[2]), 0.0), dy = fmax(fmax(b[1] - y, y - b[3]), 0.0);
  return sqrt(dx * dx + dy * dy);
}

__device__ __forceinline__ double warp_min(double v) {
  for (int o = 16; o > 0; o >>= 1) v = fmin(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// One warp per sample whose label no geometry covers: the nearest geometry by the least pointToSegment value over its
// edges, lowest index on exact ties, and whether it contains the prediction.  A part is skipped only when its box lies
// farther than the best value so far plus `slack`, a bound far above the rounding error of either distance, so the
// skipped edges can never attain the minimum; of the others, only the bands within that distance of the label's
// latitude are scanned, the lanes striding over their entries (fmin is exact, so the lane split does not matter).
__global__ void nearest_kernel(Geo g, Index ix, const int32_t* __restrict__ entries, const double* __restrict__ label,
                               const double* __restrict__ pred, int64_t N, int32_t* __restrict__ country,
                               const uint8_t* __restrict__ flags, uint8_t* __restrict__ pred_inside) {
  const int64_t n = (int64_t(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (n >= N || flags[n] == 0) return;
  const double x = label[2 * n], y = label[2 * n + 1];
  const double slack = 1e-12 * (ix.meta[0] + fabs(x) + fabs(y)) + 1e-300;
  double bound = INFINITY;  // an upper bound: the first edge of every geometry
  for (int64_t q = lane; q < g.G; q += 32) {
    const int64_t i = g.ring_off[g.part_ring_off[g.geom_part_off[q]]];
    bound = fmin(bound, point_to_segment(x, y, g.v[2 * i], g.v[2 * i + 1], g.v[2 * i + 2], g.v[2 * i + 3]));
  }
  bound = warp_min(bound);
  double best = INFINITY;
  int32_t best_q = 0;
  for (int64_t q = 0; q < g.G; ++q) {
    if (box_dist(ix.geom_box + 4 * q, x, y) > fmin(best, bound) + slack) continue;
    double dq = INFINITY;
    for (int64_t p = g.geom_part_off[q]; p < g.geom_part_off[q + 1]; ++p) {
      const double lim = fmin(fmin(best, bound), dq) + slack;
      if (box_dist(ix.part_box + 4 * p, x, y) > lim) continue;
      const double y0 = ix.part_band[2 * p], per = ix.part_band[2 * p + 1];
      const int nb = ix.part_nb[p];
      const int64_t base = ix.part_band_base[p];
      // the part's bands are consecutive, so bands blo..bhi are one run of entries
      const int64_t e0 = ix.band_off[base + band_of(y - lim, y0, per, nb)];
      const int64_t e1 = ix.band_off[base + band_of(y + lim, y0, per, nb) + 1];
      double d = INFINITY;
      for (int64_t e = e0 + lane; e < e1; e += 32) {
        const int64_t i = entries[e];
        d = fmin(d, point_to_segment(x, y, g.v[2 * i], g.v[2 * i + 1], g.v[2 * i + 2], g.v[2 * i + 3]));
      }
      dq = fmin(dq, warp_min(d));
    }
    if (dq < best) { best = dq; best_q = int32_t(q); }
  }
  if (lane == 0) {
    country[n] = best_q;
    bool bnd;
    if (pred_inside) pred_inside[n] = locate_in(g, ix, entries, best_q, pred[2 * n], pred[2 * n + 1], &bnd) && !bnd;
  }
}

// One thread per sample: the lowest-index geometry that covers the label, and whether it contains the prediction.
// Labels covered by none are flagged for nearest_kernel.
__global__ void __launch_bounds__(LOCATE_THREADS) locate_kernel(Geo g, Index ix, const int32_t* __restrict__ entries,
                                                                const double* __restrict__ label,
                                                                const double* __restrict__ pred, int64_t N,
                                                                int32_t* __restrict__ country, uint8_t* __restrict__ flags,
                                                                uint8_t* __restrict__ pred_inside) {
  const int64_t n = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (n >= N) return;
  const double lx = label[2 * n], ly = label[2 * n + 1];
  int32_t c = -1;
  bool bnd;
  for (int64_t q = 0; q < g.G && c < 0; ++q)
    if (locate_in(g, ix, entries, q, lx, ly, &bnd)) c = int32_t(q);
  country[n] = c;
  flags[n] = c < 0 ? PG_COUNTRY_NEAREST : 0;
  if (pred_inside && c >= 0) pred_inside[n] = locate_in(g, ix, entries, c, pred[2 * n], pred[2 * n + 1], &bnd) && !bnd;
}

// ---------------------------------------------------------------------------------------------------------- metrics
constexpr int NUM_COUNTS = NUM_KM + 3;  // Under_*_km, top-1, top-k, country

struct MetricWs {
  int64_t* counts;  // [blocks, NUM_COUNTS]
  double* sums;     // [blocks, 2]: km, score
  double* sel;      // [2]: the two middle order statistics
};

size_t metric_layout(int64_t N, char* base, MetricWs* w) {
  const int64_t blocks = (N + METRIC_THREADS - 1) / METRIC_THREADS;
  size_t off = 0;
  auto take = [&](size_t bytes) {
    char* p = base ? base + off : nullptr;
    off += align256(bytes);
    return p;
  };
  MetricWs t;
  t.counts = (int64_t*)take(8 * size_t(blocks) * NUM_COUNTS);
  t.sums = (double*)take(16 * size_t(blocks));
  t.sel = (double*)take(16);
  if (w) *w = t;
  return off;
}

// numpy's np.radians: x * (pi / 180) in the operand's type (NPY_PIf / 180.0f for float32).
constexpr double DEG2RAD = 3.141592653589793 / 180.0;
constexpr float DEG2RADF = 3.14159265358979323846f / 180.0f;

// preprocessing/geo_utils.py haversine_np(x = predictions, y = labels) for one row in numpy's operation order.  With
// float32 predictions numpy takes np.radians and np.cos of the prediction in float32; the rest is float64.
__device__ __forceinline__ double haversine_np(double px, double py, bool pred_f32, double lx, double ly) {
  double xr0, xr1, cx;
  if (pred_f32) {
    const float f0 = __fmul_rn(float(px), DEG2RADF), f1 = __fmul_rn(float(py), DEG2RADF);
    xr0 = f0; xr1 = f1;
    cx = double(float(cos(double(f1))));
  } else {
    xr0 = __dmul_rn(px, DEG2RAD); xr1 = __dmul_rn(py, DEG2RAD);
    cx = cos(xr1);
  }
  const double yr0 = __dmul_rn(lx, DEG2RAD), yr1 = __dmul_rn(ly, DEG2RAD);
  const double s1 = sin(__ddiv_rn(__dsub_rn(yr1, xr1), 2.0)), s0 = sin(__ddiv_rn(__dsub_rn(yr0, xr0), 2.0));
  const double a = __dadd_rn(__dmul_rn(s1, s1), __dmul_rn(__dmul_rn(cx, cos(yr1)), __dmul_rn(s0, s0)));
  const double c = __dmul_rn(2.0, asin(__dsqrt_rn(a)));
  return __ddiv_rn(__dmul_rn(6378137.0, c), 1000.0);
}

// np.round(5000 * np.exp(-d / DECAY_CONSTANT)).
__device__ __forceinline__ double geoguessr_score(double d) {
  return rint(__dmul_rn(5000.0, exp(__ddiv_rn(-d, 1492.7))));
}

__global__ void __launch_bounds__(METRIC_THREADS) metrics_kernel(const void* __restrict__ pred, int32_t pred_f32,
                                                                 const double* __restrict__ label, int64_t N,
                                                                 const int64_t* __restrict__ cell_pred,
                                                                 const int64_t* __restrict__ cell_label,
                                                                 const int64_t* __restrict__ topk, int32_t k,
                                                                 const uint8_t* __restrict__ pred_inside,
                                                                 double* __restrict__ dist, MetricWs w) {
  __shared__ int64_t s_cnt[METRIC_THREADS / 32][NUM_COUNTS];
  __shared__ double s_sum[METRIC_THREADS / 32][2];
  const int64_t n = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  int64_t cnt[NUM_COUNTS] = {};
  double km = 0.0, score = 0.0;
  if (n < N) {
    double px, py;
    if (pred_f32) { px = static_cast<const float*>(pred)[2 * n]; py = static_cast<const float*>(pred)[2 * n + 1]; }
    else { px = static_cast<const double*>(pred)[2 * n]; py = static_cast<const double*>(pred)[2 * n + 1]; }
    km = haversine_np(px, py, pred_f32 != 0, label[2 * n], label[2 * n + 1]);
    dist[n] = km;
    score = geoguessr_score(km);
#pragma unroll
    for (int t = 0; t < NUM_KM; ++t) cnt[t] = km < KM_THRESHOLDS[t];
    const int64_t lab = cell_label[n];
    cnt[NUM_KM] = cell_pred[n] == lab;
    for (int j = 0; j < k; ++j) cnt[NUM_KM + 1] |= topk[n * k + j] == lab;
    cnt[NUM_KM + 2] = pred_inside[n] != 0;
  }
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int o = 16; o > 0; o >>= 1) {
#pragma unroll
    for (int t = 0; t < NUM_COUNTS; ++t) cnt[t] += __shfl_xor_sync(0xffffffffu, cnt[t], o);
    km = __dadd_rn(km, __shfl_xor_sync(0xffffffffu, km, o));
    score = __dadd_rn(score, __shfl_xor_sync(0xffffffffu, score, o));
  }
  if (lane == 0) {
    for (int t = 0; t < NUM_COUNTS; ++t) s_cnt[warp][t] = cnt[t];
    s_sum[warp][0] = km;
    s_sum[warp][1] = score;
  }
  __syncthreads();
  if (threadIdx.x < NUM_COUNTS) {
    int64_t c = 0;
    for (int v = 0; v < METRIC_THREADS / 32; ++v) c += s_cnt[v][threadIdx.x];
    w.counts[blockIdx.x * NUM_COUNTS + threadIdx.x] = c;
  } else if (threadIdx.x >= 32 && threadIdx.x < 34) {
    const int t = threadIdx.x - 32;
    double c = 0.0;
    for (int v = 0; v < METRIC_THREADS / 32; ++v) c = __dadd_rn(c, s_sum[v][t]);
    w.sums[2 * blockIdx.x + t] = c;
  }
}

// Block 0 and 1 select the order statistics (N - 1) / 2 and N / 2 (0-based) of the distances.
__global__ void __launch_bounds__(SELECT_THREADS) median_kernel(const double* __restrict__ dist, int64_t N, MetricWs w) {
  const uint32_t k = uint32_t(blockIdx.x == 0 ? (N - 1) / 2 : N / 2) + 1;
  const uint64_t v = radix_select_kth<SELECT_THREADS>(N, k, [&](int64_t j) { return uint64_t(__double_as_longlong(dist[j])); });
  if (threadIdx.x == 0) w.sel[blockIdx.x] = __longlong_as_double(v);
}

// One CTA: block partials in a fixed order (per-thread strided sums, then a fixed tree), then the results.
__global__ void __launch_bounds__(256) finalize_kernel(int64_t N, MetricWs w, double* __restrict__ out) {
  __shared__ int64_t s_cnt[256];
  __shared__ double s_km[256];
  __shared__ double s_score[256];
  const int64_t blocks = (N + METRIC_THREADS - 1) / METRIC_THREADS;
  const double dn = double(N);
  double km = 0.0, score = 0.0;
  for (int64_t b = threadIdx.x; b < blocks; b += 256) { km = __dadd_rn(km, w.sums[2 * b]); score = __dadd_rn(score, w.sums[2 * b + 1]); }
  s_km[threadIdx.x] = km;
  s_score[threadIdx.x] = score;
  __syncthreads();
  for (int o = 128; o > 0; o >>= 1) {
    if (threadIdx.x < o) {
      s_km[threadIdx.x] = __dadd_rn(s_km[threadIdx.x], s_km[threadIdx.x + o]);
      s_score[threadIdx.x] = __dadd_rn(s_score[threadIdx.x], s_score[threadIdx.x + o]);
    }
    __syncthreads();
  }
  for (int t = 0; t < NUM_COUNTS; ++t) {
    int64_t c = 0;
    for (int64_t b = threadIdx.x; b < blocks; b += 256) c += w.counts[b * NUM_COUNTS + t];
    s_cnt[threadIdx.x] = c;
    __syncthreads();
    for (int o = 128; o > 0; o >>= 1) {
      if (threadIdx.x < o) s_cnt[threadIdx.x] += s_cnt[threadIdx.x + o];
      __syncthreads();
    }
    if (threadIdx.x == 0) {
      const double share = __ddiv_rn(double(s_cnt[0]), dn);
      if (t < NUM_KM) out[PG_GEO_UNDER_KM + t] = share;
      else if (t == NUM_KM) out[PG_GEO_TOP1] = share;
      else if (t == NUM_KM + 1) out[PG_GEO_TOPK] = share;
      else out[PG_GEO_COUNTRY] = share;
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    out[PG_GEO_MEAN_KM] = __ddiv_rn(s_km[0], dn);
    out[PG_GEO_SCORE] = __ddiv_rn(s_score[0], dn);
    out[PG_GEO_MEDIAN_KM] = (N & 1) ? w.sel[0] : __ddiv_rn(__dadd_rn(w.sel[0], w.sel[1]), 2.0);
  }
}

bool geo_args_ok(const PgCountries* c, const char* what) {
  if (!c) { set_last_error("%s: NULL countries", what); return false; }
  if (c->num_verts < 2 || c->num_rings < 1 || c->num_parts < 1 || c->num_geoms < 1 ||
      c->num_verts >= (int64_t(1) << 31) || c->num_geoms >= (int64_t(1) << 31)) {
    set_last_error("%s: bad sizes (verts %lld, rings %lld, parts %lld, geometries %lld)", what, (long long)c->num_verts,
                   (long long)c->num_rings, (long long)c->num_parts, (long long)c->num_geoms);
    return false;
  }
  if (!c->verts || !c->ring_off || !c->part_ring_off || !c->geom_part_off || !c->index) {
    set_last_error("%s: NULL argument", what);
    return false;
  }
  const size_t need = index_layout(c->num_verts, c->num_parts, c->num_geoms, nullptr, nullptr);
  if (c->index_bytes < need) {
    set_last_error("%s: index of %zu bytes is too small (need %zu)", what, c->index_bytes, need);
    return false;
  }
  return true;
}

Geo geo_of(const PgCountries* c) {
  return Geo{c->verts, c->ring_off, c->part_ring_off, c->geom_part_off, c->num_verts, c->num_rings, c->num_parts,
             c->num_geoms};
}

int launch_status(const char* what) {
  const cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) {
    set_last_error("%s: launch failed: %s", what, cudaGetErrorString(e));
    return 1;
  }
  return 0;
}

}  // namespace
}  // namespace pg

using namespace pg;

extern "C" size_t pg_country_index_bytes(int64_t num_verts, int64_t num_parts, int64_t num_geoms) {
  if (num_verts < 0 || num_parts < 0 || num_geoms < 0) return 0;
  return index_layout(num_verts, num_parts, num_geoms, nullptr, nullptr);
}

extern "C" int pg_country_index_build(const PgCountries* c, int64_t* num_entries_out, void* stream) {
  if (!geo_args_ok(c, "pg_country_index_build")) return 1;
  Index ix;
  index_layout(c->num_verts, c->num_parts, c->num_geoms, static_cast<char*>(c->index), &ix);
  const Geo g = geo_of(c);
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  part_kernel<<<unsigned(g.P), 256, 0, s>>>(g, ix);
  layout_kernel<<<1, 1024, 0, s>>>(g, ix);
  count_kernel<<<unsigned((g.V + 255) / 256), 256, 0, s>>>(g, ix);
  scan_kernel<<<1, 1024, 0, s>>>(g, ix, num_entries_out);
  return launch_status("pg_country_index_build");
}

extern "C" int pg_country_index_fill(const PgCountries* c, void* stream) {
  if (!geo_args_ok(c, "pg_country_index_fill")) return 1;
  if (!c->entries || c->num_entries < 0) {
    set_last_error("pg_country_index_fill: NULL entries");
    return 1;
  }
  Index ix;
  index_layout(c->num_verts, c->num_parts, c->num_geoms, static_cast<char*>(c->index), &ix);
  fill_kernel<<<unsigned((c->num_parts * 32 + 127) / 128), 128, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      geo_of(c), ix, c->entries);
  return launch_status("pg_country_index_fill");
}

extern "C" int pg_country_locate(const PgCountries* c, const double* label_lnglat, const double* pred_lnglat, int64_t N,
                                 int32_t* country_out, uint8_t* flags_out, uint8_t* pred_inside_out, void* stream) {
  if (!geo_args_ok(c, "pg_country_locate")) return 1;
  if (N < 0 || !c->entries) {
    set_last_error("pg_country_locate: bad N (%lld) or an index without entries", (long long)N);
    return 1;
  }
  if (N == 0) return 0;
  if (!label_lnglat || !country_out || !flags_out || (pred_inside_out && !pred_lnglat)) {
    set_last_error("pg_country_locate: NULL argument");
    return 1;
  }
  Index ix;
  index_layout(c->num_verts, c->num_parts, c->num_geoms, static_cast<char*>(c->index), &ix);
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  const Geo g = geo_of(c);
  locate_kernel<<<unsigned((N + LOCATE_THREADS - 1) / LOCATE_THREADS), LOCATE_THREADS, 0, s>>>(
      g, ix, c->entries, label_lnglat, pred_lnglat, N, country_out, flags_out, pred_inside_out);
  nearest_kernel<<<unsigned((N * 32 + 255) / 256), 256, 0, s>>>(g, ix, c->entries, label_lnglat, pred_lnglat, N,
                                                               country_out, flags_out, pred_inside_out);
  return launch_status("pg_country_locate");
}

extern "C" size_t pg_geo_metrics_workspace_bytes(int64_t N) {
  if (N < 0) return 0;
  return metric_layout(N, nullptr, nullptr);
}

extern "C" int pg_geo_metrics(const void* pred_lnglat, int32_t pred_is_f32, const double* label_lnglat, int64_t N,
                              const int64_t* cell_pred, const int64_t* cell_label, const int64_t* topk, int32_t k,
                              const uint8_t* pred_inside, void* workspace, size_t workspace_bytes, double* dist_out,
                              double* results_out, void* stream) {
  if (N < 1 || N >= (int64_t(1) << 31) || k < 1) {
    set_last_error("pg_geo_metrics: bad sizes (N %lld, k %d)", (long long)N, k);
    return 1;
  }
  if (!pred_lnglat || !label_lnglat || !cell_pred || !cell_label || !topk || !pred_inside || !dist_out || !results_out) {
    set_last_error("pg_geo_metrics: NULL argument");
    return 1;
  }
  const size_t need = metric_layout(N, nullptr, nullptr);
  if (!workspace || workspace_bytes < need) {
    set_last_error("pg_geo_metrics: workspace of %zu bytes is too small (need %zu)", workspace_bytes, need);
    return 1;
  }
  MetricWs w;
  metric_layout(N, static_cast<char*>(workspace), &w);
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  const unsigned blocks = unsigned((N + METRIC_THREADS - 1) / METRIC_THREADS);
  metrics_kernel<<<blocks, METRIC_THREADS, 0, s>>>(pred_lnglat, pred_is_f32, label_lnglat, N, cell_pred, cell_label, topk,
                                                   k, pred_inside, dist_out, w);
  median_kernel<<<2, SELECT_THREADS, 0, s>>>(dist_out, N, w);
  finalize_kernel<<<1, 256, 0, s>>>(N, w, results_out);
  return launch_status("pg_geo_metrics");
}
