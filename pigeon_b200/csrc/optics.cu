// Per-geocell OPTICS-xi clustering of training locations: what reference dataset_creation/prototype/prototype.py:121-145
// (`ProtoDataset._compute_distances` + `_compute_clusters`) runs per geocell, i.e.
//   OPTICS(min_samples=m, xi=xi, metric='precomputed').fit_predict(D)
// of scikit-learn (compute_optics_graph with max_eps=inf, then cluster_optics_xi with min_cluster_size=m and
// predecessor_correction=True), on the fp64 haversine matrix D that is never stored: every entry is recomputed on the fly.
//
// Four kernels per call, all on the caller's stream:
//   prep      per point: deg2rad and cos(lat) (numpy forms these per point too);
//   core      one CTA per point: the m-th smallest entry of its row by radix_select.cuh's exact 6-pass radix select
//             on the uint64 bit pattern of the distance (all distances are positive, so bit order is value order);
//   ordering  one CTA per cell, largest cells first: n steps of "mark p processed, update every unprocessed j, arg-min";
//             the update and the next arg-min are one pass plus one block reduction;
//   xi        one thread per cell: sklearn's _xi_cluster + _extract_xi_labels on the reachability plot.
// No atomics on values, so every result is deterministic.
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

#include "../../include/pigeon_b200.h"
#include "radix_select.cuh"
#include "tma_host.h"

namespace pg {
namespace {

constexpr int CORE_THREADS = 256;
constexpr int ORDER_THREADS = 256;
constexpr int ORDER_WARPS = ORDER_THREADS / 32;
// Cells up to this many points keep their per-point state in shared memory (37 B per point, ~104 KB, so two CTAs
// fit on an SM); larger cells keep it in their slice of the workspace, which stays L2-resident.
constexpr int SMEM_POINTS = 2800;
constexpr int SMEM_BYTES_PER_POINT = 3 * 8 + 8 + 4 + 1;
constexpr int XI_THREADS = 64;

__host__ __device__ constexpr size_t align256(size_t x) { return (x + 255) & ~size_t(255); }

// Workspace layout for N points and C cells (every array indexed by the global point index).
struct Ws {
  double *lng, *lat, *coslat, *core, *reach, *reach_plot, *sda_mib;
  int32_t *pred, *pred_plot, *ord, *pos, *sda_start, *sda_end, *uc_start, *uc_end, *lab_plot, *cell_order;
  uint8_t* done;
};

size_t ws_layout(int64_t N, int32_t C, char* base, Ws* w) {
  size_t off = 0;
  auto take = [&](size_t bytes) {
    char* p = base ? base + off : nullptr;
    off += align256(bytes);
    return p;
  };
  const size_t d = sizeof(double) * size_t(N), i = sizeof(int32_t) * size_t(N);
  Ws t;
  t.lng = (double*)take(d); t.lat = (double*)take(d); t.coslat = (double*)take(d); t.core = (double*)take(d);
  t.reach = (double*)take(d); t.reach_plot = (double*)take(d); t.sda_mib = (double*)take(d);
  t.pred = (int32_t*)take(i); t.pred_plot = (int32_t*)take(i); t.ord = (int32_t*)take(i); t.pos = (int32_t*)take(i);
  t.sda_start = (int32_t*)take(i); t.sda_end = (int32_t*)take(i); t.uc_start = (int32_t*)take(i);
  t.uc_end = (int32_t*)take(i); t.lab_plot = (int32_t*)take(i);
  t.cell_order = (int32_t*)take(sizeof(int32_t) * size_t(C > 0 ? C : 1));
  t.done = (uint8_t*)take(size_t(N));
  if (w) *w = t;
  return off;
}

// numpy's np.deg2rad is x * (pi / 180).
constexpr double DEG2RAD = 3.141592653589793 / 180.0;

__global__ void prep_kernel(const double* __restrict__ lnglat, int64_t N, Ws w) {
  const int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= N) return;
  const double lng = __dmul_rn(lnglat[2 * i], DEG2RAD), lat = __dmul_rn(lnglat[2 * i + 1], DEG2RAD);
  w.lng[i] = lng;
  w.lat[i] = lat;
  w.coslat[i] = cos(lat);
}

// preprocessing/geo_utils.py:77-93 (haversine_matrix_np) for row i, column j, in numpy's operation order, then
// prototype.py:132 (an exact 0 becomes 1e-5).  Every product and sum is rounded on its own: no FMA contraction.
__device__ __forceinline__ double haversine_km(double lng_i, double lat_i, double cos_i, double lng_j, double lat_j,
                                               double cos_j) {
  const double p = __dmul_rn(cos_i, cos_j);
  const double s_lat = sin(__dmul_rn(__dsub_rn(lat_i, lat_j), 0.5));
  const double s_lng = sin(__dmul_rn(__dsub_rn(lng_i, lng_j), 0.5));
  const double a = __dadd_rn(__dmul_rn(s_lat, s_lat), __dmul_rn(p, __dmul_rn(s_lng, s_lng)));
  const double c = __dmul_rn(2.0, asin(__dsqrt_rn(a)));
  const double km = __ddiv_rn(__dmul_rn(6378137.0, c), 1000.0);
  return km == 0.0 ? 1e-5 : km;
}

// np.around(x, 15) for float64: rint(x * 1e15) / 1e15.
__device__ __forceinline__ double around15(double x) { return __ddiv_rn(rint(__dmul_rn(x, 1e15)), 1e15); }

__device__ __forceinline__ int64_t find_cell(const int64_t* __restrict__ cell_off, int32_t C, int64_t i) {
  int lo = 0, hi = C;  // largest c with cell_off[c] <= i
  while (hi - lo > 1) {
    const int mid = (lo + hi) >> 1;
    if (cell_off[mid] <= i) lo = mid; else hi = mid;
  }
  return lo;
}

// cell_order[r] = the cell of rank r by size, descending, lower index first on ties (largest cells launch first).
__global__ void cell_order_kernel(const int64_t* __restrict__ cell_off, int32_t C, int32_t* __restrict__ cell_order) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  const int64_t n = cell_off[c + 1] - cell_off[c];
  int rank = 0;
  for (int o = 0; o < C; ++o) {
    const int64_t m = cell_off[o + 1] - cell_off[o];
    rank += (m > n) || (m == n && o < c);
  }
  cell_order[rank] = c;
}

// core[i] = around(m-th smallest of row i of D, 15): NearestNeighbors.kneighbors(X, m)[0][:, -1] of a precomputed
// matrix, the diagonal included (sklearn/cluster/_optics.py _compute_core_distances_, compute_optics_graph).
// Exact radix select (radix_select.cuh); each pass recomputes the row, so there is no per-row storage and any m works.
__global__ void __launch_bounds__(CORE_THREADS) core_kernel(const int64_t* __restrict__ cell_off, int32_t C, int32_t m,
                                                            Ws w) {
  const int64_t i = blockIdx.x;
  const int64_t c = find_cell(cell_off, C, i);
  const int64_t b = cell_off[c], n = cell_off[c + 1] - b;
  if (n < m) return;
  const double li = w.lng[i], ai = w.lat[i], ci = w.coslat[i];
  const uint64_t kth = radix_select_kth<CORE_THREADS>(n, uint32_t(m), [&](int64_t j) {
    return uint64_t(__double_as_longlong(haversine_km(li, ai, ci, w.lng[b + j], w.lat[b + j], w.coslat[b + j])));
  });
  if (threadIdx.x == 0) w.core[i] = around15(__longlong_as_double(kth));
}

// compute_optics_graph's main loop (max_eps = inf) for one cell: at each step the unprocessed point of least
// reachability (lowest index on ties, inf included) is processed, and every unprocessed j gets
// r = around(max(D[p, j], core[p]), 15); reach[j] = r and pred[j] = p where r < reach[j] (_set_reach_dist).
// Point j is only ever touched by thread j % ORDER_THREADS, so the per-point state needs no synchronisation; the one
// __syncthreads per step publishes the per-warp arg-mins (double-buffered, so the next step can overwrite the other half).
__global__ void __launch_bounds__(ORDER_THREADS, 2) ordering_kernel(const int64_t* __restrict__ cell_off, int32_t m,
                                                                 int32_t smem_points, Ws w, int32_t* __restrict__ labels,
                                                                 int64_t* __restrict__ ordering_out,
                                                                 double* __restrict__ reach_out,
                                                                 double* __restrict__ core_out,
                                                                 int64_t* __restrict__ pred_out) {
  extern __shared__ __align__(16) unsigned char smem[];
  __shared__ uint64_t red_key[2][ORDER_WARPS];
  __shared__ int32_t red_idx[2][ORDER_WARPS];
  const int cell = w.cell_order[blockIdx.x];
  const int64_t b = cell_off[cell];
  const int n = int(cell_off[cell + 1] - b);
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  if (n < m) {  // prototype.py:144-145: label 0 for every point, no OPTICS graph
    for (int j = tid; j < n; j += ORDER_THREADS) {
      labels[b + j] = 0;
      if (ordering_out) ordering_out[b + j] = -1;
      if (reach_out) reach_out[b + j] = __longlong_as_double(0x7ff8000000000000ll);
      if (core_out) core_out[b + j] = __longlong_as_double(0x7ff8000000000000ll);
      if (pred_out) pred_out[b + j] = -1;
    }
    return;
  }
  const double* lng = w.lng + b;
  const double* lat = w.lat + b;
  const double* cs = w.coslat + b;
  double* reach = w.reach + b;
  int32_t* pred = w.pred + b;
  uint8_t* done = w.done + b;
  if (n <= smem_points) {
    double* s_lng = reinterpret_cast<double*>(smem);
    double* s_lat = s_lng + n;
    double* s_cs = s_lat + n;
    double* s_reach = s_cs + n;
    int32_t* s_pred = reinterpret_cast<int32_t*>(s_reach + n);
    uint8_t* s_done = reinterpret_cast<uint8_t*>(s_pred + n);
    for (int j = tid; j < n; j += ORDER_THREADS) { s_lng[j] = lng[j]; s_lat[j] = lat[j]; s_cs[j] = cs[j]; }
    lng = s_lng; lat = s_lat; cs = s_cs; reach = s_reach; pred = s_pred; done = s_done;
  }
  for (int j = tid; j < n; j += ORDER_THREADS) { reach[j] = __longlong_as_double(0x7ff0000000000000ll); pred[j] = -1; done[j] = 0; }
  __syncthreads();
  const double* core = w.core + b;
  int p = 0;  // arg-min of an all-inf reachability: the lowest index
  for (int k = 0; k < n; ++k) {
    const double lp = lng[p], ap = lat[p], cp = cs[p], corep = core[p];
    if (tid == p % ORDER_THREADS) {
      done[p] = 1;
      w.ord[b + k] = p;
      w.pos[b + p] = k;
      w.reach_plot[b + k] = reach[p];
      w.pred_plot[b + k] = pred[p];
    }
    uint64_t best_key = ~0ull;
    int best_idx = 0x7fffffff;
    for (int j = tid; j < n; j += ORDER_THREADS) {
      if (done[j]) continue;
      double rj = reach[j];
      const double r = around15(fmax(haversine_km(lp, ap, cp, lng[j], lat[j], cs[j]), corep));
      if (r < rj) { reach[j] = r; pred[j] = p; rj = r; }
      const uint64_t key = __double_as_longlong(rj);  // non-negative: bit order is value order
      if (key < best_key) { best_key = key; best_idx = j; }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const uint64_t ok = __shfl_xor_sync(0xffffffffu, best_key, o);
      const int oi = __shfl_xor_sync(0xffffffffu, best_idx, o);
      if (ok < best_key || (ok == best_key && oi < best_idx)) { best_key = ok; best_idx = oi; }
    }
    if (lane == 0) { red_key[k & 1][warp] = best_key; red_idx[k & 1][warp] = best_idx; }
    __syncthreads();
    best_key = red_key[k & 1][0];
    best_idx = red_idx[k & 1][0];
#pragma unroll
    for (int t = 1; t < ORDER_WARPS; ++t) {
      const uint64_t ok = red_key[k & 1][t];
      const int oi = red_idx[k & 1][t];
      if (ok < best_key || (ok == best_key && oi < best_idx)) { best_key = ok; best_idx = oi; }
    }
    p = best_idx;
  }
  for (int j = tid; j < n; j += ORDER_THREADS) {
    if (reach_out) reach_out[b + j] = reach[j];
    if (pred_out) pred_out[b + j] = pred[j];
    if (core_out) core_out[b + j] = core[j];
  }
  __syncthreads();  // w.ord of every step is written by its owner thread
  if (ordering_out)
    for (int k = tid; k < n; k += ORDER_THREADS) ordering_out[b + k] = w.ord[b + k];
}

// sklearn/cluster/_optics.py cluster_optics_xi(min_cluster_size = min_samples, predecessor_correction = True): _xi_cluster
// on the reachability plot R (R[n] = inf, as its np.hstack appends) with numpy's IEEE arithmetic (inf/inf is NaN and
// every comparison with NaN is false), then _extract_xi_labels.  Each U area's clusters are labelled as soon as it is
// complete, in the order _xi_cluster appends them, so only the current U's candidate list is kept.
struct XiCell {
  const double* rp;
  const int32_t* pp;
  const int32_t* pos;
  int n;
  __device__ double R(int i) const { return (i >= 0 && i < n) ? rp[i] : __longlong_as_double(0x7ff0000000000000ll); }
  __device__ double ratio(int i) const { return __ddiv_rn(R(i), R(i + 1)); }
};

// _extend_region: steep / xward tests are chosen by `up` (steep upward region with downward points, or the reverse).
__device__ int extend_region(const XiCell& x, bool up, double xc, double inv_xc, int start, int m) {
  int non_xward = 0, end = start;
  for (int index = start; index < x.n; ++index) {
    const double q = x.ratio(index);
    const bool steep = up ? (q <= xc) : (q >= inv_xc);
    const bool xward = up ? (q > 1.0) : (q < 1.0);
    if (steep) {
      non_xward = 0;
      end = index;
    } else if (!xward) {
      if (++non_xward > m) break;
    } else {
      return end;
    }
  }
  return end;
}

__global__ void xi_kernel(const int64_t* __restrict__ cell_off, int32_t C, int32_t m, double xi, Ws w,
                          int32_t* __restrict__ labels) {
  const int cell = blockIdx.x * blockDim.x + threadIdx.x;
  if (cell >= C) return;
  const int64_t b = cell_off[cell];
  const int n = int(cell_off[cell + 1] - b);
  if (n < m) return;
  const XiCell x{w.reach_plot + b, w.pred_plot + b, w.pos + b, n};
  int32_t *sda_start = w.sda_start + b, *sda_end = w.sda_end + b, *uc_start = w.uc_start + b, *uc_end = w.uc_end + b;
  int32_t* lab = w.lab_plot + b;
  double* sda_mib = w.sda_mib + b;
  const double xc = __dsub_rn(1.0, xi), inv_xc = __ddiv_rn(1.0, xc);
  for (int k = 0; k < n; ++k) lab[k] = -1;
  int nsda = 0, index = 0, label = 0;
  double mib = 0.0;
  auto filter_sdas = [&](double mib_now) {  // _update_filter_sdas
    if (isinf(mib_now)) { nsda = 0; return; }
    int kept = 0;
    for (int t = 0; t < nsda; ++t) {
      if (mib_now <= __dmul_rn(x.R(sda_start[t]), xc)) {
        sda_start[kept] = sda_start[t];
        sda_end[kept] = sda_end[t];
        sda_mib[kept] = mib_now > sda_mib[t] ? mib_now : sda_mib[t];
        ++kept;
      }
    }
    nsda = kept;
  };
  for (int s = 0; s < n; ++s) {
    const double q = x.ratio(s);
    const bool s_up = q <= xc, s_down = q >= inv_xc;
    if (!(s_up || s_down) || s < index) continue;
    double mx = x.R(index);
    for (int t = index + 1; t <= s; ++t) mx = x.R(t) > mx ? x.R(t) : mx;
    mib = mx > mib ? mx : mib;
    filter_sdas(mib);
    if (s_down) {
      const int d_end = extend_region(x, false, xc, inv_xc, s, m);
      sda_start[nsda] = s; sda_end[nsda] = d_end; sda_mib[nsda] = 0.0; ++nsda;
      index = d_end + 1;
      mib = x.R(index);
      continue;
    }
    const int u_start = s, u_end = extend_region(x, true, xc, inv_xc, s, m);
    index = u_end + 1;
    mib = x.R(index);
    int nu = 0;
    for (int t = 0; t < nsda; ++t) {
      int c_start = sda_start[t], c_end = u_end;
      const double r_after = x.R(c_end + 1);
      if (__dmul_rn(r_after, xc) < sda_mib[t]) continue;
      const double d_max = x.R(sda_start[t]);
      if (__dmul_rn(d_max, xc) >= r_after) {
        while (x.R(c_start + 1) > r_after && c_start < sda_end[t]) ++c_start;
      } else if (__dmul_rn(r_after, xc) >= d_max) {
        while (x.R(c_end - 1) > d_max && c_end > u_start) --c_end;
      }
      // _correct_predecessor: pred_plot[e] among ordering[s:e] <=> s <= pos[pred_plot[e]] < e
      bool found = false;
      while (c_start < c_end) {
        if (x.R(c_start) > x.R(c_end)) { found = true; break; }
        const int pe = x.pp[c_end];
        if (pe >= 0 && x.pos[pe] >= c_start && x.pos[pe] < c_end) { found = true; break; }
        --c_end;
      }
      if (!found) continue;
      if (c_end - c_start + 1 < m) continue;
      if (c_start > sda_end[t]) continue;
      if (c_end < u_start) continue;
      uc_start[nu] = c_start; uc_end[nu] = c_end; ++nu;
    }
    for (int t = nu - 1; t >= 0; --t) {  // U_clusters.reverse(); then _extract_xi_labels in that order
      bool free_range = true;
      for (int k = uc_start[t]; k <= uc_end[t] && free_range; ++k) free_range = lab[k] == -1;
      if (!free_range) continue;
      for (int k = uc_start[t]; k <= uc_end[t]; ++k) lab[k] = label;
      ++label;
    }
  }
  for (int k = 0; k < n; ++k) labels[b + w.ord[b + k]] = lab[k];
}

}  // namespace
}  // namespace pg

using namespace pg;

extern "C" size_t pg_optics_workspace_bytes(int64_t N, int32_t num_cells) {
  if (N < 0 || num_cells < 0) return 0;
  return ws_layout(N, num_cells, nullptr, nullptr);
}

extern "C" int pg_optics_xi(const double* lnglat_deg, int64_t N, const int64_t* cell_off, int32_t num_cells,
                            int64_t max_cell, int32_t min_samples, double xi, void* workspace, size_t workspace_bytes,
                            int32_t* labels_out, int64_t* ordering_out, double* reach_out, double* core_out,
                            int64_t* pred_out, void* stream) {
  if (N < 0 || num_cells < 0 || max_cell < 0 || max_cell > N || max_cell >= (int64_t(1) << 31)) {
    set_last_error("pg_optics_xi: bad sizes (N %lld, num_cells %d, max_cell %lld)", (long long)N, num_cells,
                   (long long)max_cell);
    return 1;
  }
  if (min_samples < 2) {
    set_last_error("pg_optics_xi: min_samples must be an integer >= 2 (got %d)", min_samples);
    return 1;
  }
  if (!(xi > 0.0 && xi < 1.0)) {
    set_last_error("pg_optics_xi: xi must lie in (0, 1) (got %g)", xi);
    return 1;
  }
  if (num_cells == 0) return 0;
  if (!cell_off || (N > 0 && (!lnglat_deg || !labels_out))) {
    set_last_error("pg_optics_xi: NULL argument");
    return 1;
  }
  const size_t need = ws_layout(N, num_cells, nullptr, nullptr);
  if (!workspace || workspace_bytes < need) {
    set_last_error("pg_optics_xi: workspace of %zu bytes is too small (need %zu)", workspace_bytes, need);
    return 1;
  }
  if (N == 0) return 0;
  Ws w;
  ws_layout(N, num_cells, static_cast<char*>(workspace), &w);
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  const int smem_points = int(max_cell < SMEM_POINTS ? max_cell : SMEM_POINTS);
  const size_t smem = size_t(smem_points) * SMEM_BYTES_PER_POINT + 16;
  cudaError_t e = cudaFuncSetAttribute(ordering_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, int(smem));
  if (e != cudaSuccess) {
    set_last_error("pg_optics_xi: %s", cudaGetErrorString(e));
    return 1;
  }
  prep_kernel<<<unsigned((N + 255) / 256), 256, 0, s>>>(lnglat_deg, N, w);
  cell_order_kernel<<<(num_cells + 127) / 128, 128, 0, s>>>(cell_off, num_cells, w.cell_order);
  core_kernel<<<unsigned(N), CORE_THREADS, 0, s>>>(cell_off, num_cells, min_samples, w);
  ordering_kernel<<<num_cells, ORDER_THREADS, smem, s>>>(cell_off, min_samples, smem_points, w, labels_out, ordering_out,
                                                         reach_out, core_out, pred_out);
  xi_kernel<<<(num_cells + XI_THREADS - 1) / XI_THREADS, XI_THREADS, 0, s>>>(cell_off, num_cells, min_samples, xi, w,
                                                                             labels_out);
  e = cudaGetLastError();
  if (e != cudaSuccess) {
    set_last_error("pg_optics_xi: launch failed: %s", cudaGetErrorString(e));
    return 1;
  }
  return 0;
}
