// ProtoRefiner retrieval on the GPU: restates reference models/proto_refiner.py:121-255,332-357 and
// preprocessing/geo_utils.py:40-55 as three kernels over a CSR-packed prototype bank resident in HBM.
//
//   1. pool      : (B, V, D) -> (B, D) view mean                                  (proto_refiner.py:139-140)
//   2. scan      : one warp per (query, candidate cell): Euclidean arg-min over the cell's prototypes
//                  (:176-181), then the within-cluster farthest-member pick (:233-255, arg-MAX, quirk kept)
//   3. finalize  : one thread per query: temperature softmax (no max-subtraction, :346-357) x candidate
//                  probabilities, arg-max, haversine max-refinement gate (:187-203), outputs (:219-231)
//
// No tensor cores: the scan is HBM/L2-bandwidth + FP32-FMA work; loads are 128-bit, lane-strided.
#include "refiner.h"

#include <math.h>
#include <stdint.h>
#include <stdlib.h>

#include "prof.h"
#include "ptx.cuh"
#include "tma_host.h"

namespace pg {

namespace {

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

__global__ void pool_views_kernel(const float* __restrict__ emb, float* __restrict__ q, long B, int V, int D) {
  const long total = B * D;
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const long b = i / D;
    const int d = i % D;
    float s = 0.f;
    for (int v = 0; v < V; ++v) s += emb[(b * V + v) * D + d];
    q[i] = s / V;
  }
}

template <int NV4>
__device__ __forceinline__ float sqdist(const float4 (&q)[NV4], const float* __restrict__ row, int lane) {
  const float4* r4 = reinterpret_cast<const float4*>(row);
  float4 p[NV4];
#pragma unroll
  for (int i = 0; i < NV4; ++i) p[i] = __ldg(r4 + lane + 32 * i);
  float acc = 0.f;
#pragma unroll
  for (int i = 0; i < NV4; ++i) {
    const float a = p[i].x - q[i].x, b = p[i].y - q[i].y, c = p[i].z - q[i].z, d = p[i].w - q[i].w;
    acc = fmaf(a, a, acc);
    acc = fmaf(b, b, acc);
    acc = fmaf(c, c, acc);
    acc = fmaf(d, d, acc);
  }
  return warp_sum(acc);
}

template <int NV4>
__global__ void __launch_bounds__(256)
scan_kernel(const RefinerBank bank, const float* __restrict__ q, const long long* __restrict__ cand, int cand_stride,
            long B, int topk, float* __restrict__ best_logit, float* __restrict__ best_lnglat,
            int* __restrict__ best_proto) {
  constexpr int D = NV4 * 128;
  const int lane = threadIdx.x & 31;
  const long warps = ((long)gridDim.x * blockDim.x) >> 5;
  const long pairs = B * topk;
  for (long pair = ((long)blockIdx.x * blockDim.x + threadIdx.x) >> 5; pair < pairs; pair += warps) {
    const long b = pair / topk;
    const int j = pair % topk;
    const long long cell = cand[b * cand_stride + j];
    long lo = 0, hi = 0;
    if (cell >= 0 && cell < bank.num_cells) { lo = bank.cell_off[cell]; hi = bank.cell_off[cell + 1]; }
    if (hi <= lo) {
      // reference: protos[cell] is None -> logit -100000, prediction [0., 0.]   (proto_refiner.py:168-174)
      if (lane == 0) {
        best_logit[pair] = -100000.f;
        best_lnglat[2 * pair] = 0.f;
        best_lnglat[2 * pair + 1] = 0.f;
        best_proto[pair] = -1;
      }
      continue;
    }
    float4 qv[NV4];
    const float4* q4 = reinterpret_cast<const float4*>(q + b * D);
#pragma unroll
    for (int i = 0; i < NV4; ++i) qv[i] = q4[lane + 32 * i];

    float best = INFINITY;
    long bp = lo;
    for (long p = lo; p < hi; ++p) {
      const float d2 = sqdist<NV4>(qv, bank.proto_emb + p * D, lane);
      if (d2 < best) { best = d2; bp = p; }  // strict: first minimum wins (torch.argmax of -dist)
    }
    float lng = bank.proto_lnglat[2 * bp], lat = bank.proto_lnglat[2 * bp + 1];
    if (bank.proto_count[bp] != 1) {
      // within-cluster refinement: the member FARTHEST from the query (argmax of distances, :252-253)
      const long mlo = bank.member_off[bp], mhi = bank.member_off[bp + 1];
      float far = -INFINITY;
      long bm = -1;
      for (long mi = mlo; mi < mhi; ++mi) {
        const long idx = bank.member_idx[mi];
        const float d2 = sqdist<NV4>(qv, bank.data_emb + idx * D, lane);
        if (d2 > far) { far = d2; bm = idx; }
      }
      if (bm >= 0) { lng = bank.data_lnglat[2 * bm]; lat = bank.data_lnglat[2 * bm + 1]; }
    }
    if (lane == 0) {
      best_logit[pair] = -sqrtf(best);
      best_lnglat[2 * pair] = lng;
      best_lnglat[2 * pair + 1] = lat;
      best_proto[pair] = (int)bp;
    }
  }
}

// ------------------------------------------------------------------------------------------------
// Cell-major scan (v2).  (query, candidate) pairs are counting-sorted by geocell; one CTA per geocell then reads
// that cell's prototype segment from HBM ONCE (re-reads per 8-query chunk come from L2) and scores every pair of the
// cell against it.  Per warp a 4-prototype x 8-query register tile: prototype rows stay in registers, the 8 query
// rows sit in shared memory interleaved in pairs so that one float2 FMA (ffma2) advances two queries' dot products.
// Algorithmic bytes: sum over touched cells of P_c * D * 4, each once.
// ------------------------------------------------------------------------------------------------
constexpr int kQT = 8;  // queries per chunk
constexpr int kPT = 4;  // prototypes per warp register tile

__global__ void pair_hist_kernel(const RefinerBank bank, const long long* __restrict__ cand, int cand_stride, long B,
                                 int topk, int* __restrict__ cell_cnt, float* __restrict__ best_logit,
                                 float* __restrict__ best_lnglat, int* __restrict__ best_proto,
                                 unsigned long long* __restrict__ best_packed = nullptr) {
  const long pairs = B * topk;
  for (long pair = (long)blockIdx.x * blockDim.x + threadIdx.x; pair < pairs; pair += (long)gridDim.x * blockDim.x) {
    const long b = pair / topk;
    const int j = pair % topk;
    const long long cell = cand[b * cand_stride + j];
    bool live = false;
    if (cell >= 0 && cell < bank.num_cells) live = bank.cell_off[cell + 1] > bank.cell_off[cell];
    if (live) {
      atomicAdd(&cell_cnt[cell], 1);
      if (best_packed) best_packed[pair] = ~0ull;   // identity of the tile scan's atomicMin
    } else {  // reference: protos[cell] is None -> logit -100000, prediction [0., 0.]   (proto_refiner.py:168-174)
      best_logit[pair] = -100000.f;
      best_lnglat[2 * pair] = 0.f;
      best_lnglat[2 * pair + 1] = 0.f;
      best_proto[pair] = -1;
    }
  }
}

// exclusive scan of cell_cnt[0..C) -> cell_start[0..C]; also zeroes the cursors. Single block.
__global__ void cell_scan_offsets_kernel(const int* __restrict__ cell_cnt, int* __restrict__ cell_start,
                                         int* __restrict__ cursor, int C) {
  __shared__ int carry;
  __shared__ int warp_tot[32];
  if (threadIdx.x == 0) carry = 0;
  __syncthreads();
  for (int base = 0; base < C; base += blockDim.x) {
    const int i = base + threadIdx.x;
    const int v = (i < C) ? cell_cnt[i] : 0;
    int x = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int y = __shfl_up_sync(0xffffffffu, x, o);
      if ((threadIdx.x & 31) >= o) x += y;
    }
    if ((threadIdx.x & 31) == 31) warp_tot[threadIdx.x >> 5] = x;
    __syncthreads();
    if (threadIdx.x < 32) {
      int t = (threadIdx.x < (blockDim.x >> 5)) ? warp_tot[threadIdx.x] : 0;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const int y = __shfl_up_sync(0xffffffffu, t, o);
        if (threadIdx.x >= o) t += y;
      }
      warp_tot[threadIdx.x] = t;
    }
    __syncthreads();
    const int warp_off = (threadIdx.x >> 5) ? warp_tot[(threadIdx.x >> 5) - 1] : 0;
    if (i < C) {
      cell_start[i] = carry + warp_off + x - v;
      cursor[i] = 0;
    }
    __syncthreads();
    if (threadIdx.x == blockDim.x - 1) carry += warp_off + x;
    __syncthreads();
  }
  if (threadIdx.x == 0) cell_start[C] = carry;
}

__global__ void pair_scatter_kernel(const RefinerBank bank, const long long* __restrict__ cand, int cand_stride, long B,
                                    int topk, const int* __restrict__ cell_start, int* __restrict__ cursor,
                                    int* __restrict__ order) {
  const long pairs = B * topk;
  for (long pair = (long)blockIdx.x * blockDim.x + threadIdx.x; pair < pairs; pair += (long)gridDim.x * blockDim.x) {
    const long b = pair / topk;
    const int j = pair % topk;
    const long long cell = cand[b * cand_stride + j];
    if (cell >= 0 && cell < bank.num_cells && bank.cell_off[cell + 1] > bank.cell_off[cell])
      order[cell_start[cell] + atomicAdd(&cursor[cell], 1)] = (int)pair;
  }
}

// Shared-memory budget of the staged query set: 2 CTAs / SM.
constexpr int kStageBytes = 96 * 1024;

template <int NV4>
__global__ void __launch_bounds__(256, 2)
cell_major_scan_kernel(const RefinerBank bank, const float* __restrict__ q, const int* __restrict__ cell_start,
                       const int* __restrict__ order, int topk, float* __restrict__ best_logit,
                       float* __restrict__ best_lnglat, int* __restrict__ best_proto) {
  constexpr int D = NV4 * 128;
  constexpr int QS = (kStageBytes / (D * 4)) / kQT * kQT;   // queries staged per pass (32 at D = 768, 24 at D = 1024)
  static_assert(QS >= kQT, "stage holds at least one chunk");
  extern __shared__ float4 qs[];   // [QS/8][NV4][kQT/2][2][32] float4: chunk-major, lanes contiguous
  __shared__ float rbest_d[8][QS]; // per-warp running best of every staged query
  __shared__ int rbest_p[8][QS];   // ... as an offset from the cell's first prototype
  __shared__ float q_sqnorm[QS];
  const int cell = blockIdx.x;
  const int n_pairs = cell_start[cell + 1] - cell_start[cell];
  if (n_pairs == 0) return;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const long lo = bank.cell_off[cell], hi = bank.cell_off[cell + 1];
  const int* my_order = order + cell_start[cell];

  // One pass over the cell's prototype segment per staged query set: when a cell has at most QS pairs (the common
  // case) the segment is read exactly once from HBM.
  for (int c0 = 0; c0 < n_pairs; c0 += QS) {
    const int nq = min(QS, n_pairs - c0);
    const int nch = (nq + kQT - 1) / kQT;
    __syncthreads();
    // stage the queries, two interleaved per float4 (see the ffma2 loop):
    //   qs[(((ch * NV4 + i) * (kQT/2) + qp) * 2 + h) * 32 + lane] = for h = 0: (qA[4c], qB[4c], qA[4c+1], qB[4c+1]),
    //   for h = 1 the same for elements 4c+2, 4c+3;  A = ch*8 + 2qp, B = A + 1, c = lane + 32 i
    for (int idx = threadIdx.x; idx < nch * NV4 * (kQT / 2) * 32; idx += blockDim.x) {
      const int ln = idx & 31;
      const int qp = (idx >> 5) % (kQT / 2);
      const int i = ((idx >> 5) / (kQT / 2)) % NV4;
      const int ch = (idx >> 5) / (kQT / 2) / NV4;
      const int col4 = i * 32 + ln;
      const int qa = ch * kQT + 2 * qp;
      float4 a = make_float4(0.f, 0.f, 0.f, 0.f), b2 = a;
      if (qa < nq) a = reinterpret_cast<const float4*>(q + (long)(my_order[c0 + qa] / topk) * D)[col4];
      if (qa + 1 < nq) b2 = reinterpret_cast<const float4*>(q + (long)(my_order[c0 + qa + 1] / topk) * D)[col4];
      const size_t base = (size_t)(((ch * NV4 + i) * (kQT / 2) + qp) * 2) * 32 + ln;
      qs[base] = make_float4(a.x, b2.x, a.y, b2.y);
      qs[base + 32] = make_float4(a.z, b2.z, a.w, b2.w);
    }
    for (int qi = warp; qi < nch * kQT; qi += 8) {   // |q|^2, warp per query
      float acc_q = 0.f;
      if (qi < nq) {
        const float4* q4 = reinterpret_cast<const float4*>(q + (long)(my_order[c0 + qi] / topk) * D);
#pragma unroll
        for (int i = 0; i < NV4; ++i) {
          const float4 t = q4[lane + 32 * i];
          acc_q = fmaf(t.x, t.x, acc_q); acc_q = fmaf(t.y, t.y, acc_q);
          acc_q = fmaf(t.z, t.z, acc_q); acc_q = fmaf(t.w, t.w, acc_q);
        }
      }
      acc_q = warp_sum(acc_q);
      if (lane == 0) q_sqnorm[qi] = acc_q;
    }
    for (int i = lane; i < QS; i += 32) { rbest_d[warp][i] = INFINITY; rbest_p[warp][i] = 0x7fffffff; }
    __syncthreads();

    for (long p0 = lo + warp * kPT; p0 < hi; p0 += 8 * kPT) {
      // prototype tile: 4 rows in registers (all pieces requested up front), |p|^2 from the same registers
      float4 pr[NV4][kPT];
#pragma unroll
      for (int i = 0; i < NV4; ++i) {
#pragma unroll
        for (int a = 0; a < kPT; ++a) {
          const long pidx = (p0 + a < hi) ? p0 + a : hi - 1;   // clamp: duplicates are discarded below
          pr[i][a] = __ldg(reinterpret_cast<const float4*>(bank.proto_emb + pidx * D) + lane + 32 * i);
        }
      }
      float pn[kPT];
#pragma unroll
      for (int a = 0; a < kPT; ++a) {
        float t = 0.f;
#pragma unroll
        for (int i = 0; i < NV4; ++i) {
          t = fmaf(pr[i][a].x, pr[i][a].x, t); t = fmaf(pr[i][a].y, pr[i][a].y, t);
          t = fmaf(pr[i][a].z, pr[i][a].z, t); t = fmaf(pr[i][a].w, pr[i][a].w, t);
        }
        pn[a] = warp_sum(t);
      }
      const float pn_mine = (lane >> 3) == 0 ? pn[0] : (lane >> 3) == 1 ? pn[1] : (lane >> 3) == 2 ? pn[2] : pn[3];
      const int pp_mine = (int)(p0 - lo) + (lane >> 3);
      const bool p_ok = (p0 + (lane >> 3)) < hi;

      for (int ch = 0; ch < nch; ++ch) {
        // d^2 = |p|^2 + |q|^2 - 2 p.q (the form torch.cdist itself uses beyond 25 rows): one ffma2 per two (p, q)
        // element pairs.
        float2 acc[kPT][kQT / 2];
#pragma unroll
        for (int a = 0; a < kPT; ++a)
#pragma unroll
          for (int b = 0; b < kQT / 2; ++b) acc[a][b] = make_float2(0.f, 0.f);
#pragma unroll
        for (int i = 0; i < NV4; ++i) {
          const float4* qrow = qs + (size_t)((ch * NV4 + i) * (kQT / 2) * 2) * 32 + lane;
#pragma unroll
          for (int b = 0; b < kQT / 2; ++b) {
            const float4 q01 = qrow[(2 * b) * 32], q23 = qrow[(2 * b + 1) * 32];
#pragma unroll
            for (int a = 0; a < kPT; ++a) {
              acc[a][b] = ffma2(make_float2(pr[i][a].x, pr[i][a].x), make_float2(q01.x, q01.y), acc[a][b]);
              acc[a][b] = ffma2(make_float2(pr[i][a].y, pr[i][a].y), make_float2(q01.z, q01.w), acc[a][b]);
              acc[a][b] = ffma2(make_float2(pr[i][a].z, pr[i][a].z), make_float2(q23.x, q23.y), acc[a][b]);
              acc[a][b] = ffma2(make_float2(pr[i][a].w, pr[i][a].w), make_float2(q23.z, q23.w), acc[a][b]);
            }
          }
        }
        // 32 partial dot products (index = proto a * 8 + query) -> lane L ends with the warp total of index L
        float v[32];
#pragma unroll
        for (int a = 0; a < kPT; ++a)
#pragma unroll
          for (int b = 0; b < kQT / 2; ++b) { v[a * kQT + 2 * b] = acc[a][b].x; v[a * kQT + 2 * b + 1] = acc[a][b].y; }
#pragma unroll
        for (int off = 16, n = 16; off >= 1; off >>= 1, n >>= 1) {
#pragma unroll
          for (int k = 0; k < n; ++k) {
            const float send = (lane & off) ? v[k] : v[k + n];
            const float keep = (lane & off) ? v[k + n] : v[k];
            v[k] = keep + __shfl_xor_sync(0xffffffffu, send, off);
          }
        }
        // lane L: prototype (L >> 3) of the tile against query ch*8 + (L & 7); min over the 4 prototypes, first index wins
        float d2 = p_ok ? fmaxf(pn_mine + q_sqnorm[ch * kQT + (lane & 7)] - 2.f * v[0], 0.f) : INFINITY;
        int pp = pp_mine;
#pragma unroll
        for (int off = 8; off <= 16; off <<= 1) {
          const float od = __shfl_xor_sync(0xffffffffu, d2, off);
          const int op = __shfl_xor_sync(0xffffffffu, pp, off);
          if (od < d2 || (od == d2 && op < pp)) { d2 = od; pp = op; }
        }
        if (lane < kQT) {   // lanes 0..7 own the running best of query ch*8 + lane in this warp's private row
          const int qi = ch * kQT + lane;
          const float cd = rbest_d[warp][qi];
          const int cp = rbest_p[warp][qi];
          if (d2 < cd || (d2 == cd && pp < cp)) { rbest_d[warp][qi] = d2; rbest_p[warp][qi] = pp; }
        }
        __syncwarp();
      }
    }
    __syncthreads();
    // warp w finishes queries w, w+8, ...: cross-warp arg-min, then the farthest-member pick, then the outputs
    for (int qi = warp; qi < nq; qi += 8) {
      float bd = rbest_d[0][qi];
      int bpi = rbest_p[0][qi];
      for (int w = 1; w < 8; ++w) {
        const float od = rbest_d[w][qi];
        const int op = rbest_p[w][qi];
        if (od < bd || (od == bd && op < bpi)) { bd = od; bpi = op; }
      }
      const long bp = lo + bpi;
      const long pair = my_order[c0 + qi];
      const long b = pair / topk;
      float lng = bank.proto_lnglat[2 * bp], lat = bank.proto_lnglat[2 * bp + 1];
      if (bank.proto_count[bp] != 1) {
        float4 qv[NV4];
        const float4* q4 = reinterpret_cast<const float4*>(q + b * D);
#pragma unroll
        for (int i = 0; i < NV4; ++i) qv[i] = q4[lane + 32 * i];
        const long mlo = bank.member_off[bp], mhi = bank.member_off[bp + 1];
        float far = -INFINITY;
        long bm = -1;
        for (long mi = mlo; mi < mhi; ++mi) {
          const long idx = bank.member_idx[mi];
          const float dd = sqdist<NV4>(qv, bank.data_emb + idx * D, lane);
          if (dd > far) { far = dd; bm = idx; }
        }
        if (bm >= 0) { lng = bank.data_lnglat[2 * bm]; lat = bank.data_lnglat[2 * bm + 1]; }
      }
      if (lane == 0) {
        best_logit[pair] = -sqrtf(bd);
        best_lnglat[2 * pair] = lng;
        best_lnglat[2 * pair + 1] = lat;
        best_proto[pair] = (int)bp;
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------
// Tile scan (v4).  In the cell-major kernel above a warp requests 12 KB of its prototype stream, waits for it, computes, and
// only then requests again.  Here the stream is decoupled from the arithmetic:
//   * persistent CTAs (one per SM, 8 consumer warps + 1 producer warp); the work is the list of 16-prototype TILES of all
//     touched (geocell, query pass) pairs in cell order, cut into gridDim.x equal contiguous ranges (no tail, no wave
//     quantisation); a geocell that straddles two ranges is merged through a 64-bit atomicMin on (d2 bits, prototype);
//   * the producer warp copies each tile (16 rows x D floats) into a shared-memory ring with one cp.async.bulk per row,
//     completion on an mbarrier, and pulls the tiles kPrefetchTiles further ahead into L2 (cp.async.bulk.prefetch.L2),
//     so HBM latency is hidden by L2 depth rather than by shared memory;
//   * up to QS queries of the geocell sit in shared memory for the whole pass, interleaved in pairs (one ffma2 advances
//     two queries); the 8 consumer warps split D eight ways, each computing a 16 x QS block of partial dot products with
//     a 2-prototype x NCH-pair register tile per thread (lanes = 8 prototype groups x 4 query groups: every LDS.128 is a
//     single conflict-free wavefront thanks to the 16-byte row padding), then add the eight partials in a fixed order
//     through shared memory -> d2 = |p|^2 + |q|^2 - 2 p.q with |p|^2 precomputed per bank (proto_sqnorm).
// Every (prototype, query) distance is computed by the same instruction sequence wherever the tile lands, so a sharded bank
// reproduces the single-GPU selections bit for bit.
// ------------------------------------------------------------------------------------------------
constexpr int kTP = 16;                 // prototypes per tile = one ring stage
constexpr int kTileWarps = 8;           // consumer warps (D split 8 ways)
constexpr int kTileConsumers = kTileWarps * 32;
constexpr int kTileThreads = kTileConsumers + 32;
constexpr int kPrefetchTiles = 3;       // L2 prefetch distance in tiles

template <int NV4, int QS>
struct TileCfg {
  static constexpr int D = NV4 * 128;
  static constexpr int KS = D / kTileWarps;            // columns per consumer warp
  static constexpr int QROW = 2 * D + 4;               // floats per staged query-pair row (16 B pad: conflict-free)
  static constexpr int PROW = D + 4;                   // floats per staged prototype row
  static constexpr int SROW = QS + 8;                  // floats per row of partial sums
  static constexpr int NST = (D <= 512) ? 4 : 2;       // ring stages
  static constexpr int RG = kTileConsumers / QS;       // prototype rows covered by one sweep of the reduce threads
  static constexpr int RPT = kTP / RG;                 // rows per reduce thread
  static constexpr size_t q_bytes = (size_t)(QS / 2) * QROW * 4;
  static constexpr size_t p_bytes = (size_t)NST * kTP * PROW * 4;
  static constexpr size_t s_bytes = (size_t)kTileWarps * kTP * SROW * 4;
  static constexpr size_t rb_bytes = (size_t)kTileConsumers * 8;
  static constexpr size_t qn_bytes = (size_t)QS * 4;
  static constexpr size_t bar_bytes = 2 * NST * 8;
  static constexpr size_t smem = q_bytes + p_bytes + s_bytes + rb_bytes + qn_bytes + bar_bytes;
  static_assert(KS % 8 == 0 && kTP % RG == 0, "tile geometry");
  static_assert(smem <= 227 * 1024, "shared memory budget");
};

// Walks the units [x, x_hi) of the global work list (UNIT prototypes each): one item = consecutive units of one
// (geocell, query pass).
template <int UNIT>
struct UnitWalk {
  long long x, x_hi;
  int c;                  // current geocell
  long lo;                // its first prototype
  int Pc, tpc;            // prototypes / tiles of the geocell
  int pair0, n_pairs;     // its sorted pairs
  int pass, t0, t1;       // query pass, tile range of this item
  __device__ __forceinline__ void init(long long x0, long long x1, const int* __restrict__ tile_prefix, int C) {
    x = x0; x_hi = x1;
    int a = 0, b = C;     // largest c with tile_prefix[c] <= x0
    while (b - a > 1) { const int m = (a + b) >> 1; if (tile_prefix[m] <= x0) a = m; else b = m; }
    c = a;
  }
  __device__ __forceinline__ bool next(const RefinerBank& bank, const int* __restrict__ cell_start,
                                       const int* __restrict__ tile_prefix) {
    if (x >= x_hi) return false;
    while (tile_prefix[c + 1] <= x) ++c;
    lo = bank.cell_off[c];
    Pc = (int)(bank.cell_off[c + 1] - lo);
    tpc = (Pc + UNIT - 1) / UNIT;
    pair0 = cell_start[c];
    n_pairs = cell_start[c + 1] - pair0;
    const int local = (int)(x - tile_prefix[c]);
    pass = local / tpc;
    t0 = local % tpc;
    const long long rem = x_hi - x;
    t1 = (rem < (long long)(tpc - t0)) ? t0 + (int)rem : tpc;
    x += t1 - t0;
    return true;
  }
};

using TileWalk = UnitWalk<kTP>;

// The same walk one tile at a time (producer: one iterator for the copies, one running ahead for the L2 prefetch).
struct TileIter {
  TileWalk w;
  int t;
  bool valid;
  __device__ __forceinline__ void start(const RefinerBank& bank, const int* cell_start, const int* tile_prefix) {
    valid = w.next(bank, cell_start, tile_prefix);
    t = w.t0;
  }
  __device__ __forceinline__ void advance(const RefinerBank& bank, const int* cell_start, const int* tile_prefix) {
    if (++t >= w.t1) { valid = w.next(bank, cell_start, tile_prefix); t = w.t0; }
  }
};

__device__ __forceinline__ void consumer_bar() { asm volatile("bar.sync 1, %0;" ::"n"(kTileConsumers) : "memory"); }

// One item of the walk on the consumer side: NCH chunks of 8 staged queries against tiles [t0, t1).
template <int NV4, int QS, int NCH>
__device__ __forceinline__ void tile_item(const RefinerBank& bank, const TileWalk& w, const float* __restrict__ qs,
                                          const float* __restrict__ ps, float* __restrict__ scratch,
                                          const float* __restrict__ qn, uint64_t* full, uint64_t* empty, int& stage,
                                          uint32_t& phase, float (&bd)[TileCfg<NV4, QS>::RPT],
                                          int (&bp)[TileCfg<NV4, QS>::RPT]) {
  using Cfg = TileCfg<NV4, QS>;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int g = lane >> 2, h = lane & 3;
  const int j = tid % QS, rr = tid / QS;
  for (int t = w.t0; t < w.t1; ++t) {
    // |p|^2 of the rows this thread reduces: requested before the wait, used after the arithmetic
    float pn[Cfg::RPT];
    bool ok[Cfg::RPT];
#pragma unroll
    for (int i = 0; i < Cfg::RPT; ++i) {
      const int idx = t * kTP + rr + i * Cfg::RG;
      ok[i] = idx < w.Pc;
      pn[i] = ok[i] ? __ldg(bank.proto_sqnorm + w.lo + idx) : 0.f;
    }
    mbar_wait(&full[stage], phase);
    const float* pa_ptr = ps + (size_t)(stage * kTP + g) * Cfg::PROW + warp * Cfg::KS;
    const float* pb_ptr = pa_ptr + 8 * Cfg::PROW;
    const float* q_ptr = qs + (size_t)h * Cfg::QROW + 2 * warp * Cfg::KS;
    float2 acc[2][NCH];
#pragma unroll
    for (int c = 0; c < NCH; ++c) { acc[0][c] = make_float2(0.f, 0.f); acc[1][c] = make_float2(0.f, 0.f); }
    // two register sets in ping-pong: the shared-memory loads of step k + 4 are in flight while step k is on the FMA pipe
    // (only two warps per scheduler: nothing else would hide the LDS latency)
    struct Step { float4 pa, pb, q0[NCH], q1[NCH]; };
    auto load = [&](Step& s, int k) {
      s.pa = *reinterpret_cast<const float4*>(pa_ptr + k);
      s.pb = *reinterpret_cast<const float4*>(pb_ptr + k);
#pragma unroll
      for (int c = 0; c < NCH; ++c) {
        s.q0[c] = *reinterpret_cast<const float4*>(q_ptr + (size_t)c * 4 * Cfg::QROW + 2 * k);
        s.q1[c] = *reinterpret_cast<const float4*>(q_ptr + (size_t)c * 4 * Cfg::QROW + 2 * k + 4);
      }
    };
    auto fma = [&](const Step& s) {
#pragma unroll
      for (int c = 0; c < NCH; ++c) {
        acc[0][c] = ffma2(make_float2(s.pa.x, s.pa.x), make_float2(s.q0[c].x, s.q0[c].y), acc[0][c]);
        acc[1][c] = ffma2(make_float2(s.pb.x, s.pb.x), make_float2(s.q0[c].x, s.q0[c].y), acc[1][c]);
        acc[0][c] = ffma2(make_float2(s.pa.y, s.pa.y), make_float2(s.q0[c].z, s.q0[c].w), acc[0][c]);
        acc[1][c] = ffma2(make_float2(s.pb.y, s.pb.y), make_float2(s.q0[c].z, s.q0[c].w), acc[1][c]);
        acc[0][c] = ffma2(make_float2(s.pa.z, s.pa.z), make_float2(s.q1[c].x, s.q1[c].y), acc[0][c]);
        acc[1][c] = ffma2(make_float2(s.pb.z, s.pb.z), make_float2(s.q1[c].x, s.q1[c].y), acc[1][c]);
        acc[0][c] = ffma2(make_float2(s.pa.w, s.pa.w), make_float2(s.q1[c].z, s.q1[c].w), acc[0][c]);
        acc[1][c] = ffma2(make_float2(s.pb.w, s.pb.w), make_float2(s.q1[c].z, s.q1[c].w), acc[1][c]);
      }
    };
    Step sa, sb;
    load(sa, 0);
#pragma unroll 1
    for (int k = 0; k < Cfg::KS; k += 8) {
      load(sb, k + 4);
      fma(sa);
      if (k + 8 < Cfg::KS) load(sa, k + 8);
      fma(sb);
    }
    // this warp's slice of the 16 x (8 NCH) dot products; the ring slot is free once every warp has read it
#pragma unroll
    for (int c = 0; c < NCH; ++c) {
      *reinterpret_cast<float2*>(scratch + (size_t)(warp * kTP + g) * Cfg::SROW + c * 8 + 2 * h) = acc[0][c];
      *reinterpret_cast<float2*>(scratch + (size_t)(warp * kTP + g + 8) * Cfg::SROW + c * 8 + 2 * h) = acc[1][c];
    }
    __syncwarp();
    if (lane == 0) mbar_arrive(&empty[stage]);
    if (++stage == Cfg::NST) { stage = 0; phase ^= 1; }
    consumer_bar();
    if (j < 8 * NCH) {
      const float qnj = qn[j];
#pragma unroll
      for (int i = 0; i < Cfg::RPT; ++i) {
        const int row = rr + i * Cfg::RG;
        float dot = scratch[(size_t)row * Cfg::SROW + j];
#pragma unroll
        for (int ww = 1; ww < kTileWarps; ++ww) dot += scratch[(size_t)(ww * kTP + row) * Cfg::SROW + j];
        const float d2 = ok[i] ? fmaxf(pn[i] + qnj - 2.f * dot, 0.f) + 0.f : INFINITY;
        if (d2 < bd[i]) { bd[i] = d2; bp[i] = t * kTP + row; }   // strict: first minimum wins
      }
    }
    consumer_bar();
  }
}

template <int NV4, int QS>
__global__ void __launch_bounds__(kTileThreads, 1)
tile_scan_kernel(const RefinerBank bank, const float* __restrict__ q, const int* __restrict__ cell_start,
                 const int* __restrict__ order, const int* __restrict__ tile_prefix, int topk,
                 unsigned long long* __restrict__ best_packed) {
  using Cfg = TileCfg<NV4, QS>;
  constexpr int D = Cfg::D;
  extern __shared__ __align__(128) unsigned char tile_smem[];
  float* qs = reinterpret_cast<float*>(tile_smem);
  float* ps = reinterpret_cast<float*>(tile_smem + Cfg::q_bytes);
  float* scratch = reinterpret_cast<float*>(tile_smem + Cfg::q_bytes + Cfg::p_bytes);
  float* rb_d = reinterpret_cast<float*>(tile_smem + Cfg::q_bytes + Cfg::p_bytes + Cfg::s_bytes);
  int* rb_p = reinterpret_cast<int*>(rb_d + kTileConsumers);
  float* qn = reinterpret_cast<float*>(rb_p + kTileConsumers);
  uint64_t* full = reinterpret_cast<uint64_t*>(qn + QS);
  uint64_t* empty = full + Cfg::NST;

  const int C = bank.num_cells;
  const long long T = tile_prefix[C];
  const long long x_lo = T * blockIdx.x / gridDim.x, x_hi = T * (blockIdx.x + 1) / gridDim.x;
  if (threadIdx.x == 0) {
    for (int s = 0; s < Cfg::NST; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], kTileWarps); }
    fence_mbar_init();
  }
  __syncthreads();
  if (x_lo >= x_hi) return;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;

  if (warp == kTileWarps) {
    // ---------------------------------------------------------------- producer: ring copies + L2 prefetch ahead
    TileIter ld, pf;
    ld.w.init(x_lo, x_hi, tile_prefix, C);
    pf.w = ld.w;
    ld.start(bank, cell_start, tile_prefix);
    pf.start(bank, cell_start, tile_prefix);
    auto prefetch = [&](const TileIter& it) {   // the rows of a tile are contiguous in the bank: one request
      const int row0 = it.t * kTP;
      if (lane == 0)
        bulk_prefetch_l2(bank.proto_emb + (size_t)(it.w.lo + row0) * D, (uint32_t)min(kTP, it.w.Pc - row0) * D * 4);
    };
    for (int i = 0; i < kPrefetchTiles && pf.valid; ++i) { prefetch(pf); pf.advance(bank, cell_start, tile_prefix); }
    int stage = 0;
    uint32_t phase = 0;
    while (ld.valid) {
      if (pf.valid) { prefetch(pf); pf.advance(bank, cell_start, tile_prefix); }
      const int row0 = ld.t * kTP;
      const int nrows = min(kTP, ld.w.Pc - row0);
      mbar_wait(&empty[stage], phase ^ 1);
      if (lane == 0) mbar_arrive_expect_tx(&full[stage], (uint32_t)nrows * D * 4);
      __syncwarp();
      if (lane < nrows)
        bulk_load_1d(ps + (size_t)(stage * kTP + lane) * Cfg::PROW, bank.proto_emb + (size_t)(ld.w.lo + row0 + lane) * D,
                     D * 4, &full[stage]);
      if (++stage == Cfg::NST) { stage = 0; phase ^= 1; }
      ld.advance(bank, cell_start, tile_prefix);
    }
    return;
  }

  // ------------------------------------------------------------------ consumers
  TileWalk w;
  w.init(x_lo, x_hi, tile_prefix, C);
  int stage = 0;
  uint32_t phase = 0;
  while (w.next(bank, cell_start, tile_prefix)) {
    const int nq = min(QS, w.n_pairs - w.pass * QS);
    const int nch = (nq + 7) >> 3;
    const int* ord = order + w.pair0 + w.pass * QS;
    consumer_bar();   // the previous item's readers are done with qs / qn / rb
    // stage the queries two by two: pair row u holds (qA[k], qB[k]) interleaved, A = 2u, B = 2u + 1; missing ones are zero
    for (int idx = tid; idx < 4 * nch * (D / 4); idx += kTileConsumers) {
      const int u = idx / (D / 4), i4 = idx % (D / 4);
      float4 a = make_float4(0.f, 0.f, 0.f, 0.f), b = a;
      if (2 * u < nq) a = reinterpret_cast<const float4*>(q + (size_t)(ord[2 * u] / topk) * D)[i4];
      if (2 * u + 1 < nq) b = reinterpret_cast<const float4*>(q + (size_t)(ord[2 * u + 1] / topk) * D)[i4];
      float* dst = qs + (size_t)u * Cfg::QROW + 8 * i4;
      *reinterpret_cast<float4*>(dst) = make_float4(a.x, b.x, a.y, b.y);
      *reinterpret_cast<float4*>(dst + 4) = make_float4(a.z, b.z, a.w, b.w);
    }
    for (int qi = warp; qi < 8 * nch; qi += kTileWarps) {   // |q|^2, warp per query
      float acc_q = 0.f;
      if (qi < nq) {
        const float4* q4 = reinterpret_cast<const float4*>(q + (size_t)(ord[qi] / topk) * D);
#pragma unroll
        for (int i = 0; i < NV4; ++i) {
          const float4 t = q4[lane + 32 * i];
          acc_q = fmaf(t.x, t.x, acc_q); acc_q = fmaf(t.y, t.y, acc_q);
          acc_q = fmaf(t.z, t.z, acc_q); acc_q = fmaf(t.w, t.w, acc_q);
        }
      }
      acc_q = warp_sum(acc_q);
      if (lane == 0) qn[qi] = acc_q;
    }
    consumer_bar();
    float bd[Cfg::RPT];
    int bp[Cfg::RPT];
#pragma unroll
    for (int i = 0; i < Cfg::RPT; ++i) { bd[i] = INFINITY; bp[i] = 0x7fffffff; }
    switch (nch) {
      case 1: tile_item<NV4, QS, 1>(bank, w, qs, ps, scratch, qn, full, empty, stage, phase, bd, bp); break;
      case 2: tile_item<NV4, QS, 2>(bank, w, qs, ps, scratch, qn, full, empty, stage, phase, bd, bp); break;
      case 3: if constexpr (QS >= 24) tile_item<NV4, QS, 3>(bank, w, qs, ps, scratch, qn, full, empty, stage, phase, bd, bp); break;
      default: if constexpr (QS >= 32) tile_item<NV4, QS, 4>(bank, w, qs, ps, scratch, qn, full, empty, stage, phase, bd, bp); break;
    }
    // rows of one thread ascend, so do the groups rr: lexicographic (d2, prototype) minimum over the RG groups
    float d = bd[0];
    int pi = bp[0];
#pragma unroll
    for (int i = 1; i < Cfg::RPT; ++i) if (bd[i] < d || (bd[i] == d && bp[i] < pi)) { d = bd[i]; pi = bp[i]; }
    rb_d[tid] = d;
    rb_p[tid] = pi;
    consumer_bar();
    if (tid < nq) {
      for (int r = 0; r < Cfg::RG; ++r) {
        const float od = rb_d[r * QS + tid];
        const int op = rb_p[r * QS + tid];
        if (od < d || (od == d && op < pi)) { d = od; pi = op; }
      }
      const unsigned long long packed = ((unsigned long long)__float_as_uint(d) << 32) | (unsigned int)pi;
      atomicMin(&best_packed[ord[tid]], packed);
    }
  }
}

// ------------------------------------------------------------------------------------------------
// Slab scan (v5).  A kernel whose operands come from shared memory does more arithmetic per delivered float the larger its
// register tile: the tile scan's 2 x 2NCH tile does 1.5 FMA per float, the cell-major kernel 4 but it pays a 31-shuffle
// reduction per 32 results.  This kernel uses the 8-prototype x 8-query outer-product tile (4 FMA per float) without any
// cross-lane reduction:
//   * a warp owns a SLAB of 64 prototypes (lanes = 8 prototype groups x 4 query groups; thread = 8 prototypes x up to 4
//     query pairs, accumulators in registers over the whole embedding), a CTA up to 8 consecutive slabs of one geocell;
//   * the embedding dimension is streamed in chunks of 32 floats: one TMA box of [256 prototypes x 128 bytes] per half tile
//     (tensor map over the bank, 128-byte swizzle -> conflict-free LDS.128 of 8 rows), 3 stages of 64 KB, mbarrier ring;
//   * the query chunk [32 queries x 32 floats] is gathered by the consumer threads one chunk ahead (registers -> double
//     buffer, pairs interleaved for ffma2, rows padded by 16 bytes);
//   * d2 = |p|^2 + |q|^2 - 2 p.q, minimum over the thread's prototypes, three shuffles across the prototype groups, one
//     packed atomicMin per (warp, query): partition-independent like the tile scan.
// Work list = slabs of all touched (geocell, query pass) pairs, cut into gridDim.x equal contiguous ranges.
// Meant for banks whose geocells hold hundreds of prototypes (BASELINE configs[4]: 482 on average).
// ------------------------------------------------------------------------------------------------
constexpr int kSlab = 64;
constexpr int kSlabWarps = 8;
constexpr int kSlabConsumers = kSlabWarps * 32;
constexpr int kSlabThreads = kSlabConsumers + 32;
constexpr int kKC = 32;                                   // floats per embedding chunk (128 bytes)
constexpr int kSlabStages = 3;
constexpr int kBoxRows = 256;
constexpr int kBoxBytes = kBoxRows * kKC * 4;             // 32 KB
constexpr int kPStageBytes = 2 * kBoxBytes;               // 512 prototypes x 128 B
constexpr int kQS = 32;                                   // queries per pass
constexpr int kQRowF4 = 17;                               // float4 per query-pair row of a chunk (16 + 1 pad)
constexpr int kQBufBytes = (kQS / 2) * kQRowF4 * 16;
constexpr int kSlabSmem = kSlabStages * kPStageBytes + 2 * kQBufBytes + kQS * 4 + 2 * kSlabStages * 8 + 1024;
using SlabWalk = UnitWalk<kSlab>;

__device__ __forceinline__ void slab_bar() { asm volatile("bar.sync 1, %0;" ::"n"(kSlabConsumers) : "memory"); }

template <int NJ>
__device__ __forceinline__ void slab_item(const RefinerBank& bank, const SlabWalk& w, const float* __restrict__ q, int D,
                                          int topk, const int* __restrict__ ord, int nq, uint32_t pstages,
                                          uint32_t qbuf, const float* __restrict__ qn, uint64_t* full, uint64_t* empty,
                                          int& stage, uint32_t& phase, unsigned long long* __restrict__ best_packed) {
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int g = lane >> 2, h = lane & 3;
  const int nchunks = D / kKC;
  // query-chunk gather: thread = (pair row u, float2 slot part)
  const int u = tid >> 4, part = tid & 15;
  const bool stage_q = u < 4 * NJ;
  const float* qa = (2 * u < nq) ? q + (size_t)(ord[2 * u] / topk) * D + 2 * part : nullptr;
  const float* qb = (2 * u + 1 < nq) ? q + (size_t)(ord[2 * u + 1] / topk) * D + 2 * part : nullptr;
  auto fetch = [&](int c, float2& a, float2& b) {
    a = make_float2(0.f, 0.f); b = a;
    if (qa) a = *reinterpret_cast<const float2*>(qa + c * kKC);
    if (qb) b = *reinterpret_cast<const float2*>(qb + c * kKC);
  };
  for (int s0 = w.t0; s0 < w.t1; s0 += kSlabWarps) {
    const int slab = s0 + warp;
    const bool active = slab < w.t1;
    float pn[8];
    bool ok[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const int idx = slab * kSlab + g + 8 * i;
      ok[i] = active && idx < w.Pc;
      pn[i] = ok[i] ? __ldg(bank.proto_sqnorm + w.lo + idx) : 0.f;
    }
    float2 acc[8][NJ];
#pragma unroll
    for (int i = 0; i < 8; ++i)
#pragma unroll
      for (int j = 0; j < NJ; ++j) acc[i][j] = make_float2(0.f, 0.f);
    float2 ra, rb;
    fetch(0, ra, rb);
    slab_bar();   // every warp is done with both query buffers (previous tile / item)
    if (stage_q) sts_f4(qbuf + (u * kQRowF4 + part) * 16, make_float4(ra.x, rb.x, ra.y, rb.y));
    slab_bar();
    // this warp's rows inside the stage: box (rows 0..255 | 256..511), row & 7 == g
    const uint32_t prow = (uint32_t)((warp * kSlab) >> 8) * kBoxBytes + (uint32_t)((warp * kSlab) & 255) * 128 + g * 128;
    for (int c = 0; c < nchunks; ++c) {
      if (c + 1 < nchunks) fetch(c + 1, ra, rb);
      mbar_wait(&full[stage], phase);
      if (active) {
        const uint32_t pw = pstages + (uint32_t)stage * kPStageBytes + prow;
        const uint32_t qv = qbuf + ((c & 1) * ((kQS / 2) * kQRowF4) + h * kQRowF4) * 16;
#pragma unroll 2
        for (int c4 = 0; c4 < kKC / 4; ++c4) {
          float4 p[8], q0[NJ], q1[NJ];
#pragma unroll
          for (int i = 0; i < 8; ++i) p[i] = lds_f4(pw + i * 8 * 128 + ((c4 ^ g) << 4));
#pragma unroll
          for (int j = 0; j < NJ; ++j) { q0[j] = lds_f4(qv + (4 * j * kQRowF4 + 2 * c4) * 16); q1[j] = lds_f4(qv + (4 * j * kQRowF4 + 2 * c4 + 1) * 16); }
#pragma unroll
          for (int i = 0; i < 8; ++i)
#pragma unroll
            for (int j = 0; j < NJ; ++j) {
              acc[i][j] = ffma2(make_float2(p[i].x, p[i].x), make_float2(q0[j].x, q0[j].y), acc[i][j]);
              acc[i][j] = ffma2(make_float2(p[i].y, p[i].y), make_float2(q0[j].z, q0[j].w), acc[i][j]);
              acc[i][j] = ffma2(make_float2(p[i].z, p[i].z), make_float2(q1[j].x, q1[j].y), acc[i][j]);
              acc[i][j] = ffma2(make_float2(p[i].w, p[i].w), make_float2(q1[j].z, q1[j].w), acc[i][j]);
            }
        }
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(&empty[stage]);
      if (++stage == kSlabStages) { stage = 0; phase ^= 1; }
      if (c + 1 < nchunks) {
        if (stage_q) sts_f4(qbuf + (((c + 1) & 1) * ((kQS / 2) * kQRowF4) + u * kQRowF4 + part) * 16, make_float4(ra.x, rb.x, ra.y, rb.y));
        slab_bar();
      }
    }
    if (active) {
#pragma unroll
      for (int j = 0; j < NJ; ++j) {
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int qi = 8 * j + 2 * h + e;
          const float qnj = qn[qi];
          float bd = INFINITY;
          int bp = 0x7fffffff;
#pragma unroll
          for (int i = 0; i < 8; ++i) {   // rows ascend with i: strict < keeps the first minimum
            const float dot = e ? acc[i][j].y : acc[i][j].x;
            const float d2 = ok[i] ? fmaxf(pn[i] + qnj - 2.f * dot, 0.f) + 0.f : INFINITY;
            if (d2 < bd) { bd = d2; bp = slab * kSlab + g + 8 * i; }
          }
#pragma unroll
          for (int o = 4; o <= 16; o <<= 1) {   // across the 8 prototype groups (lanes with the same h)
            const float od = __shfl_xor_sync(0xffffffffu, bd, o);
            const int op = __shfl_xor_sync(0xffffffffu, bp, o);
            if (od < bd || (od == bd && op < bp)) { bd = od; bp = op; }
          }
          if (g == 0 && qi < nq) {
            const unsigned long long packed = ((unsigned long long)__float_as_uint(bd) << 32) | (unsigned int)bp;
            atomicMin(&best_packed[ord[qi]], packed);
          }
        }
      }
    }
  }
}

__global__ void __launch_bounds__(kSlabThreads, 1)
slab_scan_kernel(const __grid_constant__ CUtensorMap tmap_p, const RefinerBank bank, const float* __restrict__ q,
                 const int* __restrict__ cell_start, const int* __restrict__ order, const int* __restrict__ slab_prefix,
                 int topk, unsigned long long* __restrict__ best_packed) {
  extern __shared__ uint8_t slab_smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(slab_smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* pstages = smem;
  float4* qbuf = reinterpret_cast<float4*>(smem + kSlabStages * kPStageBytes);
  float* qn = reinterpret_cast<float*>(smem + kSlabStages * kPStageBytes + 2 * kQBufBytes);
  uint64_t* full = reinterpret_cast<uint64_t*>(qn + kQS);
  uint64_t* empty = full + kSlabStages;

  const int C = bank.num_cells, D = bank.dim;
  const long long T = slab_prefix[C];
  const long long x_lo = T * blockIdx.x / gridDim.x, x_hi = T * (blockIdx.x + 1) / gridDim.x;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  if (tid == 0) {
    tma_prefetch_desc(&tmap_p);
    for (int s = 0; s < kSlabStages; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], kSlabWarps); }
    fence_mbar_init();
  }
  __syncthreads();
  if (x_lo >= x_hi) return;

  if (warp == kSlabWarps) {
    // ---------------------------------------------------------------- producer: TMA boxes of [256 prototypes x 32 floats]
    if (lane == 0) {
      SlabWalk w;
      w.init(x_lo, x_hi, slab_prefix, C);
      int stage = 0;
      uint32_t phase = 0;
      const int nchunks = D / kKC;
      while (w.next(bank, cell_start, slab_prefix)) {
        for (int s0 = w.t0; s0 < w.t1; s0 += kSlabWarps) {
          const int nslabs = min(kSlabWarps, w.t1 - s0);
          const int rows = min(nslabs * kSlab, w.Pc - s0 * kSlab);
          const int nbox = (rows + kBoxRows - 1) / kBoxRows;
          const long row0 = w.lo + (long)s0 * kSlab;
          for (int c = 0; c < nchunks; ++c) {
            mbar_wait(&empty[stage], phase ^ 1);
            mbar_arrive_expect_tx(&full[stage], (uint32_t)nbox * kBoxBytes);
            for (int b = 0; b < nbox; ++b)
              tma_load_2d(pstages + (size_t)stage * kPStageBytes + (size_t)b * kBoxBytes, &tmap_p, &full[stage], c * kKC,
                          (int32_t)(row0 + (long)b * kBoxRows));
            if (++stage == kSlabStages) { stage = 0; phase ^= 1; }
          }
        }
      }
    }
    return;
  }

  // ------------------------------------------------------------------ consumers
  SlabWalk w;
  w.init(x_lo, x_hi, slab_prefix, C);
  int stage = 0;
  uint32_t phase = 0;
  while (w.next(bank, cell_start, slab_prefix)) {
    const int nq = min(kQS, w.n_pairs - w.pass * kQS);
    const int nj = (nq + 7) >> 3;
    const int* ord = order + w.pair0 + w.pass * kQS;
    slab_bar();   // the previous item's readers are done with qn
    for (int qi = warp; qi < kQS; qi += kSlabWarps) {   // |q|^2, warp per query
      float acc_q = 0.f;
      if (qi < nq) {
        const float4* q4 = reinterpret_cast<const float4*>(q + (size_t)(ord[qi] / topk) * D);
        for (int i = lane; i < D / 4; i += 32) {
          const float4 t = q4[i];
          acc_q = fmaf(t.x, t.x, acc_q); acc_q = fmaf(t.y, t.y, acc_q);
          acc_q = fmaf(t.z, t.z, acc_q); acc_q = fmaf(t.w, t.w, acc_q);
        }
      }
      acc_q = warp_sum(acc_q);
      if (lane == 0) qn[qi] = acc_q;
    }
    slab_bar();
    switch (nj) {
      case 1: slab_item<1>(bank, w, q, D, topk, ord, nq, smem_u32(pstages), smem_u32(qbuf), qn, full, empty, stage, phase, best_packed); break;
      case 2: slab_item<2>(bank, w, q, D, topk, ord, nq, smem_u32(pstages), smem_u32(qbuf), qn, full, empty, stage, phase, best_packed); break;
      case 3: slab_item<3>(bank, w, q, D, topk, ord, nq, smem_u32(pstages), smem_u32(qbuf), qn, full, empty, stage, phase, best_packed); break;
      default: slab_item<4>(bank, w, q, D, topk, ord, nq, smem_u32(pstages), smem_u32(qbuf), qn, full, empty, stage, phase, best_packed); break;
    }
  }
}

// After the tile scan: decode the packed winner of every live pair, farthest-member pick (:233-255), outputs.
template <int NV4>
__global__ void __launch_bounds__(256)
tile_finish_kernel(const RefinerBank bank, const float* __restrict__ q, const long long* __restrict__ cand,
                   int cand_stride, const int* __restrict__ order, const int* __restrict__ n_live, int topk,
                   const unsigned long long* __restrict__ best_packed, float* __restrict__ best_logit,
                   float* __restrict__ best_lnglat, int* __restrict__ best_proto) {
  constexpr int D = NV4 * 128;
  const int lane = threadIdx.x & 31;
  const int warps = (gridDim.x * blockDim.x) >> 5;
  const int live = *n_live;
  for (int i = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; i < live; i += warps) {
    const long pair = order[i];
    const long b = pair / topk;
    const int jj = (int)(pair % topk);
    const long long cell = cand[b * cand_stride + jj];
    const unsigned long long packed = best_packed[pair];
    const float bd = __uint_as_float((unsigned int)(packed >> 32));
    const long bp = bank.cell_off[cell] + (long)(unsigned int)(packed & 0xffffffffull);
    float lng = bank.proto_lnglat[2 * bp], lat = bank.proto_lnglat[2 * bp + 1];
    if (bank.proto_count[bp] != 1) {
      float4 qv[NV4];
      const float4* q4 = reinterpret_cast<const float4*>(q + b * D);
#pragma unroll
      for (int k = 0; k < NV4; ++k) qv[k] = q4[lane + 32 * k];
      const long mlo = bank.member_off[bp], mhi = bank.member_off[bp + 1];
      float far = -INFINITY;
      long bm = -1;
      for (long mi = mlo; mi < mhi; ++mi) {
        const long idx = bank.member_idx[mi];
        const float dd = sqdist<NV4>(qv, bank.data_emb + idx * D, lane);
        if (dd > far) { far = dd; bm = idx; }
      }
      if (bm >= 0) { lng = bank.data_lnglat[2 * bm]; lat = bank.data_lnglat[2 * bm + 1]; }
    }
    if (lane == 0) {
      best_logit[pair] = -sqrtf(bd);
      best_lnglat[2 * pair] = lng;
      best_lnglat[2 * pair + 1] = lat;
      best_proto[pair] = (int)bp;
    }
  }
}

// exclusive scans of the pair counts (-> cell_start, cursors zeroed) and of the tile counts (-> tile_prefix) of the cells:
// units(c) = ceil(n_pairs(c) / qs) query passes x ceil(P_c / unit_rows) prototype units.  Single block.
__global__ void cell_tile_offsets_kernel(const RefinerBank bank, const int* __restrict__ cell_cnt,
                                         int* __restrict__ cell_start, int* __restrict__ cursor,
                                         int* __restrict__ tile_prefix, int C, int qs, int unit_rows) {
  __shared__ int carry[2];
  __shared__ int warp_tot[2][32];
  if (threadIdx.x < 2) carry[threadIdx.x] = 0;
  __syncthreads();
  const int ln = threadIdx.x & 31, wp = threadIdx.x >> 5;
  for (int base = 0; base < C; base += blockDim.x) {
    const int i = base + threadIdx.x;
    int v[2] = {0, 0};
    if (i < C) {
      v[0] = cell_cnt[i];
      const int pc = (int)(bank.cell_off[i + 1] - bank.cell_off[i]);
      v[1] = ((v[0] + qs - 1) / qs) * ((pc + unit_rows - 1) / unit_rows);
    }
    int x[2] = {v[0], v[1]};
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
#pragma unroll
      for (int a = 0; a < 2; ++a) {
        const int y = __shfl_up_sync(0xffffffffu, x[a], o);
        if (ln >= o) x[a] += y;
      }
    }
    if (ln == 31) { warp_tot[0][wp] = x[0]; warp_tot[1][wp] = x[1]; }
    __syncthreads();
    if (threadIdx.x < 64) {
      const int a = threadIdx.x >> 5;
      int t = (ln < (int)(blockDim.x >> 5)) ? warp_tot[a][ln] : 0;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const int y = __shfl_up_sync(0xffffffffu, t, o);
        if (ln >= o) t += y;
      }
      warp_tot[a][ln] = t;
    }
    __syncthreads();
    const int off0 = wp ? warp_tot[0][wp - 1] : 0, off1 = wp ? warp_tot[1][wp - 1] : 0;
    if (i < C) {
      cell_start[i] = carry[0] + off0 + x[0] - v[0];
      tile_prefix[i] = carry[1] + off1 + x[1] - v[1];
      cursor[i] = 0;
    }
    __syncthreads();
    if (threadIdx.x == blockDim.x - 1) { carry[0] += off0 + x[0]; carry[1] += off1 + x[1]; }
    __syncthreads();
  }
  if (threadIdx.x == 0) { cell_start[C] = carry[0]; tile_prefix[C] = carry[1]; }
}

__global__ void proto_sqnorm_kernel(const float* __restrict__ proto_emb, long P, int D, float* __restrict__ out) {
  const int lane = threadIdx.x & 31;
  const long warps = ((long)gridDim.x * blockDim.x) >> 5;
  const int d4 = D >> 2;
  for (long p = ((long)blockIdx.x * blockDim.x + threadIdx.x) >> 5; p < P; p += warps) {
    const float4* r4 = reinterpret_cast<const float4*>(proto_emb + p * D);
    float t = 0.f;
    for (int c = lane; c < d4; c += 32) {
      const float4 v = __ldg(r4 + c);
      t = fmaf(v.x, v.x, t); t = fmaf(v.y, v.y, t); t = fmaf(v.z, v.z, t); t = fmaf(v.w, v.w, t);
    }
    t = warp_sum(t);
    if (lane == 0) out[p] = t;
  }
}

// ------------------------------------------------------------------------------------------------
// Bank builder (reference models/proto_refiner.py:359-378, `_compute_protos_for_cell`): prototype embedding = mean of its
// members' embeddings (members' 4-view mean first).  One warp per prototype, lanes strided over D as float4.
// ------------------------------------------------------------------------------------------------
__global__ void proto_mean_kernel(const float* __restrict__ data_emb, const long long* __restrict__ member_off,
                                  const long long* __restrict__ member_idx, long P, int D,
                                  float* __restrict__ proto_emb) {
  const int lane = threadIdx.x & 31;
  const long warps = ((long)gridDim.x * blockDim.x) >> 5;
  const int d4 = D >> 2;
  for (long p = ((long)blockIdx.x * blockDim.x + threadIdx.x) >> 5; p < P; p += warps) {
    const long lo = member_off[p], hi = member_off[p + 1];
    const float inv = 1.0f / (float)(hi - lo);
    for (int c = lane; c < d4; c += 32) {
      float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
      for (long mi = lo; mi < hi; ++mi) {
        const float4 v = __ldg(reinterpret_cast<const float4*>(data_emb + member_idx[mi] * D) + c);
        acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
      }
      reinterpret_cast<float4*>(proto_emb + p * D)[c] = make_float4(acc.x * inv, acc.y * inv, acc.z * inv, acc.w * inv);
    }
  }
}

// NaN ranks above everything, first index wins ties (torch.argmax).
__device__ __forceinline__ bool better(float v, float bv) {
  const bool vn = isnan(v), bn = isnan(bv);
  if (vn != bn) return vn;
  return v > bv;
}

// haversine(initial f64, refined f32) in km with the reference's type promotion (geo_utils.py:40-55):
// deg2rad of the fp32 point and the cosine of its latitude are fp32, everything else fp64.
__device__ double haversine_mixed(double lng0, double lat0, float lng1, float lat1) {
  const double kDeg = 3.14159265358979323846 / 180.0;
  const float kDegF = (float)kDeg;
  const double x_lng = lng0 * kDeg, x_lat = lat0 * kDeg;
  const float y_lng = lng1 * kDegF, y_lat = lat1 * kDegF;
  const double d_lng = (double)y_lng - x_lng, d_lat = (double)y_lat - x_lat;
  const double s_lat = sin(d_lat / 2), s_lng = sin(d_lng / 2);
  const double a = s_lat * s_lat + cos(x_lat) * (double)cosf(y_lat) * (s_lng * s_lng);
  const double c = 2 * asin(sqrt(a));
  return (6378137.0 * c) / 1000;
}

__global__ void finalize_kernel(const float* __restrict__ best_logit, const float* __restrict__ best_lnglat,
                                const long long* __restrict__ cand, const float* __restrict__ cand_prob,
                                int cand_stride, const double* __restrict__ init_lnglat, long B, int topk,
                                float temperature, double max_refinement, float* __restrict__ out_lnglat,
                                long long* __restrict__ out_cell, int* __restrict__ out_choice) {
  const long b = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  const float* lg = best_logit + b * topk;
  const float* cp = cand_prob + b * cand_stride;
  // temperature softmax without max-subtraction
  float sum = 0.f;
  for (int j = 0; j < topk; ++j) sum += expf(lg[j] / temperature);
  int refined = 0;
  float bestv = 0.f;
  int initial = 0;
  float besti = 0.f;
  for (int j = 0; j < topk; ++j) {
    const float pr = expf(lg[j] / temperature) / sum;
    const float f = cp[j] * pr;
    if (j == 0 || better(f, bestv)) { bestv = f; refined = j; }
    if (j == 0 || better(cp[j], besti)) { besti = cp[j]; initial = j; }
  }
  const float r_lng = best_lnglat[2 * (b * topk + refined)], r_lat = best_lnglat[2 * (b * topk + refined) + 1];
  const double dist = haversine_mixed(init_lnglat[2 * b], init_lnglat[2 * b + 1], r_lng, r_lat);
  // reference: `if distance > max_refinement: final_probs = c_probs[:topk]` -> falls back to the prior arg-max
  const int choice = (dist > max_refinement) ? initial : refined;
  out_lnglat[2 * b] = best_lnglat[2 * (b * topk + choice)];
  out_lnglat[2 * b + 1] = best_lnglat[2 * (b * topk + choice) + 1];
  out_cell[b] = cand[b * cand_stride + choice];
  if (out_choice) out_choice[b] = choice;
}

int check_launch(const char* what) {
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) { set_last_error("%s launch: %s", what, cudaGetErrorString(e)); return 1; }
  return 0;
}

}  // namespace

int refiner_pool(const float* emb, float* q, long B, int V, int D, cudaStream_t stream) {
  const long total = B * D;
  int grid = (int)((total + 255) / 256);
  if (grid > 8192) grid = 8192;
  ProfScope prof("refiner_pool", stream);
  pool_views_kernel<<<grid, 256, 0, stream>>>(emb, q, B, V, D);
  return check_launch("refiner_pool");
}

int refiner_scan(const RefinerBank& bank, const float* q, const long long* cand, int cand_stride, long B, int topk,
                 float* best_logit, float* best_lnglat, int* best_proto, int num_sms, cudaStream_t stream) {
  const long pairs = B * topk;
  if (pairs == 0) return 0;
  long blocks = (pairs + 7) / 8;
  const long cap = (long)num_sms * 8;
  if (blocks > cap) blocks = cap;
  const int grid = (int)blocks;
  ProfScope prof("refiner_scan", stream);
  switch (bank.dim / 128) {
#define PG_CASE(N)                                                                                           \
  case N:                                                                                                    \
    scan_kernel<N><<<grid, 256, 0, stream>>>(bank, q, cand, cand_stride, B, topk, best_logit, best_lnglat,   \
                                             best_proto);                                                    \
    break;
    PG_CASE(1) PG_CASE(2) PG_CASE(4) PG_CASE(6) PG_CASE(8)
#undef PG_CASE
    default:
      set_last_error("refiner: embedding dim %d unsupported (need 128*{1,2,4,6,8})", bank.dim);
      return 1;
  }
  if (bank.dim % 128) { set_last_error("refiner: embedding dim %d not a multiple of 128", bank.dim); return 1; }
  return check_launch("refiner_scan");
}

size_t refiner_sort_workspace_bytes(int num_cells, long pairs) {
  // cell_cnt, cell_start, cursor, tile_prefix [C+1] | order [pairs] | packed winners of the tile scan u64 [pairs]
  return (size_t)(4 * (num_cells + 1) + pairs + 2) * sizeof(int) + (size_t)pairs * 8 + 1024;
}

int refiner_scan_cell_major(const RefinerBank& bank, const float* q, const long long* cand, int cand_stride, long B,
                            int topk, void* sort_ws, float* best_logit, float* best_lnglat, int* best_proto,
                            int num_sms, cudaStream_t stream) {
  const long pairs = B * topk;
  if (pairs == 0) return 0;
  if (bank.dim % 128) { set_last_error("refiner: embedding dim %d not a multiple of 128", bank.dim); return 1; }
  const int C = bank.num_cells;
  int* cell_cnt = reinterpret_cast<int*>(sort_ws);
  int* cell_start = cell_cnt + (C + 1);
  int* cursor = cell_start + (C + 1);
  int* order = cursor + (C + 1);
  cudaError_t e = cudaMemsetAsync(cell_cnt, 0, (size_t)(C + 1) * sizeof(int), stream);
  if (e != cudaSuccess) { set_last_error("refiner: memset: %s", cudaGetErrorString(e)); return 1; }
  long blocks = (pairs + 255) / 256;
  if (blocks > (long)num_sms * 8) blocks = (long)num_sms * 8;
  {
    ProfScope prof("refiner_sort", stream);
    pair_hist_kernel<<<(int)blocks, 256, 0, stream>>>(bank, cand, cand_stride, B, topk, cell_cnt, best_logit, best_lnglat, best_proto);
    cell_scan_offsets_kernel<<<1, 1024, 0, stream>>>(cell_cnt, cell_start, cursor, C);
    pair_scatter_kernel<<<(int)blocks, 256, 0, stream>>>(bank, cand, cand_stride, B, topk, cell_start, cursor, order);
  }
  if (check_launch("refiner_sort")) return 1;
  // staged query set: QS = floor(96 KB / (D * 4)) rounded down to a multiple of 8 queries
  const size_t smem = (size_t)((kStageBytes / (bank.dim * 4)) / kQT * kQT) * bank.dim * sizeof(float);
  ProfScope prof("refiner_scan", stream);
  switch (bank.dim / 128) {
#define PG_CASE(N)                                                                                                   \
  case N: {                                                                                                          \
    auto kern = cell_major_scan_kernel<N>;                                                                           \
    if (smem > 48 * 1024) cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);        \
    kern<<<C, 256, smem, stream>>>(bank, q, cell_start, order, topk, best_logit, best_lnglat, best_proto);           \
    break;                                                                                                           \
  }
    PG_CASE(1) PG_CASE(2) PG_CASE(4) PG_CASE(6) PG_CASE(8)
#undef PG_CASE
    default:
      set_last_error("refiner: embedding dim %d unsupported (need 128*{1,2,4,6,8})", bank.dim);
      return 1;
  }
  return check_launch("refiner_scan_cell_major");
}

template <int NV4, int QS>
static int launch_tile_scan(const RefinerBank& bank, const float* q, const long long* cand, int cand_stride, int topk,
                            const int* cell_start, const int* order, const int* tile_prefix,
                            unsigned long long* best_packed, float* best_logit, float* best_lnglat, int* best_proto,
                            long pairs, int num_sms, cudaStream_t stream) {
  using Cfg = TileCfg<NV4, QS>;
  auto kern = tile_scan_kernel<NV4, QS>;
  cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)Cfg::smem);
  if (e != cudaSuccess) { set_last_error("refiner tile scan: shared memory attribute: %s", cudaGetErrorString(e)); return 1; }
  {
    ProfScope prof("refiner_scan", stream);
    kern<<<num_sms, kTileThreads, Cfg::smem, stream>>>(bank, q, cell_start, order, tile_prefix, topk, best_packed);
  }
  if (check_launch("refiner_tile_scan")) return 1;
  long blocks = (pairs + 7) / 8;
  if (blocks > (long)num_sms * 8) blocks = (long)num_sms * 8;
  ProfScope prof("refiner_scan_finish", stream);
  tile_finish_kernel<NV4><<<(int)blocks, 256, 0, stream>>>(bank, q, cand, cand_stride, order, cell_start + bank.num_cells,
                                                           topk, best_packed, best_logit, best_lnglat, best_proto);
  return check_launch("refiner_tile_finish");
}

int refiner_scan_tiles(const RefinerBank& bank, const float* q, const long long* cand, int cand_stride, long B, int topk,
                       void* sort_ws, float* best_logit, float* best_lnglat, int* best_proto, int num_sms,
                       cudaStream_t stream) {
  const long pairs = B * topk;
  if (pairs == 0) return 0;
  if (bank.dim % 128) { set_last_error("refiner: embedding dim %d not a multiple of 128", bank.dim); return 1; }
  if (!bank.proto_sqnorm) { set_last_error("refiner tile scan: bank.proto_sqnorm is null"); return 1; }
  if ((reinterpret_cast<uintptr_t>(bank.proto_emb) | reinterpret_cast<uintptr_t>(q)) & 15) {
    set_last_error("refiner tile scan: proto_emb / queries must be 16-byte aligned"); return 1;
  }
  const int C = bank.num_cells;
  int* cell_cnt = reinterpret_cast<int*>(sort_ws);
  int* cell_start = cell_cnt + (C + 1);
  int* cursor = cell_start + (C + 1);
  int* tile_prefix = cursor + (C + 1);
  int* order = tile_prefix + (C + 1);
  unsigned long long* best_packed =
      reinterpret_cast<unsigned long long*>((reinterpret_cast<uintptr_t>(order + pairs) + 7) & ~uintptr_t(7));
  cudaError_t e = cudaMemsetAsync(cell_cnt, 0, (size_t)(C + 1) * sizeof(int), stream);
  if (e != cudaSuccess) { set_last_error("refiner: memset: %s", cudaGetErrorString(e)); return 1; }
  long blocks = (pairs + 255) / 256;
  if (blocks > (long)num_sms * 8) blocks = (long)num_sms * 8;
  const int qs = bank.dim > 768 ? 16 : 32;
  {
    ProfScope prof("refiner_sort", stream);
    pair_hist_kernel<<<(int)blocks, 256, 0, stream>>>(bank, cand, cand_stride, B, topk, cell_cnt, best_logit, best_lnglat,
                                                      best_proto, best_packed);
    cell_tile_offsets_kernel<<<1, 1024, 0, stream>>>(bank, cell_cnt, cell_start, cursor, tile_prefix, C, qs, kTP);
    pair_scatter_kernel<<<(int)blocks, 256, 0, stream>>>(bank, cand, cand_stride, B, topk, cell_start, cursor, order);
  }
  if (check_launch("refiner_sort")) return 1;
  switch (bank.dim / 128) {
#define PG_CASE(N, Q)                                                                                                \
  case N:                                                                                                            \
    return launch_tile_scan<N, Q>(bank, q, cand, cand_stride, topk, cell_start, order, tile_prefix, best_packed,     \
                                  best_logit, best_lnglat, best_proto, pairs, num_sms, stream);
    PG_CASE(1, 32) PG_CASE(2, 32) PG_CASE(4, 32) PG_CASE(6, 32) PG_CASE(8, 16)
#undef PG_CASE
    default:
      set_last_error("refiner: embedding dim %d unsupported (need 128*{1,2,4,6,8})", bank.dim);
      return 1;
  }
}

int refiner_scan_slabs(const RefinerBank& bank, long num_protos, const float* q, const long long* cand, int cand_stride,
                       long B, int topk, void* sort_ws, float* best_logit, float* best_lnglat, int* best_proto,
                       int num_sms, cudaStream_t stream) {
  const long pairs = B * topk;
  if (pairs == 0) return 0;
  if (bank.dim % 128) { set_last_error("refiner: embedding dim %d not a multiple of 128", bank.dim); return 1; }
  if (!bank.proto_sqnorm) { set_last_error("refiner slab scan: bank.proto_sqnorm is null"); return 1; }
  if ((reinterpret_cast<uintptr_t>(bank.proto_emb) | reinterpret_cast<uintptr_t>(q)) & 15) {
    set_last_error("refiner slab scan: proto_emb / queries must be 16-byte aligned"); return 1;
  }
  CUtensorMap tp;
  if (make_tmap_f32_2d(&tp, bank.proto_emb, (uint64_t)num_protos, (uint64_t)bank.dim, (uint64_t)bank.dim, kBoxRows, kKC)) return 1;
  const int C = bank.num_cells;
  int* cell_cnt = reinterpret_cast<int*>(sort_ws);
  int* cell_start = cell_cnt + (C + 1);
  int* cursor = cell_start + (C + 1);
  int* slab_prefix = cursor + (C + 1);
  int* order = slab_prefix + (C + 1);
  unsigned long long* best_packed =
      reinterpret_cast<unsigned long long*>((reinterpret_cast<uintptr_t>(order + pairs) + 7) & ~uintptr_t(7));
  cudaError_t e = cudaMemsetAsync(cell_cnt, 0, (size_t)(C + 1) * sizeof(int), stream);
  if (e != cudaSuccess) { set_last_error("refiner: memset: %s", cudaGetErrorString(e)); return 1; }
  long blocks = (pairs + 255) / 256;
  if (blocks > (long)num_sms * 8) blocks = (long)num_sms * 8;
  {
    ProfScope prof("refiner_sort", stream);
    pair_hist_kernel<<<(int)blocks, 256, 0, stream>>>(bank, cand, cand_stride, B, topk, cell_cnt, best_logit, best_lnglat,
                                                      best_proto, best_packed);
    cell_tile_offsets_kernel<<<1, 1024, 0, stream>>>(bank, cell_cnt, cell_start, cursor, slab_prefix, C, kQS, kSlab);
    pair_scatter_kernel<<<(int)blocks, 256, 0, stream>>>(bank, cand, cand_stride, B, topk, cell_start, cursor, order);
  }
  if (check_launch("refiner_sort")) return 1;
  e = cudaFuncSetAttribute(slab_scan_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kSlabSmem);
  if (e != cudaSuccess) { set_last_error("refiner slab scan: shared memory attribute: %s", cudaGetErrorString(e)); return 1; }
  {
    ProfScope prof("refiner_scan", stream);
    slab_scan_kernel<<<num_sms, kSlabThreads, kSlabSmem, stream>>>(tp, bank, q, cell_start, order, slab_prefix, topk, best_packed);
  }
  if (check_launch("refiner_slab_scan")) return 1;
  long fblocks = (pairs + 7) / 8;
  if (fblocks > (long)num_sms * 8) fblocks = (long)num_sms * 8;
  ProfScope prof("refiner_scan_finish", stream);
  switch (bank.dim / 128) {
#define PG_CASE(N)                                                                                                       \
  case N:                                                                                                                \
    tile_finish_kernel<N><<<(int)fblocks, 256, 0, stream>>>(bank, q, cand, cand_stride, order, cell_start + C, topk,       \
                                                            best_packed, best_logit, best_lnglat, best_proto);           \
    break;
    PG_CASE(1) PG_CASE(2) PG_CASE(4) PG_CASE(6) PG_CASE(8)
#undef PG_CASE
    default:
      set_last_error("refiner: embedding dim %d unsupported (need 128*{1,2,4,6,8})", bank.dim);
      return 1;
  }
  return check_launch("refiner_tile_finish");
}

int refiner_bank_sqnorm(const float* proto_emb, long P, int D, float* out, int num_sms, cudaStream_t stream) {
  if (P == 0) return 0;
  if (D % 4) { set_last_error("refiner_bank_sqnorm: D=%d not a multiple of 4", D); return 1; }
  long blocks = (P + 7) / 8;
  if (blocks > (long)num_sms * 16) blocks = (long)num_sms * 16;
  ProfScope prof("bank_sqnorm", stream);
  proto_sqnorm_kernel<<<(int)blocks, 256, 0, stream>>>(proto_emb, P, D, out);
  return check_launch("bank_sqnorm");
}

int bank_build(const float* data_views, long N, int V, int D, const long long* member_off, const long long* member_idx,
               long P, float* data_mean, float* proto_emb, int num_sms, cudaStream_t stream) {
  if (D % 4) { set_last_error("bank_build: D=%d not a multiple of 4", D); return 1; }
  if (refiner_pool(data_views, data_mean, N, V, D, stream)) return 1;
  if (P == 0) return 0;
  long blocks = (P + 7) / 8;
  if (blocks > (long)num_sms * 16) blocks = (long)num_sms * 16;
  ProfScope prof("bank_proto_mean", stream);
  proto_mean_kernel<<<(int)blocks, 256, 0, stream>>>(data_mean, member_off, member_idx, P, D, proto_emb);
  return check_launch("bank_proto_mean");
}

int refiner_finalize(const float* best_logit, const float* best_lnglat, const long long* cand, const float* cand_prob,
                     int cand_stride, const double* init_lnglat, long B, int topk, float temperature,
                     double max_refinement, float* out_lnglat, long long* out_cell, int* out_choice,
                     cudaStream_t stream) {
  if (B == 0) return 0;
  const int grid = (int)((B + 127) / 128);
  ProfScope prof("refiner_finalize", stream);
  finalize_kernel<<<grid, 128, 0, stream>>>(best_logit, best_lnglat, cand, cand_prob, cand_stride, init_lnglat, B,
                                            topk, temperature, max_refinement, out_lnglat, out_cell, out_choice);
  return check_launch("refiner_finalize");
}

}  // namespace pg
