// Geocell head around the wgmma GEMM: restates reference models/super_guessr.py:437 (4-view mean),
// :447-448 (cell_layer Linear + softmax), :454-455 (argmax + centroid lookup), :459 (top-k).
//
// The Linear is evaluated on the fp16 tensor-core path at fp32-faithful accuracy by an error-compensated
// split: x = hi + lo, W = Whi + Wlo (all fp16) and logits = [hi | lo | hi] . [Whi | Whi | Wlo]^T, i.e. one
// GEMM with K = 3*D whose dropped term lo.Wlo is O(2^-22).
#include "head.h"

#include <cuda_fp16.h>
#include <math.h>
#include <stdint.h>

#include "prof.h"
#include "tma_host.h"

namespace pg {

namespace {

// in  : emb [B, V, D] fp32
// out : pooled [B, D] fp32 (mean over V, summed in view order then scaled, like torch.mean)
//       a3 [B, 3*D] fp16 = [hi | lo | hi]
__global__ void view_mean_split_kernel(const float* __restrict__ emb, float* __restrict__ pooled,
                                       __half* __restrict__ a3, int B, int V, int D) {
  const long total = (long)B * D;
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const int b = i / D, d = i % D;
    float s = 0.f;
    for (int v = 0; v < V; ++v) s += emb[((long)b * V + v) * D + d];
    const float x = s / V;
    pooled[i] = x;
    const __half hi = __float2half_rn(x);
    const __half lo = __float2half_rn(x - __half2float(hi));
    __half* row = a3 + (long)b * 3 * D;
    row[d] = hi;
    row[D + d] = lo;
    row[2 * D + d] = hi;
  }
}

// W [C, D] fp32 -> w3 [C, 3*D] fp16 = [Whi | Whi | Wlo]   (done once at handle creation)
__global__ void weight_split_kernel(const float* __restrict__ w, __half* __restrict__ w3, int C, int D) {
  const long total = (long)C * D;
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const int c = i / D, d = i % D;
    const float x = w[i];
    const __half hi = __float2half_rn(x);
    const __half lo = __float2half_rn(x - __half2float(hi));
    __half* row = w3 + (long)c * 3 * D;
    row[d] = hi;
    row[D + d] = hi;
    row[2 * D + d] = lo;
  }
}

struct ArgBest {
  float v;
  int i;
};
// "greater" with first-index tie-break; NaN ranks above everything (torch.argmax / topk semantics)
__device__ __forceinline__ bool better(float v, int i, float bv, int bi) {
  const bool vn = isnan(v), bn = isnan(bv);
  if (vn != bn) return vn;
  if (vn && bn) return i < bi;
  return (v > bv) || (v == bv && i < bi);
}
__device__ __forceinline__ ArgBest warp_best(ArgBest a) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float ov = __shfl_xor_sync(0xffffffffu, a.v, o);
    const int oi = __shfl_xor_sync(0xffffffffu, a.i, o);
    if (better(ov, oi, a.v, a.i)) { a.v = ov; a.i = oi; }
  }
  return a;
}

// One CTA per sample. logits [B, C] fp32 -> probs [B, C], pred cell, pred (lng, lat) f64, top-k.
__global__ void __launch_bounds__(256)
softmax_topk_kernel(const float* __restrict__ logits, float* __restrict__ probs, long long* __restrict__ pred_cell,
                    double* __restrict__ pred_lnglat, float* __restrict__ topk_val, long long* __restrict__ topk_idx,
                    const double* __restrict__ centroids, int C, int k) {
  extern __shared__ float sp[];  // C floats
  __shared__ float red_v[8];
  __shared__ int red_i[8];
  __shared__ float bcast;
  const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const float* lr = logits + (long)b * C;

  // row max
  float m = -INFINITY;
  for (int c = tid; c < C; c += 256) { const float x = lr[c]; sp[c] = x; m = fmaxf(m, x); }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  if (lane == 0) red_v[warp] = m;
  __syncthreads();
  if (tid == 0) { float t = red_v[0]; for (int w = 1; w < 8; ++w) t = fmaxf(t, red_v[w]); bcast = t; }
  __syncthreads();
  m = bcast;
  __syncthreads();
  // exp and sum
  float s = 0.f;
  for (int c = tid; c < C; c += 256) { const float e = expf(sp[c] - m); sp[c] = e; s += e; }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if (lane == 0) red_v[warp] = s;
  __syncthreads();
  if (tid == 0) { float t = 0.f; for (int w = 0; w < 8; ++w) t += red_v[w]; bcast = t; }
  __syncthreads();
  const float denom = bcast;
  for (int c = tid; c < C; c += 256) { const float p = sp[c] / denom; sp[c] = p; probs[(long)b * C + c] = p; }
  __syncthreads();

  // top-k by repeated block arg-max with removal; iteration 0 is the arg-max prediction
  for (int j = 0; j < k; ++j) {
    ArgBest best{-INFINITY, 0x7fffffff};
    for (int c = tid; c < C; c += 256) {
      const float p = sp[c];
      if (p != -1.f && better(p, c, best.v, best.i)) { best.v = p; best.i = c; }
    }
    best = warp_best(best);
    if (lane == 0) { red_v[warp] = best.v; red_i[warp] = best.i; }
    __syncthreads();
    if (tid == 0) {
      ArgBest t{red_v[0], red_i[0]};
      for (int w = 1; w < 8; ++w)
        if (better(red_v[w], red_i[w], t.v, t.i)) { t.v = red_v[w]; t.i = red_i[w]; }
      topk_val[(long)b * k + j] = t.v;
      topk_idx[(long)b * k + j] = t.i;
      if (j == 0) {
        pred_cell[b] = t.i;
        pred_lnglat[2 * (long)b + 0] = centroids[2 * (long)t.i + 0];
        pred_lnglat[2 * (long)b + 1] = centroids[2 * (long)t.i + 1];
      }
      sp[t.i] = -1.f;  // probabilities are >= 0, so -1 marks "taken"
    }
    __syncthreads();
  }
}


// ------------------------------------------------------------------------------------------------
// Classification loss of reference models/super_guessr.py:468-474 (nn.CrossEntropyLoss, mean reduction):
//   mode 0: integer class labels            loss_b = lse(x_b) - x_b[y_b]
//   mode 1: soft targets t [B, C] (f32)     loss_b = sum_c t_bc (lse(x_b) - x_bc)
//   mode 2: haversine-smoothed targets      t_bc = exp(-(d_bc - min_c d_bc) / smoothing), NaN/inf -> 0
//           with d = haversine_matrix(labels, centroids) in km, fp64 (preprocessing/geo_utils.py:58-74,
//           preprocessing/utils.py:7-19)
// One CTA per sample; per-sample losses in fp64, then a single-block mean.
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ double block_reduce(double v, double* red, bool is_max) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const double u = __shfl_xor_sync(0xffffffffu, v, o);
    v = is_max ? fmax(v, u) : v + u;
  }
  __syncthreads();
  if (lane == 0) red[warp] = v;
  __syncthreads();
  double t = red[0];
  for (int w = 1; w < (blockDim.x >> 5); ++w) t = is_max ? fmax(t, red[w]) : t + red[w];
  return t;
}

__device__ __forceinline__ double haversine_km(double lng0, double lat0, double lng1, double lat1) {
  const double kDeg = 3.14159265358979323846 / 180.0;
  const double x_lng = lng0 * kDeg, x_lat = lat0 * kDeg, y_lng = lng1 * kDeg, y_lat = lat1 * kDeg;
  const double s_lat = sin((x_lat - y_lat) / 2), s_lng = sin((x_lng - y_lng) / 2);
  const double a = s_lat * s_lat + (cos(x_lat) * cos(y_lat)) * (s_lng * s_lng);
  return (6378137.0 * (2 * asin(sqrt(a)))) / 1000;
}

__global__ void __launch_bounds__(256)
ce_loss_kernel(const float* __restrict__ logits, int C, int mode, const long long* __restrict__ labels_idx,
               const float* __restrict__ soft, const double* __restrict__ labels_lnglat,
               const double* __restrict__ centroids, double smoothing, double* __restrict__ per_sample,
               float* __restrict__ dlogits, double grad_scale) {
  __shared__ double red[8];
  const int b = blockIdx.x, tid = threadIdx.x;
  const float* x = logits + (long)b * C;
  double m = -INFINITY;
  for (int c = tid; c < C; c += 256) m = fmax(m, (double)x[c]);
  m = block_reduce(m, red, true);
  double s = 0;
  for (int c = tid; c < C; c += 256) s += exp((double)x[c] - m);
  s = block_reduce(s, red, false);
  const double lse = m + log(s);
  double loss = 0;
  // backward (dlogits != nullptr): d loss_b / d x_c = softmax_c * sum_c'(t_c') - t_c, times grad_scale
  float* g = dlogits ? dlogits + (long)b * C : nullptr;
  if (mode == 0) {
    // A label outside [0, C) never indexes memory: the sample's loss (and so the batch mean) becomes NaN and its gradient row
    // zero, which is loud instead of undefined.  torch's ignore_index (-100) is not implemented: the reference's labels on
    // this path are geocell indices produced by its own dataset code and are never negative.
    const long long y = labels_idx[b];
    const bool valid = y >= 0 && y < C;
    if (tid == 0) loss = valid ? lse - (double)x[y] : (double)NAN;
    if (g)
      for (int c = tid; c < C; c += 256)
        g[c] = valid ? (float)(grad_scale * (exp((double)x[c] - lse) - (c == y ? 1.0 : 0.0))) : 0.f;
  } else if (mode == 1) {
    double tsum = 0;
    for (int c = tid; c < C; c += 256) {
      const double t = (double)soft[(long)b * C + c];
      loss += t * (lse - (double)x[c]);
      tsum += t;
    }
    if (g) {
      tsum = block_reduce(tsum, red, false);
      for (int c = tid; c < C; c += 256)
        g[c] = (float)(grad_scale * (exp((double)x[c] - lse) * tsum - (double)soft[(long)b * C + c]));
    }
  } else {
    const double lng = labels_lnglat[2 * b], lat = labels_lnglat[2 * b + 1];
    double dmin = INFINITY;
    for (int c = tid; c < C; c += 256) dmin = fmin(dmin, haversine_km(lng, lat, centroids[2 * c], centroids[2 * c + 1]));
    dmin = -block_reduce(-dmin, red, true);
    for (int c = tid; c < C; c += 256) {
      double t = exp(-(haversine_km(lng, lat, centroids[2 * c], centroids[2 * c + 1]) - dmin) / smoothing);
      if (isnan(t) || isinf(t)) t = 0;
      loss += t * (lse - (double)x[c]);
      if (g) g[c] = (float)t;            // parked; turned into the gradient below once sum(t) is known
    }
    if (g) {
      double tsum = 0;
      for (int c = tid; c < C; c += 256) tsum += (double)g[c];   // same thread wrote these entries
      tsum = block_reduce(tsum, red, false);
      for (int c = tid; c < C; c += 256)
        g[c] = (float)(grad_scale * (exp((double)x[c] - lse) * tsum - (double)g[c]));
    }
  }
  loss = block_reduce(loss, red, false);
  if (tid == 0) per_sample[b] = loss;
}

__global__ void mean_f64_kernel(const double* __restrict__ v, int n, double* __restrict__ out) {
  __shared__ double red[8];
  double s = 0;
  for (int i = threadIdx.x; i < n; i += blockDim.x) s += v[i];
  s = block_reduce(s, red, false);
  if (threadIdx.x == 0) *out = s / n;
}

int check_launch(const char* what) {
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) { set_last_error("%s launch: %s", what, cudaGetErrorString(e)); return 1; }
  return 0;
}

}  // namespace

int view_mean_split(const float* emb, float* pooled, void* a3_f16, int B, int V, int D, cudaStream_t stream) {
  const long total = (long)B * D;
  int grid = (int)((total + 255) / 256);
  if (grid > 4096) grid = 4096;
  ProfScope prof("head_view_mean_split", stream);
  view_mean_split_kernel<<<grid, 256, 0, stream>>>(emb, pooled, reinterpret_cast<__half*>(a3_f16), B, V, D);
  return check_launch("view_mean_split");
}

int weight_split(const float* w, void* w3_f16, int C, int D, cudaStream_t stream) {
  const long total = (long)C * D;
  int grid = (int)((total + 255) / 256);
  if (grid > 4096) grid = 4096;
  weight_split_kernel<<<grid, 256, 0, stream>>>(w, reinterpret_cast<__half*>(w3_f16), C, D);
  return check_launch("weight_split");
}

int softmax_topk(const float* logits, float* probs, long long* pred_cell, double* pred_lnglat, float* topk_val,
                 long long* topk_idx, const double* centroids, int B, int C, int k, cudaStream_t stream) {
  if (k < 1 || k > C) { set_last_error("softmax_topk: k=%d out of range for C=%d", k, C); return 1; }
  if ((size_t)C * sizeof(float) > 200 * 1024) { set_last_error("softmax_topk: C=%d too large", C); return 1; }
  const size_t smem = (size_t)C * sizeof(float);
  if (smem > 48 * 1024) {
    cudaError_t e = cudaFuncSetAttribute(softmax_topk_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) { set_last_error("softmax_topk: smem attr: %s", cudaGetErrorString(e)); return 1; }
  }
  ProfScope prof("head_softmax_topk", stream);
  softmax_topk_kernel<<<B, 256, smem, stream>>>(logits, probs, pred_cell, pred_lnglat, topk_val, topk_idx, centroids,
                                                C, k);
  return check_launch("softmax_topk");
}

int ce_loss(const float* logits, int B, int C, int mode, const long long* labels_idx, const float* soft,
            const double* labels_lnglat, const double* centroids, double smoothing, double* per_sample,
            double* loss_out, float* dlogits, double grad_scale, cudaStream_t stream) {
  if (mode < 0 || mode > 2) { set_last_error("ce_loss: bad mode %d", mode); return 1; }
  if ((mode == 0 && !labels_idx) || (mode == 1 && !soft) || (mode == 2 && (!labels_lnglat || !centroids))) {
    set_last_error("ce_loss: missing labels for mode %d", mode);
    return 1;
  }
  ProfScope prof("head_ce_loss", stream);
  ce_loss_kernel<<<B, 256, 0, stream>>>(logits, C, mode, labels_idx, soft, labels_lnglat, centroids, smoothing,
                                        per_sample, dlogits, grad_scale / B);
  if (check_launch("ce_loss")) return 1;
  mean_f64_kernel<<<1, 256, 0, stream>>>(per_sample, B, loss_out);
  return check_launch("ce_loss_mean");
}

}  // namespace pg
