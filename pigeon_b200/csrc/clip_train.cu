// Kernels of the CLIPModel contrastive training step that are specific to it (HF CLIPModel, transformers 4.23.1
// modeling_clip.py, as reference training/train_modes.py:30-64 trains it with `return_loss=True`):
//   clip_loss_grad            clip_loss(logits_per_text) and its gradient through the L2 normalisation and logit_scale;
//   text_pool_ln_backward     final_layer_norm backward on the pooled (argmax-id) row of each caption only;
//   token_embedding_grad      d token_embedding.weight as a deterministic per-id sum of the embedding-output gradient.
// The encoder layers' backward is the vision tower's (vit_train_capi.cu).
#include "clip.h"

#include <math.h>
#include <stdint.h>

#include "prof.h"
#include "text_pool.cuh"
#include "tma_host.h"
#include "vit_handle.h"

namespace pg {

namespace {

constexpr int kThreads = 256;

int check_launch(const char* what) {
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) { set_last_error("%s launch: %s", what, cudaGetErrorString(e)); return 1; }
  return 0;
}

// Fixed-order block sum (deterministic); every thread gets the result.  blockDim.x == kThreads.
__device__ double block_sum(double v, double* red) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  __syncthreads();
  if (lane == 0) red[warp] = v;
  __syncthreads();
  double t = 0.0;
  for (int w = 0; w < kThreads / 32; ++w) t += red[w];
  return t;
}

struct LossWs {
  float* ih;      // [n, P] image_embeds / |image_embeds|
  float* th;      // [n, P] text_embeds / |text_embeds|
  float* inv;     // [2n]   1 / |img_i|, then 1 / |txt_t|
  double* L;      // [n, n] logits_per_text (row = caption, column = image)
  double* dL;     // [n, n] d loss / d logits_per_text, times grad_scale
};

LossWs carve_loss(int n, int P, void* ws, size_t* total) {
  Carver c(ws);
  LossWs w;
  w.ih = reinterpret_cast<float*>(c.take((size_t)n * P * 4));
  w.th = reinterpret_cast<float*>(c.take((size_t)n * P * 4));
  w.inv = reinterpret_cast<float*>(c.take((size_t)2 * n * 4));
  w.L = reinterpret_cast<double*>(c.take((size_t)n * n * 8));
  w.dL = reinterpret_cast<double*>(c.take((size_t)n * n * 8));
  *total = c.off;
  return w;
}

// Block r < n: image row r; block n + r: caption row r.  hat = x / |x| (HF `embeds / embeds.norm(p=2, dim=-1)`).
__global__ void __launch_bounds__(kThreads)
clip_normalise_kernel(const float* __restrict__ img, const float* __restrict__ txt, int n, int P, LossWs w) {
  __shared__ double red[kThreads / 32];
  const bool is_t = blockIdx.x >= (unsigned)n;
  const int row = is_t ? blockIdx.x - n : blockIdx.x;
  const float* x = (is_t ? txt : img) + (long)row * P;
  double ss = 0.0;
  for (int p = threadIdx.x; p < P; p += kThreads) ss += (double)x[p] * x[p];
  ss = block_sum(ss, red);
  const float iv = (float)(1.0 / sqrt(ss));
  float* y = (is_t ? w.th : w.ih) + (long)row * P;
  for (int p = threadIdx.x; p < P; p += kThreads) y[p] = x[p] * iv;
  if (threadIdx.x == 0) w.inv[blockIdx.x] = iv;
}

// One warp per logit: L[t, i] = exp(logit_scale) th_t . ih_i (fp64 sum); fp32 copies into lpt [t, i] / lpi [i, t].
__global__ void __launch_bounds__(kThreads)
clip_train_logits_kernel(int n, int P, const float* __restrict__ logit_scale, LossWs w, float* __restrict__ lpi,
                         float* __restrict__ lpt) {
  const int lane = threadIdx.x & 31;
  const long e = ((long)blockIdx.x * kThreads + threadIdx.x) >> 5;
  if (e >= (long)n * n) return;
  const int t = (int)(e / n), i = (int)(e % n);
  const float* a = w.th + (long)t * P;
  const float* b = w.ih + (long)i * P;
  double s = 0.0;
  for (int p = lane; p < P; p += 32) s += (double)a[p] * b[p];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if (lane == 0) {
    const double v = s * exp((double)*logit_scale);
    w.L[e] = v;
    if (lpt) lpt[e] = (float)v;
    if (lpi) lpi[(long)i * n + t] = (float)v;
  }
}

// One CTA (deterministic).  Row / column log-sum-exp of L in fp64, the loss
//   (sum_t lse_row(t) - L[t, t] + sum_i lse_col(i) - L[i, i]) / 2n,
// dL = grad_scale (softmax_rows(L) - I + softmax_cols(L) - I) / 2n and d logit_scale = sum dL o L.
__global__ void __launch_bounds__(1024)
clip_loss_grad_kernel(int n, double grad_scale, LossWs w, double* __restrict__ lse, float* __restrict__ loss,
                      float* __restrict__ d_logit_scale) {
  __shared__ double red[32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  double acc = 0.0;
  for (int r = warp; r < 2 * n; r += 32) {
    const bool col = r >= n;
    const int k = col ? r - n : r;
    const double* x = col ? w.L + k : w.L + (long)k * n;
    const long stride = col ? n : 1;
    double m = -INFINITY;
    for (int t = lane; t < n; t += 32) m = fmax(m, x[t * stride]);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) m = fmax(m, __shfl_xor_sync(0xffffffffu, m, o));
    double s = 0.0;
    for (int t = lane; t < n; t += 32) s += exp(x[t * stride] - m);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (lane == 0) {
      lse[r] = m + log(s);
      acc += m + log(s) - w.L[(long)k * n + k];
    }
  }
  if (lane == 0) red[warp] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    double t = 0.0;
    for (int i = 0; i < 32; ++i) t += red[i];
    *loss = (float)(t / (2.0 * n));
  }
  __syncthreads();
  const double c = grad_scale / (2.0 * n);
  double ds = 0.0;
  for (long e = threadIdx.x; e < (long)n * n; e += blockDim.x) {
    const int t = (int)(e / n), i = (int)(e % n);
    const double v = w.L[e];
    const double d = (exp(v - lse[t]) + exp(v - lse[n + i]) - (t == i ? 2.0 : 0.0)) * c;
    w.dL[e] = d;
    ds += d * v;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) ds += __shfl_xor_sync(0xffffffffu, ds, o);
  __syncthreads();
  if (lane == 0) red[warp] = ds;
  __syncthreads();
  if (threadIdx.x == 0) {
    double t = 0.0;
    for (int i = 0; i < 32; ++i) t += red[i];
    *d_logit_scale = (float)t;
  }
}

// Block r < n: image row r; block n + r: caption row r.  dhat = s dL^T th (images) or s dL ih (captions), then the backward
// of the L2 normalisation, dx = (dhat - hat (hat . dhat)) / |x|.  dhat is kept in shared memory (P doubles).
__global__ void __launch_bounds__(kThreads)
clip_embeds_grad_kernel(int n, int P, const float* __restrict__ logit_scale, LossWs w, float* __restrict__ d_img,
                        float* __restrict__ d_txt) {
  extern __shared__ double dh[];
  __shared__ double red[kThreads / 32];
  const bool is_t = blockIdx.x >= (unsigned)n;
  const int row = is_t ? blockIdx.x - n : blockIdx.x;
  const double s = exp((double)*logit_scale);
  const float* other = is_t ? w.ih : w.th;
  const float* hat = (is_t ? w.th : w.ih) + (long)row * P;
  double dot = 0.0;
  for (int p = threadIdx.x; p < P; p += kThreads) {
    double a = 0.0;
    for (int k = 0; k < n; ++k) {
      const double d = is_t ? w.dL[(long)row * n + k] : w.dL[(long)k * n + row];
      a += d * other[(long)k * P + p];
    }
    a *= s;
    dh[p] = a;
    dot += a * hat[p];
  }
  dot = block_sum(dot, red);
  const double iv = w.inv[blockIdx.x];
  float* out = (is_t ? d_txt : d_img) + (long)row * P;
  for (int p = threadIdx.x; p < P; p += kThreads) out[p] = (float)((dh[p] - hat[p] * dot) * iv);
}

// One warp per caption b: LayerNorm backward of x row b * S + argmax(ids[b]) with dy = d_pooled[b] (the formula of
// train_vit.cu's ln_backward_kernel); dx goes to that row of g (the caller zeroes g), the per-caption dgamma / dbeta terms
// to part [n, 2 hidden] for an ordered column sum.
template <int NV4>
__global__ void __launch_bounds__(kThreads)
text_pool_ln_backward_kernel(const float* __restrict__ x, const float* __restrict__ dy, const float* __restrict__ gamma,
                             const long long* __restrict__ ids, int n, int S, float eps, float* __restrict__ g,
                             float* __restrict__ part) {
  constexpr int hidden = NV4 * 128;
  const int lane = threadIdx.x & 31;
  const int b = (blockIdx.x * kThreads + threadIdx.x) >> 5;
  if (b >= n) return;
  const long row = (long)b * S + first_argmax_warp(ids + (long)b * S, S, lane);
  const float4* xr = reinterpret_cast<const float4*>(x + row * hidden);
  const float4* dr = reinterpret_cast<const float4*>(dy + (long)b * hidden);
  float4 xv[NV4], dv[NV4];
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < NV4; ++i) {
    xv[i] = xr[lane + 32 * i];
    dv[i] = dr[lane + 32 * i];
    s += (xv[i].x + xv[i].y) + (xv[i].z + xv[i].w);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  const float mean = s / hidden;
  float ss = 0.f;
#pragma unroll
  for (int i = 0; i < NV4; ++i) {
    xv[i].x -= mean; xv[i].y -= mean; xv[i].z -= mean; xv[i].w -= mean;
    ss += (xv[i].x * xv[i].x + xv[i].y * xv[i].y) + (xv[i].z * xv[i].z + xv[i].w * xv[i].w);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
  const float rstd = rsqrtf(ss / hidden + eps);
  float4* pg_row = reinterpret_cast<float4*>(part + (long)b * 2 * hidden);
  float4* pb_row = pg_row + hidden / 4;
  float s1 = 0.f, s2 = 0.f;
#pragma unroll
  for (int i = 0; i < NV4; ++i) {
    const float4 gm = __ldg(reinterpret_cast<const float4*>(gamma) + lane + 32 * i);
    xv[i].x *= rstd; xv[i].y *= rstd; xv[i].z *= rstd; xv[i].w *= rstd;          // xhat
    pg_row[lane + 32 * i] = make_float4(dv[i].x * xv[i].x, dv[i].y * xv[i].y, dv[i].z * xv[i].z, dv[i].w * xv[i].w);
    pb_row[lane + 32 * i] = dv[i];
    dv[i].x *= gm.x; dv[i].y *= gm.y; dv[i].z *= gm.z; dv[i].w *= gm.w;           // gamma * dy
    s1 += (dv[i].x + dv[i].y) + (dv[i].z + dv[i].w);
    s2 += (dv[i].x * xv[i].x + dv[i].y * xv[i].y) + (dv[i].z * xv[i].z + dv[i].w * xv[i].w);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    s1 += __shfl_xor_sync(0xffffffffu, s1, o);
    s2 += __shfl_xor_sync(0xffffffffu, s2, o);
  }
  s1 /= hidden;
  s2 /= hidden;
  float4* gr = reinterpret_cast<float4*>(g + row * hidden);
#pragma unroll
  for (int i = 0; i < NV4; ++i)
    gr[lane + 32 * i] = make_float4(rstd * (dv[i].x - s1 - xv[i].x * s2), rstd * (dv[i].y - s1 - xv[i].y * s2),
                                    rstd * (dv[i].z - s1 - xv[i].z * s2), rstd * (dv[i].w - s1 - xv[i].w * s2));
}

// out [cols] += sum over rows of part [rows, cols], rows in ascending order (deterministic).
__global__ void __launch_bounds__(kThreads)
ordered_column_sum_kernel(const float* __restrict__ part, int rows, int cols, float* __restrict__ out0,
                          float* __restrict__ out1, int split) {
  const int c = blockIdx.x * kThreads + threadIdx.x;
  if (c >= cols) return;
  float s = 0.f;
  for (int r = 0; r < rows; ++r) s += part[(long)r * cols + c];
  if (c < split) out0[c] += s;
  else out1[c - split] += s;
}

// Block per row r of dx [rows, hidden].  The block of the FIRST row holding an id sums the rows of that id in ascending
// order and adds the sum to dtok[id]; every other block returns.  No atomics: the result does not depend on scheduling.
// Ids outside [0, vocab) are never used as an index (the forward made their rows NaN).
__global__ void __launch_bounds__(kThreads)
token_embedding_grad_kernel(const long long* __restrict__ ids, const float* __restrict__ dx, long rows, int hidden,
                            int vocab, float* __restrict__ dtok) {
  const long r = blockIdx.x;
  const long long id = ids[r];
  if (id < 0 || id >= vocab) return;
  int dup = 0;
  for (long q = threadIdx.x; q < r; q += kThreads) dup |= (ids[q] == id);
  if (__syncthreads_or(dup)) return;
  for (int c = threadIdx.x; c < hidden; c += kThreads) {
    float s = 0.f;
    for (long q = r; q < rows; ++q)
      if (__ldg(ids + q) == id) s += dx[q * hidden + c];
    dtok[id * hidden + c] += s;
  }
}

}  // namespace

size_t clip_loss_grad_workspace_bytes(int n, int P) {
  size_t total = 0;
  carve_loss(n, P, nullptr, &total);
  return total + align_up((size_t)2 * n * 8, 1024);
}

int clip_loss_grad(const float* img, const float* txt, int n, int P, const float* logit_scale, double grad_scale,
                   void* workspace, size_t workspace_bytes, float* loss, float* d_img, float* d_txt, float* d_logit_scale,
                   float* lpi, float* lpt, cudaStream_t stream) {
  if (n <= 0) return 0;
  if (P <= 0 || P > 4096) { set_last_error("clip_loss_grad: projection dim %d not in [1, 4096]", P); return 1; }
  if (n > 16384) { set_last_error("clip_loss_grad: n %d > 16384", n); return 1; }
  if (workspace_bytes < clip_loss_grad_workspace_bytes(n, P)) { set_last_error("clip_loss_grad: workspace too small"); return 1; }
  size_t off = 0;
  const LossWs w = carve_loss(n, P, workspace, &off);
  double* lse = reinterpret_cast<double*>(reinterpret_cast<uint8_t*>(workspace) + off);
  ProfScope prof("clip_loss_grad", stream);
  clip_normalise_kernel<<<2 * n, kThreads, 0, stream>>>(img, txt, n, P, w);
  if (check_launch("clip_normalise")) return 1;
  const long warps = (long)n * n;
  clip_train_logits_kernel<<<(unsigned)((warps * 32 + kThreads - 1) / kThreads), kThreads, 0, stream>>>(n, P, logit_scale, w,
                                                                                                         lpi, lpt);
  if (check_launch("clip_train_logits")) return 1;
  clip_loss_grad_kernel<<<1, 1024, 0, stream>>>(n, grad_scale, w, lse, loss, d_logit_scale);
  if (check_launch("clip_loss_grad")) return 1;
  const size_t smem = (size_t)P * sizeof(double);
  clip_embeds_grad_kernel<<<2 * n, kThreads, smem, stream>>>(n, P, logit_scale, w, d_img, d_txt);
  return check_launch("clip_embeds_grad");
}

#define PG_DISPATCH_NV4(hidden, CALL)                                                        \
  switch ((hidden) / 128) {                                                                  \
    case 1: { constexpr int NV4 = 1; CALL; break; }                                          \
    case 2: { constexpr int NV4 = 2; CALL; break; }                                          \
    case 4: { constexpr int NV4 = 4; CALL; break; }                                          \
    case 6: { constexpr int NV4 = 6; CALL; break; }                                          \
    case 8: { constexpr int NV4 = 8; CALL; break; }                                          \
    default: set_last_error("hidden size %d unsupported (need 128*{1,2,4,6,8})", (hidden)); return 1; \
  }

int text_pool_ln_backward(const float* x, const float* d_pooled, const float* gamma, const long long* ids, int n, int S,
                          int hidden, float eps, float* g, float* part, float* dgamma, float* dbeta, cudaStream_t stream) {
  if (n <= 0) return 0;
  if (hidden % 128) { set_last_error("text_pool_ln_backward: hidden %d not a multiple of 128", hidden); return 1; }
  ProfScope prof("text_pool_ln_backward", stream);
  const int blocks = (n + kThreads / 32 - 1) / (kThreads / 32);
  PG_DISPATCH_NV4(hidden, (text_pool_ln_backward_kernel<NV4><<<blocks, kThreads, 0, stream>>>(x, d_pooled, gamma, ids, n, S,
                                                                                              eps, g, part)));
  if (check_launch("text_pool_ln_backward")) return 1;
  ordered_column_sum_kernel<<<(2 * hidden + kThreads - 1) / kThreads, kThreads, 0, stream>>>(part, n, 2 * hidden, dgamma,
                                                                                           dbeta, hidden);
  return check_launch("text_pool_ln_param_sum");
}

int token_embedding_grad(const long long* ids, const float* dx, long rows, int hidden, int vocab, float* dtok,
                         cudaStream_t stream) {
  if (rows <= 0) return 0;
  if (rows > 0x7fffffffL) { set_last_error("token_embedding_grad: %ld rows exceed the grid", rows); return 1; }
  ProfScope prof("token_embedding_grad", stream);
  token_embedding_grad_kernel<<<(unsigned)rows, kThreads, 0, stream>>>(ids, dx, rows, hidden, vocab, dtok);
  return check_launch("token_embedding_grad");
}

}  // namespace pg
