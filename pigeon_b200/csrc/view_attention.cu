// Hierarchical panorama head: the view self-attention of reference models/super_guessr.py:94-103,414-433 with
// models/layers/positional_encoder.py, forward and backward.
//
//   x   = dropout(emb + PE[n])                              emb f32 [N, 4, E]; PE row n (the sample's index in the batch)
//   q0  = x[:, 0] Wq^T + bq;  k, v = x Wk^T + bk, x Wv^T + bv   (nn.MultiheadAttention in_proj, error-compensated split GEMM)
//   P   = softmax(q0 k^T / sqrt(E / H)) per head over the 4 views;  o = dropout(P) v   (query row 0 only: only output[:, 0]
//         reaches the cell layer)
//   cls = o Wo^T + bo                                       (out_proj, split GEMM)
//
// Dropout draws are counter-based Philox4x32-10 keyed by (seed, offset) and indexed by the element's position in the whole
// batch (sample n0 + n), so a batch split into chunks draws the same masks as the whole batch, and the backward regenerates
// them instead of storing them.
#include <cuda_fp16.h>
#include <math.h>
#include <stdint.h>

#include "../../include/pigeon_b200.h"
#include "gemm.h"
#include "prof.h"
#include "tma_host.h"
#include "train.h"
#include "vit_handle.h"

namespace pg {
namespace {

constexpr int kViews = 4;

__device__ __forceinline__ uint4 philox4x32_10(uint4 c, uint2 k) {
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    const uint32_t hi0 = __umulhi(0xD2511F53u, c.x), lo0 = 0xD2511F53u * c.x;
    const uint32_t hi1 = __umulhi(0xCD9E8D57u, c.z), lo1 = 0xCD9E8D57u * c.z;
    c = make_uint4(hi1 ^ c.y ^ k.x, lo1, hi0 ^ c.w ^ k.y, lo0);
    k.x += 0x9E3779B9u;
    k.y += 0xBB67AE85u;
  }
  return c;
}

// Four uniform draws for group `g` of dropout stream `stream` (0: positional-encoding dropout, 1: attention dropout).
__device__ __forceinline__ uint4 draws(unsigned long long g, uint32_t stream, unsigned long long seed,
                                       unsigned long long offset) {
  return philox4x32_10(make_uint4((uint32_t)g, (uint32_t)(g >> 32) | (stream << 31), (uint32_t)offset,
                                  (uint32_t)(offset >> 32)),
                       make_uint2((uint32_t)seed, (uint32_t)(seed >> 32)));
}

// Keep with probability 1 - p (p = 0 keeps everything).
__device__ __forceinline__ bool keep(uint32_t r, float p) { return (float)(r >> 8) * (1.0f / 16777216.0f) >= p; }

__device__ __forceinline__ void split_store(__half* row, int E, int d, float x) {
  const __half hi = __float2half_rn(x);
  row[d] = hi;
  row[E + d] = __float2half_rn(x - __half2float(hi));
  row[2 * E + d] = hi;
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// x = dropout(emb + PE[n0 + n]) f32 [N*4, E] and its split x3 fp16 [N*4, 3E] = [hi | lo | hi]; 4 elements per thread.
__global__ void __launch_bounds__(256)
pe_dropout_split_kernel(const float* __restrict__ emb, const float* __restrict__ pe, int n0, int N, int E, float p,
                        float scale, unsigned long long seed, unsigned long long offset, float* __restrict__ x,
                        __half* __restrict__ x3, uint8_t* __restrict__ mask) {
  const long groups = (long)N * kViews * E / 4;
  const long g0 = (long)n0 * kViews * E / 4;
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < groups; i += (long)gridDim.x * blockDim.x) {
    const long e = 4 * i;
    const long row = e / E;
    const int d = (int)(e % E);
    const int n = (int)(row / kViews);
    const float4 a = *reinterpret_cast<const float4*>(emb + e);
    const float4 b = *reinterpret_cast<const float4*>(pe + (long)(n0 + n) * E + d);
    const uint4 r = p > 0.f ? draws(g0 + i, 0, seed, offset) : make_uint4(0xffffffffu, 0xffffffffu, 0xffffffffu, 0xffffffffu);
    const float s[4] = {a.x + b.x, a.y + b.y, a.z + b.z, a.w + b.w};
    const uint32_t rv[4] = {r.x, r.y, r.z, r.w};
    float y[4];
    __half* xrow = x3 + row * 3 * E;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const bool k = keep(rv[j], p);
      y[j] = k ? s[j] * scale : 0.f;
      split_store(xrow, E, d + j, y[j]);
      if (mask) mask[e + j] = k;
    }
    *reinterpret_cast<float4*>(x + e) = make_float4(y[0], y[1], y[2], y[3]);
  }
}

// One warp per (sample, head): scores of query row 0 against the 4 views, softmax, dropout, P.v.
//   q0 f32 [N, E], kv f32 [N*4, 2E] = [k | v]  ->  probs f32 [N, H, 4] (before dropout), o f32 [N, E], o3 fp16 [N, 3E].
__global__ void __launch_bounds__(256)
attn_core_kernel(const float* __restrict__ q0, const float* __restrict__ kv, int n0, int N, int E, int H, float qk_scale,
                 float p, float scale, unsigned long long seed, unsigned long long offset, float* __restrict__ probs,
                 float* __restrict__ o, __half* __restrict__ o3, uint8_t* __restrict__ mask) {
  const int lane = threadIdx.x & 31;
  const int hd = E / H;
  const long warps = (long)N * H;
  for (long w = ((long)blockIdx.x * blockDim.x + threadIdx.x) >> 5; w < warps; w += ((long)gridDim.x * blockDim.x) >> 5) {
    const int n = (int)(w / H), h = (int)(w % H);
    const float* q = q0 + (long)n * E + h * hd;
    const float* kvn = kv + (long)n * kViews * 2 * E + h * hd;
    float s[kViews];
#pragma unroll
    for (int j = 0; j < kViews; ++j) {
      float acc = 0.f;
      for (int d = lane; d < hd; d += 32) acc = fmaf(q[d], kvn[(long)j * 2 * E + d], acc);
      s[j] = warp_sum(acc) * qk_scale;
    }
    const float m = fmaxf(fmaxf(s[0], s[1]), fmaxf(s[2], s[3]));
    float sum = 0.f;
#pragma unroll
    for (int j = 0; j < kViews; ++j) { s[j] = expf(s[j] - m); sum += s[j]; }
    const uint4 r = p > 0.f ? draws((unsigned long long)(n0 + n) * H + h, 1, seed, offset)
                            : make_uint4(0xffffffffu, 0xffffffffu, 0xffffffffu, 0xffffffffu);
    const uint32_t rv[kViews] = {r.x, r.y, r.z, r.w};
    float pd[kViews];
#pragma unroll
    for (int j = 0; j < kViews; ++j) {
      const float pj = s[j] / sum;
      const bool k = keep(rv[j], p);
      pd[j] = k ? pj * scale : 0.f;
      if (lane == 0) {
        probs[w * kViews + j] = pj;
        if (mask) mask[w * kViews + j] = k;
      }
    }
    for (int d = lane; d < hd; d += 32) {
      float acc = 0.f;
#pragma unroll
      for (int j = 0; j < kViews; ++j) acc = fmaf(pd[j], kvn[(long)j * 2 * E + E + d], acc);
      o[(long)n * E + h * hd + d] = acc;
      split_store(o3 + (long)n * 3 * E, E, h * hd + d, acc);
    }
  }
}

// Backward of attn_core_kernel, one warp per (sample, head), masks regenerated:
//   do f32 [N, E]  ->  dqkv f32 [N*4, 3E]: row (n, view j) = [dq (view 0 only, else 0) | dk_j | dv_j].
__global__ void __launch_bounds__(256)
attn_core_backward_kernel(const float* __restrict__ dout, const float* __restrict__ q0, const float* __restrict__ kv,
                          const float* __restrict__ probs, int n0, int N, int E, int H, float qk_scale, float p, float scale,
                          unsigned long long seed, unsigned long long offset, float* __restrict__ dqkv) {
  const int lane = threadIdx.x & 31;
  const int hd = E / H;
  const long warps = (long)N * H;
  for (long w = ((long)blockIdx.x * blockDim.x + threadIdx.x) >> 5; w < warps; w += ((long)gridDim.x * blockDim.x) >> 5) {
    const int n = (int)(w / H), h = (int)(w % H);
    const float* q = q0 + (long)n * E + h * hd;
    const float* kvn = kv + (long)n * kViews * 2 * E + h * hd;
    const float* dn = dout + (long)n * E + h * hd;
    float* g = dqkv + (long)n * kViews * 3 * E + h * hd;
    const uint4 r = p > 0.f ? draws((unsigned long long)(n0 + n) * H + h, 1, seed, offset)
                            : make_uint4(0xffffffffu, 0xffffffffu, 0xffffffffu, 0xffffffffu);
    const uint32_t rv[kViews] = {r.x, r.y, r.z, r.w};
    float P[kViews], pd[kViews], dp[kViews];
    float t = 0.f;
#pragma unroll
    for (int j = 0; j < kViews; ++j) {
      float acc = 0.f;
      for (int d = lane; d < hd; d += 32) acc = fmaf(dn[d], kvn[(long)j * 2 * E + E + d], acc);
      const float dpd = warp_sum(acc);
      const bool k = keep(rv[j], p);
      P[j] = probs[w * kViews + j];
      pd[j] = k ? P[j] * scale : 0.f;
      dp[j] = k ? dpd * scale : 0.f;
      t = fmaf(P[j], dp[j], t);
    }
    float ds[kViews];
#pragma unroll
    for (int j = 0; j < kViews; ++j) ds[j] = P[j] * (dp[j] - t) * qk_scale;
    for (int d = lane; d < hd; d += 32) {
      float dq = 0.f;
      const float qd = q[d], dod = dn[d];
#pragma unroll
      for (int j = 0; j < kViews; ++j) {
        float* gj = g + (long)j * 3 * E;
        dq = fmaf(ds[j], kvn[(long)j * 2 * E + d], dq);
        gj[E + d] = ds[j] * qd;
        gj[2 * E + d] = pd[j] * dod;
        if (j > 0) gj[d] = 0.f;
      }
      g[d] = dq;
    }
  }
}

// d emb = d x * keep / (1 - p), in place (the positional encoding is a constant: its gradient is the identity).
__global__ void __launch_bounds__(256)
pe_dropout_backward_kernel(float* __restrict__ dx, int n0, int N, int E, float p, float scale, unsigned long long seed,
                           unsigned long long offset) {
  const long groups = (long)N * kViews * E / 4;
  const long g0 = (long)n0 * kViews * E / 4;
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < groups; i += (long)gridDim.x * blockDim.x) {
    const uint4 r = draws(g0 + i, 0, seed, offset);
    float4 v = *reinterpret_cast<float4*>(dx + 4 * i);
    v.x = keep(r.x, p) ? v.x * scale : 0.f;
    v.y = keep(r.y, p) ? v.y * scale : 0.f;
    v.z = keep(r.z, p) ? v.z * scale : 0.f;
    v.w = keep(r.w, p) ? v.w * scale : 0.f;
    *reinterpret_cast<float4*>(dx + 4 * i) = v;
  }
}

// out f32 [M, N] (row pitch ldo) = a [M, 3E] . w [N, 3E]^T + bias, both operands in the hi / lo split layout of
// pg_head_pack_weight, as K slices of at most kSliceK: the first writes acc + bias, the rest add through the fp32 residual
// epilogue.  The tensor cores' fp32 accumulation truncates, so one long chain drifts toward zero (about 5e-6 relative at
// K = 3072, which the cell layer's logits then carry); slices of 512 summed with rounded fp32 adds stay near 5e-7.
constexpr int kSliceK = 512;

int split_gemm(const __half* a, int lda, const __half* w, int M, int N, int E, float* out, int ldo, const float* bias, int sms,
               cudaStream_t stream) {
  const int K = 3 * E;
  for (int k0 = 0; k0 < K; k0 += kSliceK) {
    GemmProblem g{};
    g.M = M; g.N = N; g.K = K - k0 < kSliceK ? K - k0 : kSliceK;
    g.a = a + k0; g.lda = lda; g.w = w + k0; g.ldw = K;
    g.out = out; g.ldo = ldo;
    g.bias = k0 == 0 ? bias : nullptr;
    g.epi = k0 == 0 ? EPI_F32_BIAS : EPI_F32_BIAS_RESID;
    if (gemm_f16(g, sms, stream)) return 1;
  }
  return 0;
}

int check_launch(const char* what) {
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) { set_last_error("%s launch: %s", what, cudaGetErrorString(e)); return 1; }
  return 0;
}

int grid_for(long items, int per_block, int sms, int blocks_per_sm) {
  const long g = (items + per_block - 1) / per_block;
  const long cap = (long)sms * blocks_per_sm;
  return (int)(g < cap ? (g > 0 ? g : 1) : cap);
}

int check_shape(const char* what, int N, int E, int heads, float p_x, float p_attn) {
  if (N < 0 || E <= 0 || E % 16 || heads <= 0 || E % heads) {
    set_last_error("%s: bad shape N=%d E=%d heads=%d (E %% 16 == 0 and E %% heads == 0)", what, N, E, heads);
    return 1;
  }
  if (!(p_x >= 0.f && p_x < 1.f && p_attn >= 0.f && p_attn < 1.f)) {
    set_last_error("%s: dropout probabilities %g, %g not in [0, 1)", what, p_x, p_attn);
    return 1;
  }
  return 0;
}

// Saved activations (f32): x [N*4, E] | q0 [N, E] | kv [N*4, 2E] | o [N, E] | probs [N, H, 4]
struct Saved {
  float *x, *q0, *kv, *o, *probs;
  Saved(float* s, long N, long E) : x(s), q0(s + 4 * N * E), kv(s + 5 * N * E), o(s + 13 * N * E), probs(s + 14 * N * E) {}
};

}  // namespace
}  // namespace pg

using namespace pg;

extern "C" {

size_t pg_view_attn_saved_floats(int32_t N, int32_t E, int32_t heads) {
  if (N <= 0 || E <= 0 || heads <= 0) return 0;
  return (size_t)14 * N * E + (size_t)4 * N * heads;
}

size_t pg_view_attn_workspace_bytes(int32_t N, int32_t E) {
  if (N <= 0 || E <= 0) return 0;
  const size_t fwd = (size_t)15 * N * E * sizeof(__half);            // x3 [N*4, 3E] | o3 [N, 3E]
  const size_t bwd = (size_t)13 * N * E * sizeof(float);             // do [N, E] | dqkv [N*4, 3E]
  return align_up(fwd > bwd ? fwd : bwd, 1024);
}

int pg_view_attn_forward(const float* emb, int32_t N, int32_t E, int32_t heads, const float* pe, int32_t pe_rows,
                         int32_t n0, const void* w_in3, const float* b_in, const void* w_out3, const float* b_out,
                         float p_x, float p_attn, uint64_t seed, uint64_t offset, void* workspace, size_t workspace_bytes,
                         float* saved, uint8_t* mask_x, uint8_t* mask_p, float* cls, void* stream_) {
  if (check_shape("pg_view_attn_forward", N, E, heads, p_x, p_attn)) return 1;
  if (!emb || !pe || !w_in3 || !b_in || !w_out3 || !b_out || !workspace || !saved || !cls) {
    set_last_error("pg_view_attn_forward: null argument");
    return 1;
  }
  if (n0 < 0 || (long)n0 + N > pe_rows) {
    set_last_error("pg_view_attn_forward: samples %d..%d need positional-encoding rows the table of %d rows does not have",
                   n0, n0 + N - 1, pe_rows);
    return 1;
  }
  if (N == 0) return 0;
  if (workspace_bytes < pg_view_attn_workspace_bytes(N, E)) { set_last_error("pg_view_attn_forward: workspace too small"); return 1; }
  if ((reinterpret_cast<uintptr_t>(emb) | reinterpret_cast<uintptr_t>(pe) | reinterpret_cast<uintptr_t>(saved)) & 15) {
    set_last_error("pg_view_attn_forward: emb, pe and saved must be 16-byte aligned");
    return 1;
  }
  const int sms = sm_count();
  if (sms < 0) return 1;
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  Saved s(saved, N, E);
  __half* x3 = reinterpret_cast<__half*>(workspace);
  __half* o3 = x3 + (size_t)12 * N * E;
  {
    ProfScope prof("view_attn_pe_dropout", stream);
    pe_dropout_split_kernel<<<grid_for((long)N * E, 256, sms, 8), 256, 0, stream>>>(
        emb, pe, n0, N, E, p_x, 1.f / (1.f - p_x), seed, offset, s.x, x3, mask_x);
    if (check_launch("view_attn_pe_dropout")) return 1;
  }
  // k, v of all four views: [N*4, 3E] x [2E, 3E]^T; q of view 0 only: every fourth row of x3 (lda = 4 * 3E)
  const __half* w_in = reinterpret_cast<const __half*>(w_in3);
  if (split_gemm(x3, 3 * E, w_in + (size_t)E * 3 * E, 4 * N, 2 * E, E, s.kv, 2 * E, b_in + E, sms, stream)) return 1;
  if (split_gemm(x3, 4 * 3 * E, w_in, N, E, E, s.q0, E, b_in, sms, stream)) return 1;
  {
    ProfScope prof("view_attn_core", stream);
    attn_core_kernel<<<grid_for((long)N * heads, 8, sms, 4), 256, 0, stream>>>(
        s.q0, s.kv, n0, N, E, heads, 1.f / sqrtf((float)(E / heads)), p_attn, 1.f / (1.f - p_attn), seed, offset, s.probs,
        s.o, o3, mask_p);
    if (check_launch("view_attn_core")) return 1;
  }
  return split_gemm(o3, 3 * E, reinterpret_cast<const __half*>(w_out3), N, E, E, cls, E, b_out, sms, stream);
}

int pg_view_attn_backward(const float* dcls, int32_t N, int32_t E, int32_t heads, int32_t n0, const float* w_in,
                          const float* w_out, const float* saved, float p_x, float p_attn, uint64_t seed, uint64_t offset,
                          int32_t accumulate, float* dw_in, float* db_in, float* dw_out, float* db_out, float* demb,
                          void* workspace, size_t workspace_bytes, void* stream_) {
  if (check_shape("pg_view_attn_backward", N, E, heads, p_x, p_attn)) return 1;
  if (!dcls || !w_in || !w_out || !saved || !demb || !workspace || n0 < 0) {
    set_last_error("pg_view_attn_backward: null argument");
    return 1;
  }
  if (N == 0) return 0;
  if (workspace_bytes < pg_view_attn_workspace_bytes(N, E)) { set_last_error("pg_view_attn_backward: workspace too small"); return 1; }
  if ((reinterpret_cast<uintptr_t>(saved) | reinterpret_cast<uintptr_t>(demb)) & 15) {
    set_last_error("pg_view_attn_backward: saved and demb must be 16-byte aligned");
    return 1;
  }
  const int sms = sm_count();
  if (sms < 0) return 1;
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  Saved s(const_cast<float*>(saved), N, E);
  float* dout = reinterpret_cast<float*>(workspace);
  float* dqkv = dout + (size_t)N * E;
  const float beta = accumulate ? 1.f : 0.f;
  // out_proj: dWo (+)= dcls^T o;  dbo (+)= column sums of dcls;  do = dcls Wo
  if (dw_out && sgemm_f32(true, dcls, s.o, dw_out, E, E, N, beta, stream)) return 1;
  if (db_out && column_sum_f32(dcls, db_out, N, E, beta, stream)) return 1;
  if (sgemm_f32(false, dcls, w_out, dout, N, E, E, 0.f, stream)) return 1;
  {
    ProfScope prof("view_attn_core_backward", stream);
    attn_core_backward_kernel<<<grid_for((long)N * heads, 8, sms, 4), 256, 0, stream>>>(
        dout, s.q0, s.kv, s.probs, n0, N, E, heads, 1.f / sqrtf((float)(E / heads)), p_attn, 1.f / (1.f - p_attn), seed,
        offset, dqkv);
    if (check_launch("view_attn_core_backward")) return 1;
  }
  // in_proj: dWin (+)= dqkv^T x;  dbin (+)= column sums of dqkv;  dx = dqkv Win
  if (dw_in && sgemm_f32(true, dqkv, s.x, dw_in, 3 * E, E, 4 * N, beta, stream)) return 1;
  if (db_in && column_sum_f32(dqkv, db_in, 4 * N, 3 * E, beta, stream)) return 1;
  if (sgemm_f32(false, dqkv, w_in, demb, 4 * N, E, 3 * E, 0.f, stream)) return 1;
  if (p_x > 0.f) {
    ProfScope prof("view_attn_pe_dropout_backward", stream);
    pe_dropout_backward_kernel<<<grid_for((long)N * E, 256, sms, 8), 256, 0, stream>>>(demb, n0, N, E, p_x,
                                                                                         1.f / (1.f - p_x), seed, offset);
    if (check_launch("view_attn_pe_dropout_backward")) return 1;
  }
  return 0;
}

}  // extern "C"
