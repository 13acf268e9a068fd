// Memory-bound kernels of the vision-tower backward pass ("next" row N1: the fine-tune step of reference
// training/train_eval_loop.py:215-221 through HF CLIPVisionTransformer, i.e. what loss.backward() runs between the
// GEMMs): dtype casts and transposes feeding the bf16 wgmma GEMMs, quick-GELU and LayerNorm backward, the softmax
// correction term of attention backward, token-mean / embedding backward and bias gradients.  All HBM-bound:
// vectorised, coalesced, grid-stride over the SMs.
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "prof.h"
#include "tma_host.h"
#include "train_vit.h"

namespace pg {
namespace {

int check_launch(const char* what) {
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) { set_last_error("%s launch: %s", what, cudaGetErrorString(e)); return 1; }
  return 0;
}

inline int grid_1d(long work_items, int per_block, int cap = 132 * 16) {
  long b = (work_items + per_block - 1) / per_block;
  if (b < 1) b = 1;
  return (int)(b > cap ? cap : b);
}

template <typename T> __device__ __forceinline__ float to_f32(T v);
template <> __device__ __forceinline__ float to_f32<float>(float v) { return v; }
template <> __device__ __forceinline__ float to_f32<__half>(__half v) { return __half2float(v); }
template <> __device__ __forceinline__ float to_f32<__nv_bfloat16>(__nv_bfloat16 v) { return __bfloat162float(v); }

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// ------------------------------------------------------------------------------------------------ casts
template <typename T> struct Vec8;   // 8 source elements in one or two 16-byte loads
template <> struct Vec8<float> {
  static __device__ __forceinline__ void load(const float* p, float (&v)[8]) {
    const float4 a = reinterpret_cast<const float4*>(p)[0], b = reinterpret_cast<const float4*>(p)[1];
    v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
  }
};
template <> struct Vec8<__half> {
  static __device__ __forceinline__ void load(const __half* p, float (&v)[8]) {
    const uint4 a = *reinterpret_cast<const uint4*>(p);
    const uint32_t w[4] = {a.x, a.y, a.z, a.w};
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const float2 f = __half22float2(*reinterpret_cast<const __half2*>(&w[k]));
      v[2 * k] = f.x; v[2 * k + 1] = f.y;
    }
  }
};

// 8 elements per thread and iteration: 16/32-byte loads, one 16-byte store (src and out 16-byte aligned, checked by the host)
template <typename T>
__global__ void __launch_bounds__(256) cast_kernel(const T* __restrict__ src, __nv_bfloat16* __restrict__ out, long n) {
  const long stride = (long)gridDim.x * 256 * 8;
  for (long i = ((long)blockIdx.x * 256 + threadIdx.x) * 8; i < n; i += stride) {
    if (i + 8 <= n) {
      float v[8];
      Vec8<T>::load(src + i, v);
      uint4 pk;
      __nv_bfloat162 b0 = __floats2bfloat162_rn(v[0], v[1]), b1 = __floats2bfloat162_rn(v[2], v[3]);
      __nv_bfloat162 b2 = __floats2bfloat162_rn(v[4], v[5]), b3 = __floats2bfloat162_rn(v[6], v[7]);
      pk.x = *reinterpret_cast<uint32_t*>(&b0); pk.y = *reinterpret_cast<uint32_t*>(&b1);
      pk.z = *reinterpret_cast<uint32_t*>(&b2); pk.w = *reinterpret_cast<uint32_t*>(&b3);
      *reinterpret_cast<uint4*>(out + i) = pk;
    } else {
      for (long k = i; k < n; ++k) out[k] = __float2bfloat16_rn(to_f32<T>(src[k]));
    }
  }
}

// ------------------------------------------------------------------------------------------------ transpose
// 64 x 64 tiles through shared memory, block (32, 8): every thread moves PAIRS (two adjacent source columns in, two
// adjacent output columns = source rows out), so a warp reads 128-256 B and writes 128 B per instruction.
template <typename T> struct Pair;
template <> struct Pair<float> { using type = float2; };
template <> struct Pair<__half> { using type = __half2; };
template <> struct Pair<__nv_bfloat16> { using type = __nv_bfloat162; };
__device__ __forceinline__ float2 pair_to_f32(float2 v) { return v; }
__device__ __forceinline__ float2 pair_to_f32(__half2 v) { return __half22float2(v); }
__device__ __forceinline__ float2 pair_to_f32(__nv_bfloat162 v) { return __bfloat1622float2(v); }

template <typename T>
__global__ void __launch_bounds__(256)
transpose_kernel(const T* __restrict__ src, long lds, __nv_bfloat16* __restrict__ out, long ldo, long rows, int cols,
                 int rowmap_div, int rowmap_mul, int rowmap_add) {
  using P = typename Pair<T>::type;
  __shared__ float tile[64][65];               // tile[c][r]
  const long r0 = (long)blockIdx.x * 64;
  const int c0 = blockIdx.y * 64;
  const int tx = threadIdx.x, ty = threadIdx.y;
  const bool src_pairs = ((lds & 1) == 0) && ((reinterpret_cast<uintptr_t>(src) & (2 * sizeof(T) - 1)) == 0);
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int rl = ty + 8 * i;
    const long r = r0 + rl;
    const int c = c0 + 2 * tx;
    float2 v = make_float2(0.f, 0.f);
    if (r < rows && c < cols) {
      const long sr = rowmap_div > 0 ? (long)rowmap_mul * (r / rowmap_div) + (r % rowmap_div) + rowmap_add : r;
      const T* p = src + sr * lds + c;
      if (src_pairs && c + 1 < cols) v = pair_to_f32(*reinterpret_cast<const P*>(p));
      else { v.x = to_f32<T>(p[0]); if (c + 1 < cols) v.y = to_f32<T>(p[1]); }
    }
    tile[2 * tx][rl] = v.x;
    tile[2 * tx + 1][rl] = v.y;
  }
  __syncthreads();
  const bool dst_pairs = ((ldo & 1) == 0) && ((reinterpret_cast<uintptr_t>(out) & 3) == 0);
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int cl = ty + 8 * i;
    const int c = c0 + cl;
    const long r = r0 + 2 * tx;
    if (c >= cols || r >= rows) continue;
    __nv_bfloat16* q = out + (long)c * ldo + r;
    if (dst_pairs && r + 1 < rows) *reinterpret_cast<__nv_bfloat162*>(q) = __floats2bfloat162_rn(tile[cl][2 * tx], tile[cl][2 * tx + 1]);
    else { q[0] = __float2bfloat16_rn(tile[cl][2 * tx]); if (r + 1 < rows) q[1] = __float2bfloat16_rn(tile[cl][2 * tx + 1]); }
  }
}

// ------------------------------------------------------------------------------------------------ quick-GELU backward
__global__ void __launch_bounds__(256)
dgelu_kernel(const float* __restrict__ dh, const __half* __restrict__ u, __nv_bfloat16* __restrict__ du, long n) {
  const long stride = (long)gridDim.x * 256 * 4;
  for (long i = ((long)blockIdx.x * 256 + threadIdx.x) * 4; i < n; i += stride) {
    const int cnt = (i + 4 <= n) ? 4 : (int)(n - i);
    float r[4];
    for (int k = 0; k < cnt; ++k) {
      const float x = __half2float(u[i + k]);
      const float s = 1.0f / (1.0f + __expf(-1.702f * x));
      r[k] = dh[i + k] * (s * (1.0f + 1.702f * x * (1.0f - s)));   // d/dx [x * sigmoid(1.702 x)]
    }
    for (int k = 0; k < cnt; ++k) du[i + k] = __float2bfloat16_rn(r[k]);
  }
}

// ------------------------------------------------------------------------------------------------ LayerNorm backward
// One warp per row, row in registers as NV4 float4 per lane (same lane-strided mapping as the forward kernel).
//   xhat = (x - mean) * rstd;  g = gamma * dy;  dx = rstd * (g - mean(g) - xhat * mean(g * xhat))
template <int NV4, bool PARAM_GRADS>
__global__ void __launch_bounds__(256, 2)
ln_backward_kernel(const float* __restrict__ dy, const float* __restrict__ x, const float* __restrict__ gamma,
                   float* __restrict__ dx_out, int accumulate, float* __restrict__ dgamma, float* __restrict__ dbeta,
                   __nv_bfloat16* __restrict__ dx_bf16, long rows, float eps) {
  constexpr int hidden = NV4 * 128;
  // PARAM_GRADS: warp-private gamma / beta gradient accumulators in shared memory, [warp][gamma|beta][NV4][lane] float4
  // (64 KB at hidden 1024; registers would cost 64 per thread and halve the occupancy of this HBM-bound kernel)
  extern __shared__ float4 acc_sm[];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const long warps = ((long)gridDim.x * blockDim.x) >> 5;
  float4* my_g = acc_sm + (size_t)(warp * 2 + 0) * NV4 * 32 + lane;
  float4* my_b = acc_sm + (size_t)(warp * 2 + 1) * NV4 * 32 + lane;
  if (PARAM_GRADS) {
#pragma unroll
    for (int i = 0; i < NV4; ++i) my_g[i * 32] = my_b[i * 32] = make_float4(0.f, 0.f, 0.f, 0.f);
  }
  for (long row = ((long)blockIdx.x * blockDim.x + threadIdx.x) >> 5; row < rows; row += warps) {
    float4 xv[NV4], dv[NV4];
    const float4* xr = reinterpret_cast<const float4*>(x + row * hidden);
    const float4* dr = reinterpret_cast<const float4*>(dy + row * hidden);
#pragma unroll
    for (int i = 0; i < NV4; ++i) { xv[i] = xr[lane + 32 * i]; dv[i] = dr[lane + 32 * i]; }
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < NV4; ++i) s += (xv[i].x + xv[i].y) + (xv[i].z + xv[i].w);
    const float mean = warp_sum(s) / hidden;
    float ss = 0.f;
#pragma unroll
    for (int i = 0; i < NV4; ++i) {
      xv[i].x -= mean; xv[i].y -= mean; xv[i].z -= mean; xv[i].w -= mean;
      ss += (xv[i].x * xv[i].x + xv[i].y * xv[i].y) + (xv[i].z * xv[i].z + xv[i].w * xv[i].w);
    }
    const float rstd = rsqrtf(warp_sum(ss) / hidden + eps);
    float s1 = 0.f, s2 = 0.f;
#pragma unroll
    for (int i = 0; i < NV4; ++i) {
      const float4 gm = __ldg(reinterpret_cast<const float4*>(gamma) + lane + 32 * i);
      xv[i].x *= rstd; xv[i].y *= rstd; xv[i].z *= rstd; xv[i].w *= rstd;       // xhat
      if (PARAM_GRADS) {
        float4 g = my_g[i * 32], b = my_b[i * 32];
        g.x += dv[i].x * xv[i].x; g.y += dv[i].y * xv[i].y; g.z += dv[i].z * xv[i].z; g.w += dv[i].w * xv[i].w;
        b.x += dv[i].x; b.y += dv[i].y; b.z += dv[i].z; b.w += dv[i].w;
        my_g[i * 32] = g;
        my_b[i * 32] = b;
      }
      dv[i].x *= gm.x; dv[i].y *= gm.y; dv[i].z *= gm.z; dv[i].w *= gm.w;       // g = gamma * dy
      s1 += (dv[i].x + dv[i].y) + (dv[i].z + dv[i].w);
      s2 += (dv[i].x * xv[i].x + dv[i].y * xv[i].y) + (dv[i].z * xv[i].z + dv[i].w * xv[i].w);
    }
    s1 = warp_sum(s1) / hidden;
    s2 = warp_sum(s2) / hidden;
    float4* outr = reinterpret_cast<float4*>(dx_out + row * hidden);
#pragma unroll
    for (int i = 0; i < NV4; ++i) {
      float4 o;
      o.x = rstd * (dv[i].x - s1 - xv[i].x * s2);
      o.y = rstd * (dv[i].y - s1 - xv[i].y * s2);
      o.z = rstd * (dv[i].z - s1 - xv[i].z * s2);
      o.w = rstd * (dv[i].w - s1 - xv[i].w * s2);
      if (accumulate) {
        const float4 p = outr[lane + 32 * i];
        o.x += p.x; o.y += p.y; o.z += p.z; o.w += p.w;
      }
      outr[lane + 32 * i] = o;
      if (dx_bf16 != nullptr) {
        __nv_bfloat162 a = __floats2bfloat162_rn(o.x, o.y), b = __floats2bfloat162_rn(o.z, o.w);
        uint2 pk;
        pk.x = *reinterpret_cast<uint32_t*>(&a);
        pk.y = *reinterpret_cast<uint32_t*>(&b);
        reinterpret_cast<uint2*>(dx_bf16 + row * hidden)[lane + 32 * i] = pk;
      }
    }
  }
  if (PARAM_GRADS) {
    __syncthreads();
    // column c = 128 i + 4 lane + e lives in float4 slot (i, lane), component e, of every warp's accumulators
    const float* flat = reinterpret_cast<const float*>(acc_sm);
    for (int idx = threadIdx.x; idx < 2 * hidden; idx += 256) {
      const int which = idx / hidden, c = idx - which * hidden;
      float t = 0.f;
#pragma unroll
      for (int w = 0; w < 8; ++w) t += flat[((size_t)(w * 2 + which) * NV4 * 32) * 4 + c];
      atomicAdd((which == 0 ? dgamma : dbeta) + c, t);
    }
  }
}

// ------------------------------------------------------------------------------------------------ attention delta
// Half-warp per (row, head) unit: lane l covers the head's columns 4 (l & 15) .. + 3, and a warp takes units 2 w and 2 w + 1
// (for even head counts, two heads of one row).  Every unit's products and shuffle order do not depend on the head count.
__global__ void __launch_bounds__(256)
attention_delta_kernel(const float* __restrict__ d_out, const __half* __restrict__ out, float* __restrict__ delta,
                       __nv_bfloat16* __restrict__ do_bf16, long units, int seq, int heads) {
  const int lane = threadIdx.x & 31;
  const long warps = ((long)gridDim.x * blockDim.x) >> 5;
  for (long pair = ((long)blockIdx.x * blockDim.x + threadIdx.x) >> 5; 2 * pair < units; pair += warps) {
    const long unit = 2 * pair + (lane >> 4);   // the loop bound is warp-uniform, so the full-warp shuffles below are legal
    const bool ok = unit < units;
    const long row = unit / heads;
    const int head = (int)(unit - row * heads);
    const long view = row / seq;
    const int t = (int)(row - view * seq);
    const size_t col = (size_t)row * heads * 64 + head * 64 + 4 * (lane & 15);
    float4 d = make_float4(0.f, 0.f, 0.f, 0.f);
    uint2 o = make_uint2(0u, 0u);
    if (ok) {
      d = *reinterpret_cast<const float4*>(d_out + col);
      o = *reinterpret_cast<const uint2*>(out + col);
    }
    const float2 o01 = __half22float2(*reinterpret_cast<const __half2*>(&o.x));
    const float2 o23 = __half22float2(*reinterpret_cast<const __half2*>(&o.y));
    float p = (d.x * o01.x + d.y * o01.y) + (d.z * o23.x + d.w * o23.y);
#pragma unroll
    for (int s = 8; s > 0; s >>= 1) p += __shfl_xor_sync(0xffffffffu, p, s);   // within each half-warp
    if (!ok) continue;
    if ((lane & 15) == 0) delta[(view * heads + head) * seq + t] = p;
    __nv_bfloat162 a = __floats2bfloat162_rn(d.x, d.y), b = __floats2bfloat162_rn(d.z, d.w);
    uint2 pk;
    pk.x = *reinterpret_cast<uint32_t*>(&a);
    pk.y = *reinterpret_cast<uint32_t*>(&b);
    *reinterpret_cast<uint2*>(do_bf16 + col) = pk;
  }
}

// ------------------------------------------------------------------------------------------------ token mean / embedding
__global__ void __launch_bounds__(256)
token_mean_backward_kernel(const float* __restrict__ d_emb, float* __restrict__ g, int tokens, int hidden, float inv) {
  const int view = blockIdx.x;
  const int h4 = hidden >> 2;
  const float4* src = reinterpret_cast<const float4*>(d_emb + (long)view * hidden);
  float4* dst = reinterpret_cast<float4*>(g + (long)view * tokens * hidden);
  for (long i = (long)blockIdx.y * 256 + threadIdx.x; i < (long)tokens * h4; i += (long)gridDim.y * 256) {
    float4 v = src[i % h4];
    v.x *= inv; v.y *= inv; v.z *= inv; v.w *= inv;
    dst[i] = v;
  }
}

__global__ void __launch_bounds__(256)
embed_backward_kernel(const float* __restrict__ d_e, float* __restrict__ dpos, float* __restrict__ dcls, int n_views,
                      int tokens, int hidden) {
  const long total = (long)tokens * hidden;
  for (long i = (long)blockIdx.x * 256 + threadIdx.x; i < total; i += (long)gridDim.x * 256) {
    float s = 0.f;
    for (int v = 0; v < n_views; ++v) s += d_e[(long)v * total + i];
    dpos[i] += s;
    if (dcls && i < hidden) dcls[i] += s;     // token 0 is the class token (the text tower has none)
  }
}

// ------------------------------------------------------------------------------------------------ bias gradients
// grid (cols / 256, row chunks); partial column sums combined with atomics.
template <typename T>
__global__ void __launch_bounds__(256)
column_sum_kernel(const T* __restrict__ x, long ldx, float* __restrict__ out, long rows, int cols, int rows_per_block) {
  const int c = blockIdx.x * 256 + threadIdx.x;
  if (c >= cols) return;
  const long r0 = (long)blockIdx.y * rows_per_block;
  long r1 = r0 + rows_per_block;
  if (r1 > rows) r1 = rows;
  float s = 0.f;
  for (long r = r0; r < r1; ++r) s += to_f32<T>(x[r * ldx + c]);
  atomicAdd(out + c, s);
}

}  // namespace

int cast_to_bf16(const void* src, int src_type, void* out, long n, cudaStream_t stream) {
  if (n <= 0) return 0;
  if ((reinterpret_cast<uintptr_t>(src) | reinterpret_cast<uintptr_t>(out)) & 15) {
    set_last_error("cast_to_bf16: buffers must be 16-byte aligned");
    return 1;
  }
  ProfScope prof("train_cast_bf16", stream);
  const int grid = grid_1d(n, 2048);
  if (src_type == SRC_F32) cast_kernel<float><<<grid, 256, 0, stream>>>(reinterpret_cast<const float*>(src), reinterpret_cast<__nv_bfloat16*>(out), n);
  else if (src_type == SRC_F16) cast_kernel<__half><<<grid, 256, 0, stream>>>(reinterpret_cast<const __half*>(src), reinterpret_cast<__nv_bfloat16*>(out), n);
  else { set_last_error("cast_to_bf16: bad source type %d", src_type); return 1; }
  return check_launch("cast_to_bf16");
}

int transpose_to_bf16(const void* src, int src_type, long lds, void* out, long ldo, long rows, int cols, int rowmap_div,
                      int rowmap_mul, int rowmap_add, cudaStream_t stream) {
  if (rows <= 0 || cols <= 0) return 0;
  if (ldo < rows) { set_last_error("transpose_to_bf16: ldo %ld < rows %ld", ldo, rows); return 1; }
  ProfScope prof("train_transpose_bf16", stream);
  const dim3 grid((unsigned)((rows + 63) / 64), (unsigned)((cols + 63) / 64)), block(32, 8);
  __nv_bfloat16* o = reinterpret_cast<__nv_bfloat16*>(out);
  if (src_type == SRC_F32) transpose_kernel<float><<<grid, block, 0, stream>>>(reinterpret_cast<const float*>(src), lds, o, ldo, rows, cols, rowmap_div, rowmap_mul, rowmap_add);
  else if (src_type == SRC_F16) transpose_kernel<__half><<<grid, block, 0, stream>>>(reinterpret_cast<const __half*>(src), lds, o, ldo, rows, cols, rowmap_div, rowmap_mul, rowmap_add);
  else if (src_type == SRC_BF16) transpose_kernel<__nv_bfloat16><<<grid, block, 0, stream>>>(reinterpret_cast<const __nv_bfloat16*>(src), lds, o, ldo, rows, cols, rowmap_div, rowmap_mul, rowmap_add);
  else { set_last_error("transpose_to_bf16: bad source type %d", src_type); return 1; }
  return check_launch("transpose_to_bf16");
}

int dgelu_bf16(const float* dh, const void* u, void* du, long n, cudaStream_t stream) {
  if (n <= 0) return 0;
  ProfScope prof("train_dgelu", stream);
  dgelu_kernel<<<grid_1d(n, 1024), 256, 0, stream>>>(dh, reinterpret_cast<const __half*>(u), reinterpret_cast<__nv_bfloat16*>(du), n);
  return check_launch("dgelu_bf16");
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

template <int NV4>
void launch_ln_backward_params(int blocks, size_t smem, cudaStream_t stream, const float* dy, const float* x,
                               const float* gamma, float* dx_out, int accumulate, float* dgamma, float* dbeta,
                               __nv_bfloat16* d16, long rows, float eps) {
  auto kern = ln_backward_kernel<NV4, true>;
  if (smem > 48 * 1024) cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  kern<<<blocks, 256, smem, stream>>>(dy, x, gamma, dx_out, accumulate, dgamma, dbeta, d16, rows, eps);
}

int layernorm_backward(const float* dy, const float* x, const float* gamma, float* dx_out, int accumulate, float* dgamma,
                       float* dbeta, void* dx_bf16, long rows, int hidden, float eps, int num_sms, cudaStream_t stream) {
  if (hidden % 128) { set_last_error("layernorm_backward: hidden %d not a multiple of 128", hidden); return 1; }
  if ((dgamma == nullptr) != (dbeta == nullptr)) { set_last_error("layernorm_backward: dgamma and dbeta go together"); return 1; }
  if (rows <= 0) return 0;
  long blocks = (rows + 7) / 8;
  const long cap = (long)(num_sms > 0 ? num_sms : 132) * 8;
  if (blocks > cap) blocks = cap;
  ProfScope prof("train_ln_backward", stream);
  __nv_bfloat16* d16 = reinterpret_cast<__nv_bfloat16*>(dx_bf16);
  if (dgamma != nullptr) {
    const size_t smem = (size_t)8 * 2 * hidden * sizeof(float);
    PG_DISPATCH_NV4(hidden, (launch_ln_backward_params<NV4>((int)blocks, smem, stream, dy, x, gamma, dx_out, accumulate,
                                                            dgamma, dbeta, d16, rows, eps)));
  } else {
    PG_DISPATCH_NV4(hidden, (ln_backward_kernel<NV4, false><<<(int)blocks, 256, 0, stream>>>(dy, x, gamma, dx_out, accumulate,
                                                                                           dgamma, dbeta, d16, rows, eps)));
  }
  return check_launch("layernorm_backward");
}

int attention_delta(const float* d_out, const void* out_f16, float* delta, void* do_bf16, int n_views, int seq, int heads,
                    int num_sms, cudaStream_t stream) {
  if (heads <= 0) { set_last_error("attention_delta: heads %d < 1", heads); return 1; }
  const long units = (long)n_views * seq * heads;
  if (units <= 0) return 0;
  long blocks = (units + 15) / 16;   // 8 warps per block, two units per warp
  const long cap = (long)(num_sms > 0 ? num_sms : 132) * 8;
  if (blocks > cap) blocks = cap;
  ProfScope prof("train_attention_delta", stream);
  attention_delta_kernel<<<(int)blocks, 256, 0, stream>>>(d_out, reinterpret_cast<const __half*>(out_f16), delta,
                                                          reinterpret_cast<__nv_bfloat16*>(do_bf16), units, seq, heads);
  return check_launch("attention_delta");
}

int token_mean_backward(const float* d_emb, float* g, int n_views, int tokens, int hidden, cudaStream_t stream) {
  if (hidden % 4) { set_last_error("token_mean_backward: hidden %d not a multiple of 4", hidden); return 1; }
  if (n_views <= 0) return 0;
  ProfScope prof("train_token_mean_backward", stream);
  token_mean_backward_kernel<<<dim3(n_views, 8), 256, 0, stream>>>(d_emb, g, tokens, hidden, 1.0f / tokens);
  return check_launch("token_mean_backward");
}

int embed_backward(const float* d_e, float* dpos, float* dcls, int n_views, int tokens, int hidden, cudaStream_t stream) {
  if (n_views <= 0) return 0;
  ProfScope prof("train_embed_backward", stream);
  embed_backward_kernel<<<grid_1d((long)tokens * hidden, 256), 256, 0, stream>>>(d_e, dpos, dcls, n_views, tokens, hidden);
  return check_launch("embed_backward");
}

int column_sum_accumulate(const void* x, int src_type, long ldx, float* out, long rows, int cols, cudaStream_t stream) {
  if (rows <= 0 || cols <= 0) return 0;
  const int rpb = 128;
  const dim3 grid((cols + 255) / 256, (unsigned)((rows + rpb - 1) / rpb));
  ProfScope prof("train_column_sum", stream);
  if (src_type == SRC_F32) column_sum_kernel<float><<<grid, 256, 0, stream>>>(reinterpret_cast<const float*>(x), ldx, out, rows, cols, rpb);
  else if (src_type == SRC_BF16) column_sum_kernel<__nv_bfloat16><<<grid, 256, 0, stream>>>(reinterpret_cast<const __nv_bfloat16*>(x), ldx, out, rows, cols, rpb);
  else { set_last_error("column_sum_accumulate: bad source type %d", src_type); return 1; }
  return check_launch("column_sum_accumulate");
}

}  // namespace pg
