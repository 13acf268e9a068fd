// Memory-bound pieces of the CLIP vision tower around the wgmma GEMM / attention kernels:
// patch extraction (im2col), class-token + position embedding + pre_layrnorm, per-block LayerNorm,
// the token mean-pool that the reference applies to last_hidden_state
// (models/clip_embedder.py:64-65, models/super_guessr.py:396-398), and the text tower's token + position embedding.
#include "vit_misc.h"

#include <cuda_fp16.h>
#include <limits.h>
#include <stdint.h>

#include "prof.h"
#include "text_pool.cuh"
#include "tma_host.h"

namespace pg {

namespace {

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// ------------------------------------------------------------------------------------------------
// im2col: pixels [n, 3, img, img] -> A [n * gp * gp, kpad] fp16, k = c*P*P + ky*P + kx (the flattening
// of nn.Conv2d(3, hidden, P, P).weight), columns [3*P*P, kpad) zero.
// ------------------------------------------------------------------------------------------------
// One thread per 16-byte piece of the output (8 consecutive k of one patch row): the 8 source pixels are gathered (runs of
// up to `patch` contiguous pixels; neighbouring threads read neighbouring addresses, so the lines come from L1), the store is
// one coalesced 128-bit write.  (The first version wrote 2 bytes per thread at a 28-byte granularity: 0.5 TB/s.)
template <typename T>
__global__ void im2col_kernel(const T* __restrict__ px, __half* __restrict__ out, int n_views, int img, int patch,
                              int kpad) {
  const int gp = img / patch;
  const int pp = patch * patch;
  const int kreal = 3 * pp;
  const int groups = kpad >> 3;                              // 16-byte pieces per output row (kpad % 64 == 0)
  const long total = (long)n_views * gp * gp * groups;
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const int g = (int)(i % groups);
    const long row = i / groups;                             // (view, py, pxx)
    const int pxx = (int)(row % gp);
    const int py = (int)((row / gp) % gp);
    const long n = row / ((long)gp * gp);
    const T* src = px + n * 3 * (long)img * img + (long)(py * patch) * img + pxx * patch;
    __align__(16) __half v[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int k = g * 8 + j;
      float f = 0.f;
      if (k < kreal) {
        const int c = k / pp, r = k - c * pp;
        const int ky = r / patch, kx = r - ky * patch;
        f = (float)src[(long)c * img * img + (long)ky * img + kx];
      }
      v[j] = __float2half_rn(f);
    }
    *reinterpret_cast<uint4*>(out + row * kpad + g * 8) = *reinterpret_cast<const uint4*>(v);
  }
}

// ------------------------------------------------------------------------------------------------
// LayerNorm helpers: one warp per row, row held in registers as NV4 float4 per lane
// (lane-strided so that global accesses are fully coalesced 512-byte warp transactions).
// ------------------------------------------------------------------------------------------------
template <int NV4>
__device__ __forceinline__ void ln_row(float4 (&v)[NV4], const float* __restrict__ g, const float* __restrict__ b,
                                       int hidden, float eps, int lane) {
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < NV4; ++i) s += (v[i].x + v[i].y) + (v[i].z + v[i].w);
  const float mean = warp_sum(s) / hidden;
  float ss = 0.f;
#pragma unroll
  for (int i = 0; i < NV4; ++i) {
    const float a = v[i].x - mean, bb = v[i].y - mean, c = v[i].z - mean, d = v[i].w - mean;
    ss += (a * a + bb * bb) + (c * c + d * d);
  }
  const float rstd = rsqrtf(warp_sum(ss) / hidden + eps);
#pragma unroll
  for (int i = 0; i < NV4; ++i) {
    const float4 gg = __ldg(reinterpret_cast<const float4*>(g) + lane + 32 * i);
    const float4 bb = __ldg(reinterpret_cast<const float4*>(b) + lane + 32 * i);
    v[i].x = (v[i].x - mean) * rstd * gg.x + bb.x;
    v[i].y = (v[i].y - mean) * rstd * gg.y + bb.y;
    v[i].z = (v[i].z - mean) * rstd * gg.z + bb.z;
    v[i].w = (v[i].w - mean) * rstd * gg.w + bb.w;
  }
}

// x fp32 [rows, hidden] -> y fp16 [rows, hidden]
template <int NV4>
__global__ void layernorm_f16_kernel(const float* __restrict__ x, __half* __restrict__ y, const float* __restrict__ g,
                                     const float* __restrict__ b, long rows, float eps) {
  constexpr int hidden = NV4 * 128;
  const int lane = threadIdx.x & 31;
  const long warps = ((long)gridDim.x * blockDim.x) >> 5;
  for (long row = ((long)blockIdx.x * blockDim.x + threadIdx.x) >> 5; row < rows; row += warps) {
    float4 v[NV4];
    const float4* xr = reinterpret_cast<const float4*>(x + row * hidden);
#pragma unroll
    for (int i = 0; i < NV4; ++i) v[i] = xr[lane + 32 * i];
    ln_row<NV4>(v, g, b, hidden, eps, lane);
    uint2* yr = reinterpret_cast<uint2*>(y + row * hidden);
#pragma unroll
    for (int i = 0; i < NV4; ++i) {
      __half2 lo = __floats2half2_rn(v[i].x, v[i].y), hi = __floats2half2_rn(v[i].z, v[i].w);
      uint2 pk;
      pk.x = *reinterpret_cast<uint32_t*>(&lo);
      pk.y = *reinterpret_cast<uint32_t*>(&hi);
      yr[lane + 32 * i] = pk;
    }
  }
}

// Residual-stream initialisation, in place on x fp32 [n_views*tokens, hidden]:
//   token 0   : class_embedding + position_embedding[0]
//   token t>0 : x (patch GEMM output already stored there) + position_embedding[t]
// followed by pre_layrnorm (HF CLIPVisionTransformer: embeddings -> pre_layrnorm -> encoder).
template <int NV4>
__global__ void embed_preln_kernel(float* __restrict__ x, const float* __restrict__ cls, const float* __restrict__ pos,
                                   const float* __restrict__ g, const float* __restrict__ b, long rows, int tokens,
                                   float eps, float* __restrict__ e_out, __half* __restrict__ x16,
                                   float2* __restrict__ stats, int stats_slots) {
  constexpr int hidden = NV4 * 128;
  const int lane = threadIdx.x & 31;
  const long warps = ((long)gridDim.x * blockDim.x) >> 5;
  for (long row = ((long)blockIdx.x * blockDim.x + threadIdx.x) >> 5; row < rows; row += warps) {
    const int t = row % tokens;
    float4 v[NV4];
    float4* xr = reinterpret_cast<float4*>(x + row * hidden);
    const float4* src = (t == 0) ? reinterpret_cast<const float4*>(cls) : xr;
    const float4* pr = reinterpret_cast<const float4*>(pos + (long)t * hidden);
#pragma unroll
    for (int i = 0; i < NV4; ++i) {
      const float4 a = src[lane + 32 * i];
      const float4 p = __ldg(pr + lane + 32 * i);
      v[i] = make_float4(a.x + p.x, a.y + p.y, a.z + p.z, a.w + p.w);
    }
    if (e_out != nullptr) {   // training: keep the pre-LayerNorm embedding sum for the backward pass
      float4* er = reinterpret_cast<float4*>(e_out + row * hidden);
#pragma unroll
      for (int i = 0; i < NV4; ++i) er[lane + 32 * i] = v[i];
    }
    ln_row<NV4>(v, g, b, hidden, eps, lane);
#pragma unroll
    for (int i = 0; i < NV4; ++i) xr[lane + 32 * i] = v[i];
    if (x16 != nullptr) {   // LayerNorm-folded tower: fp16 copy of the row (the first GEMM's A operand) and its moments
      uint2* hr = reinterpret_cast<uint2*>(x16 + row * hidden);
      float s1 = 0.f, s2 = 0.f;
#pragma unroll
      for (int i = 0; i < NV4; ++i) {
        const __half2 lo = __floats2half2_rn(v[i].x, v[i].y), hi = __floats2half2_rn(v[i].z, v[i].w);
        uint2 pk;
        pk.x = *reinterpret_cast<const uint32_t*>(&lo);
        pk.y = *reinterpret_cast<const uint32_t*>(&hi);
        hr[lane + 32 * i] = pk;
        const float2 a = __half22float2(lo), c = __half22float2(hi);
        s1 += (a.x + a.y) + (c.x + c.y);
        s2 += fmaf(a.x, a.x, a.y * a.y) + fmaf(c.x, c.x, c.y * c.y);
      }
      s1 = warp_sum(s1);
      s2 = warp_sum(s2);
      if (lane < stats_slots) stats[row * stats_slots + lane] = (lane == 0) ? make_float2(s1, s2) : make_float2(0.f, 0.f);
    }
  }
}

// Text embeddings (HF CLIPTextEmbeddings, modeling_clip.py 4.23.1): x fp32 [n * S, hidden] row (b, t) =
// token_embedding[ids[b, t]] + position_embedding[t].  No LayerNorm follows (the text tower has no pre-LN).  An id outside
// [0, vocab) is never used as an index: its row becomes NaN, which is loud where HF raises an index error.
__global__ void text_embed_kernel(const long long* __restrict__ ids, const float* __restrict__ tok,
                                  const float* __restrict__ pos, float* __restrict__ x, long rows, int S, int hidden,
                                  int vocab) {
  const int lane = threadIdx.x & 31;
  const int h4 = hidden >> 2;
  const long warps = ((long)gridDim.x * blockDim.x) >> 5;
  for (long row = ((long)blockIdx.x * blockDim.x + threadIdx.x) >> 5; row < rows; row += warps) {
    const long long id = ids[row];
    const bool ok = id >= 0 && id < vocab;
    const float4* tr = reinterpret_cast<const float4*>(tok + (ok ? id : 0) * (long)hidden);
    const float4* pr = reinterpret_cast<const float4*>(pos + (long)(row % S) * hidden);
    float4* xr = reinterpret_cast<float4*>(x + row * hidden);
    for (int i = lane; i < h4; i += 32) {
      const float4 a = __ldg(tr + i), p = __ldg(pr + i);
      xr[i] = ok ? make_float4(a.x + p.x, a.y + p.y, a.z + p.z, a.w + p.w) : make_float4(NAN, NAN, NAN, NAN);
    }
  }
}

// Final LayerNorm of the text tower in fp32 (HF CLIPTextTransformer.final_layer_norm), row by row:
//   ids == nullptr: y[r] = LN(x[r])                                 (last_hidden_state, rows = n * S)
//   ids != nullptr: y[r] = LN(x[r * S + argmax_t ids[r, t]])         (pooled output, rows = n; first index of the largest
//                   id, transformers 4.23.1 `input_ids.argmax(dim=-1)`; the LayerNorm is per row, so pooling before or
//                   after it gives the same row)
template <int NV4>
__global__ void rows_layernorm_f32_kernel(const float* __restrict__ x, float* __restrict__ y, const float* __restrict__ g,
                                          const float* __restrict__ b, long rows, float eps,
                                          const long long* __restrict__ ids, int S) {
  constexpr int hidden = NV4 * 128;
  const int lane = threadIdx.x & 31;
  const long warps = ((long)gridDim.x * blockDim.x) >> 5;
  for (long row = ((long)blockIdx.x * blockDim.x + threadIdx.x) >> 5; row < rows; row += warps) {
    long src = row;
    if (ids != nullptr) src = row * S + first_argmax_warp(ids + row * S, S, lane);
    float4 v[NV4];
    const float4* xr = reinterpret_cast<const float4*>(x + src * hidden);
#pragma unroll
    for (int i = 0; i < NV4; ++i) v[i] = xr[lane + 32 * i];
    ln_row<NV4>(v, g, b, hidden, eps, lane);
    float4* yr = reinterpret_cast<float4*>(y + row * hidden);
#pragma unroll
    for (int i = 0; i < NV4; ++i) yr[lane + 32 * i] = v[i];
  }
}

// Operand of the error-compensated projection GEMM (the geocell head's scheme, head.cu): optional fp32 LayerNorm
// (g == nullptr: none), then x = hi + lo in fp16 and a3 [rows, 3 * hidden] = [hi | lo | hi], to be multiplied by the
// [Whi | Whi | Wlo] packing of pg_head_pack_weight.
template <int NV4>
__global__ void ln_split3_kernel(const float* __restrict__ x, __half* __restrict__ a3, const float* __restrict__ g,
                                 const float* __restrict__ b, long rows, float eps) {
  constexpr int hidden = NV4 * 128;
  const int lane = threadIdx.x & 31;
  const long warps = ((long)gridDim.x * blockDim.x) >> 5;
  for (long row = ((long)blockIdx.x * blockDim.x + threadIdx.x) >> 5; row < rows; row += warps) {
    float4 v[NV4];
    const float4* xr = reinterpret_cast<const float4*>(x + row * hidden);
#pragma unroll
    for (int i = 0; i < NV4; ++i) v[i] = xr[lane + 32 * i];
    if (g != nullptr) ln_row<NV4>(v, g, b, hidden, eps, lane);
    uint2* hr = reinterpret_cast<uint2*>(a3 + row * 3 * hidden);
    uint2* lr = reinterpret_cast<uint2*>(a3 + row * 3 * hidden + hidden);
    uint2* h2 = reinterpret_cast<uint2*>(a3 + row * 3 * hidden + 2 * hidden);
#pragma unroll
    for (int i = 0; i < NV4; ++i) {
      const __half2 h01 = __floats2half2_rn(v[i].x, v[i].y), h23 = __floats2half2_rn(v[i].z, v[i].w);
      const float2 f01 = __half22float2(h01), f23 = __half22float2(h23);
      const __half2 l01 = __floats2half2_rn(v[i].x - f01.x, v[i].y - f01.y);
      const __half2 l23 = __floats2half2_rn(v[i].z - f23.x, v[i].w - f23.y);
      uint2 ph, pl;
      ph.x = *reinterpret_cast<const uint32_t*>(&h01);
      ph.y = *reinterpret_cast<const uint32_t*>(&h23);
      pl.x = *reinterpret_cast<const uint32_t*>(&l01);
      pl.y = *reinterpret_cast<const uint32_t*>(&l23);
      hr[lane + 32 * i] = ph;
      lr[lane + 32 * i] = pl;
      h2[lane + 32 * i] = ph;
    }
  }
}

// mean over tokens: x fp32 [n_views, tokens, hidden] -> out fp32 [n_views, hidden]
// block = (hidden/4 threads, 1); each thread owns 4 adjacent columns; grid = (n_views, splits) with
// partial sums combined through shared memory when blockDim.y > 1.
__global__ void token_mean_kernel(const float* __restrict__ x, float* __restrict__ out, int tokens, int hidden) {
  extern __shared__ float4 red[];
  const int view = blockIdx.x;
  const int c4 = threadIdx.x;  // float4 column index
  const int h4 = hidden >> 2;
  const float4* xv = reinterpret_cast<const float4*>(x + (long)view * tokens * hidden);
  float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
  for (int t = threadIdx.y; t < tokens; t += blockDim.y) {
    const float4 a = xv[(long)t * h4 + c4];
    acc.x += a.x; acc.y += a.y; acc.z += a.z; acc.w += a.w;
  }
  red[threadIdx.y * h4 + c4] = acc;
  __syncthreads();
  if (threadIdx.y == 0) {
    for (int y = 1; y < blockDim.y; ++y) {
      const float4 a = red[y * h4 + c4];
      acc.x += a.x; acc.y += a.y; acc.z += a.z; acc.w += a.w;
    }
    const float inv = 1.0f / tokens;
    reinterpret_cast<float4*>(out + (long)view * hidden)[c4] =
        make_float4(acc.x * inv, acc.y * inv, acc.z * inv, acc.w * inv);
  }
}

int check_launch(const char* what) {
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) {
    set_last_error("%s launch: %s", what, cudaGetErrorString(e));
    return 1;
  }
  return 0;
}

inline int grid_for(long work_items, int per_block, int num_sms) {
  long blocks = (work_items + per_block - 1) / per_block;
  const long cap = (long)num_sms * 16;
  if (blocks > cap) blocks = cap;
  if (blocks < 1) blocks = 1;
  return (int)blocks;
}

}  // namespace

int im2col(const void* pixels, int pixels_are_f16, void* out, int n_views, int img, int patch, int kpad, int num_sms,
           cudaStream_t stream) {
  if (img % patch) { set_last_error("im2col: image size %d not a multiple of patch %d", img, patch); return 1; }
  if (kpad < 3 * patch * patch || (kpad & 7)) { set_last_error("im2col: kpad must cover 3 * patch^2 and be a multiple of 8"); return 1; }
  if (reinterpret_cast<uintptr_t>(out) & 15) { set_last_error("im2col: output must be 16-byte aligned"); return 1; }
  const long total = (long)n_views * (img / patch) * (img / patch) * (kpad >> 3);
  const int grid = grid_for(total, 256 * 2, num_sms);
  ProfScope prof("im2col", stream);
  if (pixels_are_f16)
    im2col_kernel<__half><<<grid, 256, 0, stream>>>(reinterpret_cast<const __half*>(pixels),
                                                    reinterpret_cast<__half*>(out), n_views, img, patch, kpad);
  else
    im2col_kernel<float><<<grid, 256, 0, stream>>>(reinterpret_cast<const float*>(pixels),
                                                   reinterpret_cast<__half*>(out), n_views, img, patch, kpad);
  return check_launch("im2col");
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

int layernorm_f16(const float* x, void* y, const float* gamma, const float* beta, long rows, int hidden, float eps,
                  int num_sms, cudaStream_t stream) {
  if (hidden % 128) { set_last_error("layernorm: hidden %d not a multiple of 128", hidden); return 1; }
  const int grid = grid_for(rows, 8, num_sms);
  ProfScope prof("layernorm", stream);
  PG_DISPATCH_NV4(hidden, (layernorm_f16_kernel<NV4><<<grid, 256, 0, stream>>>(
                              x, reinterpret_cast<__half*>(y), gamma, beta, rows, eps)));
  return check_launch("layernorm");
}

int embed_preln(float* x, const float* cls, const float* pos, const float* gamma, const float* beta, long rows,
                int tokens, int hidden, float eps, int num_sms, cudaStream_t stream, float* e_out, void* x16,
                float* stats) {
  if (hidden % 128) { set_last_error("embed_preln: hidden %d not a multiple of 128", hidden); return 1; }
  if ((x16 == nullptr) != (stats == nullptr) || hidden / 128 > 32) { set_last_error("embed_preln: x16 and stats go together (hidden <= 4096)"); return 1; }
  const int grid = grid_for(rows, 8, num_sms);
  ProfScope prof("embed_preln", stream);
  PG_DISPATCH_NV4(hidden, (embed_preln_kernel<NV4><<<grid, 256, 0, stream>>>(x, cls, pos, gamma, beta, rows,
                                                                               tokens, eps, e_out,
                                                                               reinterpret_cast<__half*>(x16),
                                                                               reinterpret_cast<float2*>(stats),
                                                                               hidden / 128)));
  return check_launch("embed_preln");
}

int rows_layernorm_f32(const float* x, float* y, const float* gamma, const float* beta, long rows, int hidden, float eps,
                       const long long* ids, int S, int num_sms, cudaStream_t stream) {
  if (hidden % 128) { set_last_error("rows_layernorm_f32: hidden %d not a multiple of 128", hidden); return 1; }
  const int grid = grid_for(rows, 8, num_sms);
  ProfScope prof(ids ? "text_pool_ln" : "layernorm_f32", stream);
  PG_DISPATCH_NV4(hidden, (rows_layernorm_f32_kernel<NV4><<<grid, 256, 0, stream>>>(x, y, gamma, beta, rows, eps, ids, S)));
  return check_launch("rows_layernorm_f32");
}

int ln_split3(const float* x, void* a3, const float* gamma, const float* beta, long rows, int hidden, float eps, int num_sms,
              cudaStream_t stream) {
  if (hidden % 128) { set_last_error("ln_split3: hidden %d not a multiple of 128", hidden); return 1; }
  if ((gamma == nullptr) != (beta == nullptr)) { set_last_error("ln_split3: LayerNorm gamma and beta go together"); return 1; }
  const int grid = grid_for(rows, 8, num_sms);
  ProfScope prof("clip_project_split", stream);
  PG_DISPATCH_NV4(hidden, (ln_split3_kernel<NV4><<<grid, 256, 0, stream>>>(x, reinterpret_cast<__half*>(a3), gamma, beta,
                                                                             rows, eps)));
  return check_launch("ln_split3");
}

int text_embed(const long long* ids, const float* tok, const float* pos, float* x, long rows, int S, int hidden, int vocab,
               int num_sms, cudaStream_t stream) {
  if (hidden % 4) { set_last_error("text_embed: hidden %d not a multiple of 4", hidden); return 1; }
  const int grid = grid_for(rows, 8, num_sms);
  ProfScope prof("text_embed", stream);
  text_embed_kernel<<<grid, 256, 0, stream>>>(ids, tok, pos, x, rows, S, hidden, vocab);
  return check_launch("text_embed");
}

int token_mean(const float* x, float* out, int n_views, int tokens, int hidden, cudaStream_t stream) {
  if (hidden % 4 || hidden / 4 > 1024) { set_last_error("token_mean: hidden %d unsupported", hidden); return 1; }
  const int h4 = hidden / 4;
  int ny = 1024 / h4;
  if (ny > 8) ny = 8;
  if (ny < 1) ny = 1;
  dim3 block(h4, ny);
  ProfScope prof("token_mean", stream);
  token_mean_kernel<<<n_views, block, (size_t)ny * h4 * sizeof(float4), stream>>>(x, out, tokens, hidden);
  return check_launch("token_mean");
}

}  // namespace pg
