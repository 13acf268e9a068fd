// Optimizer step of the CLIP contrastive pretraining (reference training/train_modes.py:30-64, an HF Trainer of
// transformers 4.23.1 with PRETAIN_ARGS): `torch.nn.utils.clip_grad_norm_(model.parameters(), max_grad_norm)` over the
// whole flat gradient, then `transformers.optimization.AdamW.step()` (the Trainer's default optim="adamw_hf").
// Both are streaming, HBM-bound passes; the clip coefficient stays on the device so a step never waits on the host.
#include <cuda_runtime.h>
#include <math.h>

#include "pretrain.h"
#include "prof.h"
#include "tma_host.h"

namespace pg {
namespace {

constexpr int NORM_THREADS = 256;
// A fixed grid (not derived from the SM count), so the partials, and hence the bits, are the same on every device.
constexpr long NORM_MAX_BLOCKS = 1024;

long norm_blocks(long n) {
  const long b = (n + NORM_THREADS - 1) / NORM_THREADS;
  return b < NORM_MAX_BLOCKS ? b : NORM_MAX_BLOCKS;
}

// Tree sum of one double per thread over the block, in a fixed order; the result is valid in thread 0.
__device__ double block_sum(double s) {
  __shared__ double warp_sums[NORM_THREADS / 32];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_down_sync(0xffffffffu, s, o);
  if ((threadIdx.x & 31) == 0) warp_sums[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x < 32) {
    s = threadIdx.x < NORM_THREADS / 32 ? warp_sums[threadIdx.x] : 0.0;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_down_sync(0xffffffffu, s, o);
  }
  return s;
}

// Each thread sums the exact fp64 squares of its grid-stride elements (g * grad_scale rounded to fp32 first, as the
// scaled gradient torch would hold); one fp64 partial per block.
__global__ void __launch_bounds__(NORM_THREADS)
sq_norm_partial_kernel(const float* __restrict__ g, long n, float grad_scale, double* __restrict__ partial) {
  const long stride = (long)gridDim.x * NORM_THREADS;
  long i = (long)blockIdx.x * NORM_THREADS + threadIdx.x;
  double s = 0.0;
  for (; i + 3 * stride < n; i += 4 * stride) {
    const float a = __fmul_rn(g[i], grad_scale), b = __fmul_rn(g[i + stride], grad_scale);
    const float c = __fmul_rn(g[i + 2 * stride], grad_scale), d = __fmul_rn(g[i + 3 * stride], grad_scale);
    s += (double)a * a;
    s += (double)b * b;
    s += (double)c * c;
    s += (double)d * d;
  }
  for (; i < n; i += stride) {
    const float a = __fmul_rn(g[i], grad_scale);
    s += (double)a * a;
  }
  s = block_sum(s);
  if (threadIdx.x == 0) partial[blockIdx.x] = s;
}

// One block: the partials in a fixed order, then torch's fp32 arithmetic of clip_grad_norm_:
//   clip_coef = max_norm / (total_norm + 1e-6), clamped to at most 1 (a NaN norm gives a NaN coefficient, as torch's clamp).
__global__ void __launch_bounds__(NORM_THREADS)
norm_finish_kernel(const double* __restrict__ partial, int blocks, float max_norm, float* __restrict__ total_norm,
                   float* __restrict__ clip_coef) {
  double s = 0.0;
  for (int b = threadIdx.x; b < blocks; b += NORM_THREADS) s += partial[b];
  s = block_sum(s);
  if (threadIdx.x == 0) {
    const float t = (float)sqrt(s);
    const float c = __fdiv_rn(max_norm, __fadd_rn(t, 1e-6f));
    *total_norm = t;
    *clip_coef = c > 1.f ? 1.f : c;
  }
}

// transformers/optimization.py AdamW.step (4.23.1), per element, in its operation order, with the fused multiply-adds that
// torch's CUDA kernels compute (`a + alpha * b`, `a + alpha * (b * c)` and `a + alpha * (b / c)`, each one FMA), so the result
// follows the same torch ops on the GPU even where two terms nearly cancel:
//   grad = grad * grad_scale * clip_coef
//   exp_avg.mul_(beta1).add_(grad, alpha=1 - beta1)
//   exp_avg_sq.mul_(beta2).addcmul_(grad, grad, value=1 - beta2)
//   denom = exp_avg_sq.sqrt().add_(eps)
//   p.addcdiv_(exp_avg, denom, value=-step_size)      step_size = lr * sqrt(1 - beta2^t) / (1 - beta1^t)
//   p.add_(p, alpha=-lr * weight_decay)                  (weight_decay > 0 only: decoupled decay after the update)
__global__ void __launch_bounds__(256)
adamw_hf_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ m, float* __restrict__ v, long n,
                float grad_scale, const float* __restrict__ clip_coef, float beta1, float one_minus_beta1, float beta2,
                float one_minus_beta2, float eps, float neg_step_size, float neg_lr_wd, int decay) {
  const float coef = clip_coef ? *clip_coef : 1.f;
  for (long i = (long)blockIdx.x * 256 + threadIdx.x; i < n; i += (long)gridDim.x * 256) {
    const float gi = __fmul_rn(__fmul_rn(g[i], grad_scale), coef);
    const float mi = __fmaf_rn(one_minus_beta1, gi, __fmul_rn(m[i], beta1));
    const float vi = __fmaf_rn(one_minus_beta2, __fmul_rn(gi, gi), __fmul_rn(v[i], beta2));
    const float denom = __fadd_rn(__fsqrt_rn(vi), eps);
    float pi = __fmaf_rn(neg_step_size, __fdiv_rn(mi, denom), p[i]);
    if (decay) pi = __fmaf_rn(neg_lr_wd, pi, pi);
    p[i] = pi;
    m[i] = mi;
    v[i] = vi;
  }
}

int check_launch(const char* what) {
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) { set_last_error("%s launch: %s", what, cudaGetErrorString(e)); return 1; }
  return 0;
}

}  // namespace

size_t grad_norm_clip_workspace_bytes(long n) { return n > 0 ? (size_t)norm_blocks(n) * sizeof(double) : 0; }

int grad_norm_clip(const float* grad, long n, double grad_scale, double max_norm, float* total_norm, float* clip_coef,
                   void* workspace, size_t workspace_bytes, cudaStream_t stream) {
  const long blocks = norm_blocks(n);
  if (workspace_bytes < grad_norm_clip_workspace_bytes(n)) {
    set_last_error("grad_norm_clip: workspace of %zu bytes, need %zu", workspace_bytes, grad_norm_clip_workspace_bytes(n));
    return 1;
  }
  ProfScope prof("pretrain_grad_norm", stream);
  double* partial = static_cast<double*>(workspace);
  sq_norm_partial_kernel<<<(int)blocks, NORM_THREADS, 0, stream>>>(grad, n, (float)grad_scale, partial);
  if (check_launch("grad_norm_clip")) return 1;
  norm_finish_kernel<<<1, NORM_THREADS, 0, stream>>>(partial, (int)blocks, (float)max_norm, total_norm, clip_coef);
  return check_launch("grad_norm_clip");
}

int adamw_hf_step(float* p, const float* g, float* m, float* v, long n, double lr, double beta1, double beta2, double eps,
                  double weight_decay, long step, double grad_scale, const float* clip_coef, cudaStream_t stream) {
  const double bc1 = 1.0 - pow(beta1, (double)step), bc2 = 1.0 - pow(beta2, (double)step);
  const double step_size = lr * sqrt(bc2) / bc1;
  long blocks = (n + 255) / 256;
  if (blocks > 132 * 16) blocks = 132 * 16;
  ProfScope prof("pretrain_adamw_hf", stream);
  adamw_hf_kernel<<<(int)blocks, 256, 0, stream>>>(p, g, m, v, n, (float)grad_scale, clip_coef, (float)beta1,
                                                   (float)(1.0 - beta1), (float)beta2, (float)(1.0 - beta2), (float)eps,
                                                   (float)(-step_size), (float)(-lr * weight_decay),
                                                   weight_decay > 0.0 ? 1 : 0);
  return check_launch("adamw_hf_step");
}

}  // namespace pg
