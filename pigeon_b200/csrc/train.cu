// Fine-tune step, head-only part (reference training/train_eval_loop.py:164-253 with a frozen / absent base model:
// loss.backward() through cell_layer, torch.optim.AdamW.step()).  The Linear's backward is two small fp32 GEMMs
// (C x D x B, about 1 GFLOP) and the optimizer is a 28 B/parameter streaming update: CUDA-core kernels, HBM/launch-bound.
#include <cuda_runtime.h>
#include <math.h>

#include "prof.h"
#include "tma_host.h"
#include "train.h"

namespace pg {
namespace {

constexpr int TM = 64, TN = 64, TK = 16;

// 256 threads, 4x4 register tile per thread, operands staged k-major in shared memory.
template <bool A_T>
__global__ void __launch_bounds__(256)
sgemm_kernel(const float* __restrict__ A, const float* __restrict__ B, float* __restrict__ C, int M, int N, int K,
             float beta) {
  __shared__ __align__(16) float As[TK][TM + 4];
  __shared__ __align__(16) float Bs[TK][TN + 4];
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  const int m0 = blockIdx.y * TM, n0 = blockIdx.x * TN;
  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;

  for (int k0 = 0; k0 < K; k0 += TK) {
    // A tile -> As[k][m]
    if (A_T) {
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int e = tid + i * 256, k = e >> 6, m = e & 63;
        As[k][m] = (k0 + k < K && m0 + m < M) ? A[(long)(k0 + k) * M + m0 + m] : 0.f;
      }
    } else {
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int e = tid + i * 256, m = e >> 4, k = e & 15;
        As[k][m] = (k0 + k < K && m0 + m < M) ? A[(long)(m0 + m) * K + k0 + k] : 0.f;
      }
    }
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int e = tid + i * 256, k = e >> 6, n = e & 63;
      Bs[k][n] = (k0 + k < K && n0 + n < N) ? B[(long)(k0 + k) * N + n0 + n] : 0.f;
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < TK; ++k) {
      const float4 a = *reinterpret_cast<const float4*>(&As[k][ty * 4]);
      const float4 b = *reinterpret_cast<const float4*>(&Bs[k][tx * 4]);
      const float av[4] = {a.x, a.y, a.z, a.w}, bv[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int m = m0 + ty * 4 + i;
    if (m >= M) continue;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int n = n0 + tx * 4 + j;
      if (n >= N) continue;
      float* c = C + (long)m * N + n;
      *c = beta != 0.f ? fmaf(beta, *c, acc[i][j]) : acc[i][j];
    }
  }
}

__global__ void __launch_bounds__(256)
column_sum_kernel(const float* __restrict__ x, float* __restrict__ out, int rows, int cols, float beta) {
  const int c = blockIdx.x * 256 + threadIdx.x;
  if (c >= cols) return;
  float s = 0.f;
  for (int r = 0; r < rows; ++r) s += x[(long)r * cols + c];
  out[c] = beta != 0.f ? fmaf(beta, out[c], s) : s;
}

// Operation order of torch/optim/adamw.py (_single_tensor_adamw): decay, lerp, second moment, bias-corrected step.
__global__ void __launch_bounds__(256)
adamw_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ m, float* __restrict__ v, long n,
             float decay, float w1, float beta2, float one_minus_beta2, float bc2_sqrt, float eps, float neg_step_size,
             float grad_scale) {
  for (long i = (long)blockIdx.x * 256 + threadIdx.x; i < n; i += (long)gridDim.x * 256) {
    const float gi = __fmul_rn(g[i], grad_scale);
    float pi = __fmul_rn(p[i], decay);
    const float mi = __fadd_rn(m[i], __fmul_rn(w1, __fsub_rn(gi, m[i])));
    const float vi = __fadd_rn(__fmul_rn(v[i], beta2), __fmul_rn(__fmul_rn(one_minus_beta2, gi), gi));
    const float denom = __fadd_rn(__fdiv_rn(__fsqrt_rn(vi), bc2_sqrt), eps);
    pi = __fadd_rn(pi, __fmul_rn(neg_step_size, __fdiv_rn(mi, denom)));
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

int sgemm_f32(bool a_transposed, const float* A, const float* B, float* C, int M, int N, int K, float beta,
              cudaStream_t stream) {
  ProfScope prof("train_sgemm", stream);
  dim3 grid((N + TN - 1) / TN, (M + TM - 1) / TM);
  if (a_transposed) sgemm_kernel<true><<<grid, 256, 0, stream>>>(A, B, C, M, N, K, beta);
  else sgemm_kernel<false><<<grid, 256, 0, stream>>>(A, B, C, M, N, K, beta);
  return check_launch("sgemm_f32");
}

int column_sum_f32(const float* x, float* out, int rows, int cols, float beta, cudaStream_t stream) {
  ProfScope prof("train_column_sum", stream);
  column_sum_kernel<<<(cols + 255) / 256, 256, 0, stream>>>(x, out, rows, cols, beta);
  return check_launch("column_sum_f32");
}

int adamw_step(float* p, const float* g, float* m, float* v, long n, double lr, double beta1, double beta2, double eps,
               double weight_decay, long step, double grad_scale, cudaStream_t stream) {
  const double bc1 = 1.0 - pow(beta1, (double)step), bc2 = 1.0 - pow(beta2, (double)step);
  long blocks = (n + 255) / 256;
  if (blocks > 132 * 16) blocks = 132 * 16;
  ProfScope prof("train_adamw", stream);
  adamw_kernel<<<(int)blocks, 256, 0, stream>>>(p, g, m, v, n, (float)(1.0 - lr * weight_decay), (float)(1.0 - beta1),
                                                (float)beta2, (float)(1.0 - beta2), (float)sqrt(bc2), (float)eps,
                                                (float)(-(lr / bc1)), (float)grad_scale);
  return check_launch("adamw_step");
}

}  // namespace pg
