// Internal (C++) interface of the wgmma GEMM; the C ABI in capi.cu wraps it.
#pragma once
#include <cuda_runtime.h>

namespace pg {

enum GemmEpilogue {
  EPI_F16_BIAS = 0,        // out fp16 = acc + bias
  EPI_F16_BIAS_QGELU = 1,  // out fp16 = quick_gelu(acc + bias)
  EPI_F32_BIAS_RESID = 2,  // out fp32 += acc + bias     (in-place residual stream update)
  EPI_F32_BIAS = 3,        // out fp32 = acc + bias      (bias may be null)
  EPI_F32_ROWMAP = 4,      // out fp32[rowmap(row)] = acc + bias ; rowmap(r) = mul*(r/div) + r%div + add
  EPI_BF16_DGELU = 5,      // out bf16 = acc * quick_gelu'(aux fp16)          (backward through mlp.fc1's activation)
  EPI_F16_BIAS_QGELU_SAVE = 6,  // out fp16 = quick_gelu(acc + bias), aux fp16 = acc + bias (training forward of mlp.fc1)
  // LayerNorm folded into the GEMMs either side of it (inference tower; no LayerNorm kernel, no normalised copy in HBM):
  EPI_F32_BIAS_RESID_STATS = 7,  // EPI_F32_BIAS_RESID + aux fp16 = the new residual row, stats[row][col / 128] = (sum, sum of
                                 // squares) of those fp16 values over 128 columns  (producer: out_proj, fc2)
  EPI_F16_LN_BIAS = 8,           // out fp16 = rstd * (acc - mu * colsum) + bias, (mu, rstd) of the A row from `stats`;
                                 // A = the raw fp16 residual row, W = gamma-scaled weight, bias = b + W beta  (consumer: qkv)
  EPI_F16_LN_BIAS_QGELU = 9,     // quick_gelu of the same                                        (consumer: fc1)
};

struct GemmProblem {
  int M, N, K;
  const void* a;  // fp16 [M, lda]
  int lda;
  const void* w;  // fp16 [N, ldw]
  int ldw;
  void* out;
  int ldo;
  const float* bias;
  int epi;
  int rowmap_div, rowmap_mul, rowmap_add;
  int operand_bf16;     // A and W both hold bf16 instead of fp16 (backward GEMMs; mixed pairs are illegal on the tensor cores)
  const float* resid;   // EPI_F32_BIAS_RESID: residual read from here instead of `out` (same ldo); nullptr = in place
  void* aux;            // fp16 [M, ldo]: pre-activation read by EPI_BF16_DGELU / written by EPI_F16_BIAS_QGELU_SAVE
  // Both operands stored with the CONTRACTION index outermost: a = [K, lda] (M contiguous), w = [K, ldw] (N contiguous),
  // i.e. D = a^T w — the weight-gradient form (dW = dY^T X) fed straight from row-major activations as MN-major wgmma
  // operands (M > 128, N % 256 == 0).
  int mn_major;
  // LayerNorm-folded epilogues: stats float2 [M, K / 128] (consumer, read) or [M, N / 128] (producer, written);
  // colsum fp32 [N] = row sums of the (gamma-scaled, fp16-rounded) weight; ln_eps of the LayerNorm.
  float* stats;
  const float* colsum;
  float ln_eps;
};

// Enqueues the GEMM on `stream`. Returns 0 on success; on failure the message is in pg::last_error().
int gemm_f16(const GemmProblem& p, int num_sms, cudaStream_t stream);

// Kernel choice for K-major problems, process-wide: 0 = automatic (the 128 x 256 kernel for the fp16-output and fp32 residual
// epilogues, else the ping-pong kernel), 1 = the single-warpgroup kernel, 2 = the ping-pong kernel.
int gemm_set_schedule(int mode);

}  // namespace pg
