// Internal (C++) interface of the memory-bound kernels of the vision-tower backward pass; see train_vit.cu.
#pragma once
#include <cuda_runtime.h>

namespace pg {

enum CastSrc { SRC_F32 = 0, SRC_F16 = 1, SRC_BF16 = 2 };

// out bf16 [n] = src (f32 | f16) [n]
int cast_to_bf16(const void* src, int src_type, void* out_bf16, long n, cudaStream_t stream);
// out bf16 [cols, ldo] = transpose of src [rows, lds] (f32 | f16 | bf16).  With rowmap_div > 0 the source row of
// output column r is rowmap_mul * (r / rowmap_div) + r % rowmap_div + rowmap_add (patch-token gather).
int transpose_to_bf16(const void* src, int src_type, long lds, void* out_bf16, long ldo, long rows, int cols,
                      int rowmap_div, int rowmap_mul, int rowmap_add, cudaStream_t stream);
// du bf16 [n] = dh f32 [n] * quick_gelu'(u f16 [n])
int dgelu_bf16(const float* dh, const void* u_f16, void* du_bf16, long n, cudaStream_t stream);
// LayerNorm backward over the last dim.  dx_out (+)= dLN/dx; dgamma / dbeta (nullable) += their gradients.
// dx_bf16 (nullable): bf16 copy of the final dx_out row, so that the next GEMM needs no separate cast pass.
int layernorm_backward(const float* dy, const float* x, const float* gamma, float* dx_out, int accumulate,
                       float* dgamma, float* dbeta, void* dx_bf16, long rows, int hidden, float eps, int num_sms,
                       cudaStream_t stream);
// delta f32 [n_views*heads, seq] = sum over head_dim of dO * O;  do_bf16 = bf16(dO).  dO f32 / O f16: [n_views*seq, heads*64]
int attention_delta(const float* d_out, const void* out_f16, float* delta, void* do_bf16, int n_views, int seq, int heads,
                    int num_sms, cudaStream_t stream);
// g f32 [n_views, tokens, hidden] = d_emb [n_views, hidden] / tokens   (backward of the token mean)
int token_mean_backward(const float* d_emb, float* g, int n_views, int tokens, int hidden, cudaStream_t stream);
// dpos [tokens, hidden] += sum_views dE;  dcls [hidden] (nullable) += sum_views dE[:, 0]
int embed_backward(const float* d_e, float* dpos, float* dcls, int n_views, int tokens, int hidden, cudaStream_t stream);
// out f32 [cols] += column sums of x [rows, ldx] (f32 | bf16)
int column_sum_accumulate(const void* x, int src_type, long ldx, float* out, long rows, int cols, cudaStream_t stream);

}  // namespace pg
