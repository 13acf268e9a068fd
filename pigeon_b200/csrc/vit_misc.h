// Internal (C++) interface of the memory-bound vision-tower kernels; see vit_misc.cu.
#pragma once
#include <cuda_runtime.h>

namespace pg {

int im2col(const void* pixels, int pixels_are_f16, void* out_f16, int n_views, int img, int patch, int kpad,
           int num_sms, cudaStream_t stream);
int layernorm_f16(const float* x, void* y_f16, const float* gamma, const float* beta, long rows, int hidden, float eps,
                  int num_sms, cudaStream_t stream);
int embed_preln(float* x, const float* cls, const float* pos, const float* gamma, const float* beta, long rows,
                int tokens, int hidden, float eps, int num_sms, cudaStream_t stream, float* e_out = nullptr,
                void* x16 = nullptr, float* stats = nullptr);   // x16 fp16 [rows, hidden] + stats float2 [rows, hidden / 128]:
                                                                // LayerNorm-folded tower (see gemm.h)
// Text tower: x f32 [rows, hidden] = tok[ids[row]] + pos[row % S] (ids i64 [rows]; out-of-range id -> NaN row).
int text_embed(const long long* ids, const float* tok, const float* pos, float* x, long rows, int S, int hidden, int vocab,
               int num_sms, cudaStream_t stream);
// fp32 LayerNorm of rows of x f32 [., hidden] into y f32 [rows, hidden]; with ids i64 [rows, S], output row r is the LayerNorm
// of x row r * S + (first index of the largest id of row r)  (the text tower's EOS pooling).
int rows_layernorm_f32(const float* x, float* y, const float* gamma, const float* beta, long rows, int hidden, float eps,
                       const long long* ids, int S, int num_sms, cudaStream_t stream);
// Optional fp32 LayerNorm (gamma == beta == nullptr: none), then a3 fp16 [rows, 3 * hidden] = [hi | lo | hi] of the result.
int ln_split3(const float* x, void* a3, const float* gamma, const float* beta, long rows, int hidden, float eps, int num_sms,
              cudaStream_t stream);
int token_mean(const float* x, float* out, int n_views, int tokens, int hidden, cudaStream_t stream);

}  // namespace pg
