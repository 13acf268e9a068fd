// Internal (C++) interface of the wgmma attention core; the C ABI in capi.cu wraps it.
#pragma once
#include <cuda_runtime.h>

namespace pg {

// qkv: fp16 [n_views*seq, 3*heads*64]; out: fp16 [n_views*seq, heads*64]. head_dim is 64.
// lse2 (optional): f32 [n_views*heads, seq], log2-domain log-sum-exp of the scaled logits, kept for the backward pass.
int attention_f16(const void* qkv, void* out, int n_views, int seq, int heads, cudaStream_t stream,
                  float* lse2 = nullptr);
// The text tower's variant: causal (key j admissible for query i only if j <= i) and / or a key mask i64 [n_views, seq]
// (0 = excluded).  mask == nullptr and causal == 0 runs attention_f16 itself.  mask[v, 0] must be non-zero.
// lse2 (optional) as for attention_f16, over the admissible keys of each query.
int attention_f16_masked(const void* qkv, void* out, const long long* mask, int causal, int n_views, int seq, int heads,
                         cudaStream_t stream, float* lse2 = nullptr);

// Backward of the attention core (attention_bwd_wgmma.cu).
//   qkv f16 / qkv_bf16 [n_views*seq, 3*heads*64] (same values, two operand types), d_out_bf16 [n_views*seq, heads*64],
//   lse2 / delta f32 [n_views*heads, seq]  ->  dqkv bf16 [n_views*seq, 3*heads*64]
int attention_backward(const void* qkv_f16, const void* qkv_bf16, const void* d_out_bf16, const float* lse2,
                       const float* delta, void* dqkv_bf16, int n_views, int seq, int heads, cudaStream_t stream);
// The same with the admissibility predicate of attention_f16_masked applied to the recomputed logits (lse2 must come from
// the masked forward).  mask == nullptr and causal == 0 runs attention_backward itself.
int attention_backward_masked(const void* qkv_f16, const void* qkv_bf16, const void* d_out_bf16, const float* lse2,
                              const float* delta, void* dqkv_bf16, const long long* mask, int causal, int n_views, int seq,
                              int heads, cudaStream_t stream);

}  // namespace pg
