// Internal (C++) interface of the CLIP pretraining optimizer step (global-norm clipping, the HF AdamW update); see
// pretrain.cu.
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>

namespace pg {

// Bytes of workspace grad_norm_clip needs for n elements (one fp64 partial per block).
size_t grad_norm_clip_workspace_bytes(long n);
// total_norm = ||grad * grad_scale||_2, clip_coef = min(max_norm / (total_norm + 1e-6), 1) (NaN passes through);
// deterministic: fixed grid for a given n, fixed-order fp64 partials, one finishing block.
int grad_norm_clip(const float* grad, long n, double grad_scale, double max_norm, float* total_norm, float* clip_coef,
                   void* workspace, size_t workspace_bytes, cudaStream_t stream);
// transformers.optimization.AdamW.step (4.23.1, correct_bias=True) on one flat fp32 tensor; clip_coef may be NULL.
int adamw_hf_step(float* p, const float* g, float* m, float* v, long n, double lr, double beta1, double beta2, double eps,
                  double weight_decay, long step, double grad_scale, const float* clip_coef, cudaStream_t stream);

}  // namespace pg
