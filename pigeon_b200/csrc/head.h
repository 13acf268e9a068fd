// Internal (C++) interface of the geocell-head kernels; see head.cu.
#pragma once
#include <cuda_runtime.h>

namespace pg {

int view_mean_split(const float* emb, float* pooled, void* a3_f16, int B, int V, int D, cudaStream_t stream);
int weight_split(const float* w, void* w3_f16, int C, int D, cudaStream_t stream);
int softmax_topk(const float* logits, float* probs, long long* pred_cell, double* pred_lnglat, float* topk_val,
                 long long* topk_idx, const double* centroids, int B, int C, int k, cudaStream_t stream);

// The three steps above as one kernel (head_fused_wgmma.cu): view mean + split into the A operand tiles, wgmma GEMM,
// bias, and softmax / arg-max / top-k by the CTA that completes a block of 128 samples last.  `tickets`: int per block.
bool head_fused_supported(int B, int V, int D, int C, int k);
size_t head_fused_workspace_bytes(int B);
int head_fused_forward(const float* emb, int B, int V, int D, const void* w3_f16, const float* bias,
                       const double* centroids, int C, int k, void* tickets, float* pooled, float* logits, float* probs,
                       long long* pred_cell, double* pred_lnglat, float* topk_val, long long* topk_idx,
                       cudaStream_t stream);

int ce_loss(const float* logits, int B, int C, int mode, const long long* labels_idx, const float* soft,
            const double* labels_lnglat, const double* centroids, double smoothing, double* per_sample,
            double* loss_out, float* dlogits, double grad_scale, cudaStream_t stream);

}  // namespace pg
