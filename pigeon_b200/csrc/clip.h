// Internal (C++) interface of the image-text logits kernels; see clip.cu.
#pragma once
#include <cuda_runtime.h>

namespace pg {

// img f32 [Ni, P], txt f32 [Nt, P] (not normalised) -> lpi f32 [Ni, Nt] = cos(img_i, txt_t) * exp(logit_scale);
// optional: lpt f32 [Nt, Ni] (its transpose), probs f32 [Ni, Nt] (softmax over captions), pred i64 [Ni] (first argmax),
// loss f32 [1] (symmetric cross-entropy against arange; Ni == Nt).
int clip_logits(const float* img, int Ni, const float* txt, int Nt, int P, float logit_scale, float* lpi, float* lpt,
                float* probs, long long* pred, float* loss, cudaStream_t stream);

// Training step (clip_train.cu).  img / txt f32 [n, P] (not normalised), logit_scale: DEVICE f32 scalar ->
// loss f32 [1] = clip_loss(logits_per_text); d_img / d_txt f32 [n, P] (overwritten) and d_logit_scale f32 [1] (overwritten),
// all gradients times grad_scale; lpi / lpt (nullable) f32 [n, n] logits_per_image / logits_per_text.
size_t clip_loss_grad_workspace_bytes(int n, int P);
int clip_loss_grad(const float* img, const float* txt, int n, int P, const float* logit_scale, double grad_scale,
                   void* workspace, size_t workspace_bytes, float* loss, float* d_img, float* d_txt, float* d_logit_scale,
                   float* lpi, float* lpt, cudaStream_t stream);
// final_layer_norm backward on the pooled row of each caption: x f32 [n * S, hidden] (pre-LN residual), d_pooled f32
// [n, hidden] -> g f32 [n * S, hidden] pooled rows written (the caller zeroes the rest); dgamma / dbeta += (ordered sums;
// part f32 [n, 2 hidden] is scratch).
int text_pool_ln_backward(const float* x, const float* d_pooled, const float* gamma, const long long* ids, int n, int S,
                          int hidden, float eps, float* g, float* part, float* dgamma, float* dbeta, cudaStream_t stream);
// dtok f32 [vocab, hidden] += per-id sums of dx f32 [rows, hidden] over ids i64 [rows] (deterministic; ids outside
// [0, vocab) skipped).
int token_embedding_grad(const long long* ids, const float* dx, long rows, int hidden, int vocab, float* dtok,
                         cudaStream_t stream);

}  // namespace pg
