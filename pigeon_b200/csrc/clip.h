// Internal (C++) interface of the image-text logits kernels; see clip.cu.
#pragma once
#include <cuda_runtime.h>

namespace pg {

// img f32 [Ni, P], txt f32 [Nt, P] (not normalised) -> lpi f32 [Ni, Nt] = cos(img_i, txt_t) * exp(logit_scale);
// optional: lpt f32 [Nt, Ni] (its transpose), probs f32 [Ni, Nt] (softmax over captions), pred i64 [Ni] (first argmax),
// loss f32 [1] (symmetric cross-entropy against arange; Ni == Nt).
int clip_logits(const float* img, int Ni, const float* txt, int Nt, int P, float logit_scale, float* lpi, float* lpt,
                float* probs, long long* pred, float* loss, cudaStream_t stream);

}  // namespace pg
