// Pooled row of the text tower (transformers 4.23.1 CLIPTextTransformer: `input_ids.argmax(dim=-1)`), shared by the
// forward's pooling LayerNorm (vit_misc.cu) and its backward (clip_train.cu).
#pragma once
#include <limits.h>

namespace pg {

// First index of the largest id of ids[0 .. S), computed by the 32 lanes of a warp; every lane returns it.
__device__ __forceinline__ int first_argmax_warp(const long long* __restrict__ ids, int S, int lane) {
  long long bv = LLONG_MIN;
  int bt = S;
  for (int t = lane; t < S; t += 32) {
    const long long v = ids[t];
    if (v > bv) { bv = v; bt = t; }   // ascending t per lane: the first maximum of the lane
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const long long ov = __shfl_xor_sync(0xffffffffu, bv, o);
    const int ot = __shfl_xor_sync(0xffffffffu, bt, o);
    if (ov > bv || (ov == bv && ot < bt)) { bv = ov; bt = ot; }
  }
  return bt;
}

}  // namespace pg
