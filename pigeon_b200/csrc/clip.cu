// Image-text logits of HF CLIPModel.forward (transformers 4.23.1 modeling_clip.py), fp32 on the CUDA cores:
//   image_embeds / |image_embeds|, text_embeds / |text_embeds|,
//   logits_per_text = text @ image^T * exp(logit_scale),  logits_per_image = logits_per_text^T,
//   loss = (CE(logits_per_text, arange) + CE(logits_per_image, arange)) / 2           (clip_loss)
// and what the reference reads from them (dataset_creation/pretrain/pretrain_dataset.py:299-330):
// logits_per_image.softmax(1) and its first-max argmax per image.
// The sizes are small (1024 images x 1000 captions x 768 is 0.8 GFMA), so a register-blocked fp32 tile GEMM does it.
#include "clip.h"

#include <math.h>
#include <stdint.h>

#include "prof.h"
#include "tma_host.h"

namespace pg {

namespace {

constexpr int kTile = 64;   // 64 images x 64 captions per CTA, 4 x 4 per thread
constexpr int kBK = 16;

// The row norms come out of the same pass: every CTA streams its 64 image rows and 64 caption rows over all of P.
__global__ void __launch_bounds__(256)
clip_logits_kernel(const float* __restrict__ img, int Ni, const float* __restrict__ txt, int Nt, int P, float scale,
                   float* __restrict__ lpi, float* __restrict__ lpt) {
  __shared__ float As[kBK][kTile + 4], Bs[kBK][kTile + 4];
  __shared__ float inv_a[kTile], inv_b[kTile];
  const int tid = threadIdx.x;
  const int i0 = blockIdx.y * kTile, t0 = blockIdx.x * kTile;
  const int lr = tid >> 2, lk = (tid & 3) * 4;   // loader: row lr of the tile, 4 consecutive k from lk
  const int ty = tid >> 4, tx = tid & 15;        // compute: rows 4 ty .. 4 ty + 3, columns 4 tx .. 4 tx + 3
  const float* ar = img + (long)(i0 + lr) * P;
  const float* br = txt + (long)(t0 + lr) * P;
  const bool a_ok = i0 + lr < Ni, b_ok = t0 + lr < Nt;
  float ssa = 0.f, ssb = 0.f;
  float acc[4][4];
#pragma unroll
  for (int r = 0; r < 4; ++r)
#pragma unroll
    for (int c = 0; c < 4; ++c) acc[r][c] = 0.f;
  for (int k0 = 0; k0 < P; k0 += kBK) {
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const int k = k0 + lk + q;
      const float a = (a_ok && k < P) ? __ldg(ar + k) : 0.f;
      const float b = (b_ok && k < P) ? __ldg(br + k) : 0.f;
      As[lk + q][lr] = a;
      Bs[lk + q][lr] = b;
      ssa = fmaf(a, a, ssa);
      ssb = fmaf(b, b, ssb);
    }
    __syncthreads();
#pragma unroll
    for (int kk = 0; kk < kBK; ++kk) {
      const float4 a = *reinterpret_cast<const float4*>(&As[kk][4 * ty]);
      const float4 b = *reinterpret_cast<const float4*>(&Bs[kk][4 * tx]);
      const float av[4] = {a.x, a.y, a.z, a.w}, bv[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
      for (int r = 0; r < 4; ++r)
#pragma unroll
        for (int c = 0; c < 4; ++c) acc[r][c] = fmaf(av[r], bv[c], acc[r][c]);
    }
    __syncthreads();
  }
  // the four loader lanes of a row are adjacent in the warp
  ssa += __shfl_xor_sync(0xffffffffu, ssa, 1);
  ssa += __shfl_xor_sync(0xffffffffu, ssa, 2);
  ssb += __shfl_xor_sync(0xffffffffu, ssb, 1);
  ssb += __shfl_xor_sync(0xffffffffu, ssb, 2);
  if ((tid & 3) == 0) {
    inv_a[lr] = 1.0f / sqrtf(ssa);
    inv_b[lr] = 1.0f / sqrtf(ssb);
  }
  __syncthreads();
#pragma unroll
  for (int r = 0; r < 4; ++r) {
    const int i = i0 + 4 * ty + r;
    if (i >= Ni) continue;
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      const int t = t0 + 4 * tx + c;
      if (t >= Nt) continue;
      const float v = (acc[r][c] * inv_a[4 * ty + r]) * inv_b[4 * tx + c] * scale;
      lpi[(long)i * Nt + t] = v;
      if (lpt) lpt[(long)t * Ni + i] = v;
    }
  }
}

// One warp per image row of logits_per_image [Ni, Nt]: softmax over the captions (torch: exp(x - max) / sum) and the
// first index of the maximum logit (torch.argmax; the softmax is monotone, so it is the argmax of the probabilities too).
__global__ void clip_softmax_argmax_kernel(const float* __restrict__ lpi, int Ni, int Nt, float* __restrict__ probs,
                                           long long* __restrict__ pred) {
  const int lane = threadIdx.x & 31;
  const int row = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (row >= Ni) return;
  const float* x = lpi + (long)row * Nt;
  float m = -INFINITY;
  int mi = Nt;
  for (int t = lane; t < Nt; t += 32) {
    const float v = x[t];
    if (v > m) { m = v; mi = t; }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float om = __shfl_xor_sync(0xffffffffu, m, o);
    const int oi = __shfl_xor_sync(0xffffffffu, mi, o);
    if (om > m || (om == m && oi < mi)) { m = om; mi = oi; }
  }
  if (pred && lane == 0) pred[row] = mi;
  if (!probs) return;
  float s = 0.f;
  for (int t = lane; t < Nt; t += 32) s += expf(x[t] - m);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  const float inv = 1.0f / s;
  for (int t = lane; t < Nt; t += 32) probs[(long)row * Nt + t] = expf(x[t] - m) * inv;
}

// Symmetric cross-entropy against arange(N) in one CTA (deterministic): warp w takes rows w, w + 32, ...; per row the
// log-sum-exp in fp64 of the image row lpi[r, :] and of the caption row (lpt[r, :] when given, else column r of lpi).
__global__ void __launch_bounds__(1024)
clip_loss_kernel(const float* __restrict__ lpi, const float* __restrict__ lpt, int N, float* __restrict__ loss) {
  __shared__ double red[32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  double acc = 0.0;
  for (int r = warp; r < N; r += 32) {
    for (int side = 0; side < 2; ++side) {
      const float* x = side == 0 ? lpi + (long)r * N : (lpt ? lpt + (long)r * N : lpi + r);
      const long stride = (side == 1 && !lpt) ? N : 1;
      double m = -INFINITY;
      for (int t = lane; t < N; t += 32) m = fmax(m, (double)x[t * stride]);
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) m = fmax(m, __shfl_xor_sync(0xffffffffu, m, o));
      double s = 0.0;
      for (int t = lane; t < N; t += 32) s += exp((double)x[t * stride] - m);
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
      if (lane == 0) acc += m + log(s) - (double)lpi[(long)r * N + r];
    }
  }
  if (lane == 0) red[warp] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    double t = 0.0;
    for (int w = 0; w < 32; ++w) t += red[w];
    *loss = (float)(t / (2.0 * N));
  }
}

int check_launch(const char* what) {
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) { set_last_error("%s launch: %s", what, cudaGetErrorString(e)); return 1; }
  return 0;
}

}  // namespace

int clip_logits(const float* img, int Ni, const float* txt, int Nt, int P, float logit_scale, float* lpi, float* lpt,
                float* probs, long long* pred, float* loss, cudaStream_t stream) {
  if (Ni <= 0 || Nt <= 0) return 0;
  if (P <= 0) { set_last_error("clip_logits: bad projection dim %d", P); return 1; }
  if (loss && Ni != Nt) { set_last_error("clip_logits: the loss needs as many images as captions (%d != %d)", Ni, Nt); return 1; }
  if ((Ni + kTile - 1) / kTile > 65535) { set_last_error("clip_logits: %d images exceed the grid", Ni); return 1; }
  const float scale = expf(logit_scale);
  {
    ProfScope prof("clip_logits", stream);
    dim3 grid((Nt + kTile - 1) / kTile, (Ni + kTile - 1) / kTile);
    clip_logits_kernel<<<grid, 256, 0, stream>>>(img, Ni, txt, Nt, P, scale, lpi, lpt);
    if (check_launch("clip_logits")) return 1;
  }
  if (probs || pred) {
    ProfScope prof("clip_softmax_argmax", stream);
    clip_softmax_argmax_kernel<<<(Ni + 7) / 8, 256, 0, stream>>>(lpi, Ni, Nt, probs, pred);
    if (check_launch("clip_softmax_argmax")) return 1;
  }
  if (loss) {
    ProfScope prof("clip_loss", stream);
    clip_loss_kernel<<<1, 1024, 0, stream>>>(lpi, lpt, Ni, loss);
    if (check_launch("clip_loss")) return 1;
  }
  return 0;
}

}  // namespace pg
