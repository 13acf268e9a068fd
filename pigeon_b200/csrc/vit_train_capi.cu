// C ABI of the vision-tower fine-tune step (include/pigeon_b200.h, "Fine-tune step, vision tower"): the training-mode
// forward that keeps its activations and the backward launch sequence.  Host-side orchestration only.
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

#include "../../include/pigeon_b200.h"
#include "attention.h"
#include "clip.h"
#include "gemm.h"
#include "tma_host.h"
#include "train.h"
#include "train_vit.h"
#include "vit_handle.h"
#include "vit_misc.h"

using namespace pg;

namespace {

struct BwdWs {
  float* g;        // f32 [rows, hidden]   gradient of the residual stream
  void* g16;       // bf16 [rows, hidden]
  float* t32;      // f32 [rows, hidden]   data-gradient GEMM outputs (dXn2 | dAO | dXn1 | dE)
  void* t16;       // bf16 [rows, wide]    dU | dqkv
  void* qkv_bf;    // bf16 [rows, 3 hidden]
  void* do_bf;     // bf16 [rows, hidden]
  float* delta;    // f32 [n_views*heads*tokens]
  void* at;        // bf16 [wide, rows_p]  transposed left operand of the weight-gradient GEMMs
  void* bt;        // bf16 [wide, rows_p]  transposed right operand
  long rows_p;
  size_t total;
};

// Workspace of the encoder-layer backward for n_seq sequences of seq tokens; wide_b_min widens the right transposed operand
// (the vision tower's patch embedding gradient).
BwdWs carve_encoder_bwd(int n_seq, int seq, int hidden, int heads, int intermediate, int wide_b_min, Carver& cv) {
  const size_t rows = (size_t)n_seq * seq;
  int wide = intermediate > 3 * hidden ? intermediate : 3 * hidden;
  int wide_b = wide > wide_b_min ? wide : wide_b_min;
  BwdWs w;
  w.rows_p = (long)align_up(rows, 64);
  w.g = reinterpret_cast<float*>(cv.take(rows * hidden * 4));
  w.g16 = cv.take(rows * hidden * 2);
  w.t32 = reinterpret_cast<float*>(cv.take(rows * (size_t)hidden * 4));
  w.t16 = cv.take(rows * (size_t)wide * 2);
  w.qkv_bf = cv.take(rows * (size_t)3 * hidden * 2);
  w.do_bf = cv.take(rows * hidden * 2);
  w.delta = reinterpret_cast<float*>(cv.take((size_t)n_seq * heads * seq * 4));
  w.at = cv.take((size_t)wide * w.rows_p * 2);
  w.bt = cv.take((size_t)wide_b * w.rows_p * 2);
  w.total = cv.off;
  return w;
}

BwdWs carve_bwd(const pg_vit* h, int n_views, void* ws) {
  const pg_vit_config& c = h->cfg;
  Carver cv(ws);
  return carve_encoder_bwd(n_views, h->tokens, c.hidden, c.heads, c.intermediate, c.patch_k_pad, cv);
}

// out f32 [M, N] = a bf16 [M, K] . w bf16 [N, K]^T       (data gradient)
int dgrad(const void* a, const void* w_t, float* out, long M, int N, int K, int sms, cudaStream_t st) {
  GemmProblem p{};
  p.M = (int)M; p.N = N; p.K = K;
  p.a = a; p.lda = K; p.w = w_t; p.ldw = K;
  p.out = out; p.ldo = N; p.bias = nullptr; p.epi = EPI_F32_BIAS; p.operand_bf16 = 1;
  return gemm_f16(p, sms, st);
}

// dw f32 [M, N] += left^T . right, with left [rows, M] and right [rows, N] row-major in any supported type.
// Fast path: both operands as bf16 [rows, *] straight into the GEMM as MN-major wgmma operands (a cast where the saved
// activation is fp16 — wgmma wants A and B of one type — and no transposes).  Otherwise (N % 256 != 0, the
// patch embedding, or gathered rows): transpose both to bf16 [*, rows_p] and use the K-major kernel.
int wgrad(const void* left, int left_type, long ld_left, int M, const void* right, int right_type, long ld_right, int N,
          long rows, float* dw, const BwdWs& w, int sms, cudaStream_t st, int map_div = 0, int map_mul = 0, int map_add = 0) {
  GemmProblem p{};
  p.M = M; p.N = N; p.K = (int)rows;
  p.out = dw; p.ldo = N; p.bias = nullptr; p.epi = EPI_F32_BIAS_RESID; p.operand_bf16 = 1;
  const bool direct = map_div == 0 && N % 256 == 0 && M % 64 == 0 && M > 128 && ld_left == M && ld_right == N &&
                      ld_left % 8 == 0 && ld_right % 8 == 0;
  if (direct) {
    const void* l = left;
    const void* r = right;
    if (left_type != SRC_BF16) { if (cast_to_bf16(left, left_type, w.at, rows * M, st)) return 1; l = w.at; }
    if (right_type != SRC_BF16) { if (cast_to_bf16(right, right_type, w.bt, rows * N, st)) return 1; r = w.bt; }
    p.a = l; p.lda = M; p.w = r; p.ldw = N; p.mn_major = 1;
    return gemm_f16(p, sms, st);
  }
  if (transpose_to_bf16(left, left_type, ld_left, w.at, w.rows_p, rows, M, map_div, map_mul, map_add, st)) return 1;
  if (transpose_to_bf16(right, right_type, ld_right, w.bt, w.rows_p, rows, N, 0, 0, 0, st)) return 1;
  p.a = w.at; p.lda = (int)w.rows_p; p.w = w.bt; p.ldw = (int)w.rows_p;
  return gemm_f16(p, sms, st);
}

// Training forward of the encoder-layer stack: the encoder_layers sequence with every activation the backward needs kept
// in saved[l] (saved[0].x0 holds the input; layer l writes saved[l + 1].x0, the last one x_out).  The vision tower passes
// mask NULL and causal 0, the text tower its attention_mask and causal 1.
int encoder_layers_train(const pg_vit_layer* layers, const pg_vit_saved_layer* saved, float* x_out, int n_layers, int hidden,
                         int heads, int intermediate, float eps, int n_seq, int seq, const int64_t* mask, int causal, int sms,
                         cudaStream_t stream) {
  const long rows = (long)n_seq * seq;
  for (int l = 0; l < n_layers; ++l) {
    const pg_vit_layer& L = layers[l];
    const pg_vit_saved_layer& s = saved[l];
    float* x_next = (l + 1 < n_layers) ? saved[l + 1].x0 : x_out;
    if (layernorm_f16(s.x0, s.xn1, L.ln1_g, L.ln1_b, rows, hidden, eps, sms, stream)) return 1;
    GemmProblem p{};
    p.M = (int)rows; p.N = 3 * hidden; p.K = hidden;
    p.a = s.xn1; p.lda = hidden; p.w = L.w_qkv; p.ldw = hidden;
    p.out = s.qkv; p.ldo = 3 * hidden; p.bias = L.b_qkv; p.epi = EPI_F16_BIAS;
    if (gemm_f16(p, sms, stream)) return 1;
    if (attention_f16_masked(s.qkv, s.ao, reinterpret_cast<const long long*>(mask), causal, n_seq, seq, heads, stream, s.lse2))
      return 1;
    p = GemmProblem{};
    p.M = (int)rows; p.N = hidden; p.K = hidden;
    p.a = s.ao; p.lda = hidden; p.w = L.w_o; p.ldw = hidden;
    p.out = s.x1; p.ldo = hidden; p.bias = L.b_o; p.epi = EPI_F32_BIAS_RESID; p.resid = s.x0;
    if (gemm_f16(p, sms, stream)) return 1;
    if (layernorm_f16(s.x1, s.xn2, L.ln2_g, L.ln2_b, rows, hidden, eps, sms, stream)) return 1;
    p = GemmProblem{};
    p.M = (int)rows; p.N = intermediate; p.K = hidden;
    p.a = s.xn2; p.lda = hidden; p.w = L.w_fc1; p.ldw = hidden;
    p.out = s.h; p.ldo = intermediate; p.bias = L.b_fc1; p.epi = EPI_F16_BIAS_QGELU_SAVE; p.aux = s.u;
    if (gemm_f16(p, sms, stream)) return 1;
    p = GemmProblem{};
    p.M = (int)rows; p.N = hidden; p.K = intermediate;
    p.a = s.h; p.lda = intermediate; p.w = L.w_fc2; p.ldw = intermediate;
    p.out = x_next; p.ldo = hidden; p.bias = L.b_fc2; p.epi = EPI_F32_BIAS_RESID; p.resid = s.x1;
    if (gemm_f16(p, sms, stream)) return 1;
  }
  return 0;
}

// Backward of the encoder-layer stack from w.g = d(output of layer n_layers - 1) down to layer `lowest`; leaves
// w.g = d(input of layer `lowest`).  Weight gradients of the layers whose pg_vit_layer_bwd has them accumulate (+=);
// events (nullable) as pg_vit_grads.layer_done_events.  Shared by both towers (the vision tower: mask NULL, causal 0).
int encoder_layers_backward(const pg_vit_layer* layers, const pg_vit_saved_layer* saved, const pg_vit_layer_bwd* bwd,
                            int n_layers, int lowest, int hidden, int heads, int intermediate, float eps, int n_seq, int seq,
                            const int64_t* mask, int causal, void* const* events, const BwdWs& w, int sms, cudaStream_t st,
                            const char* name) {
  const long rows = (long)n_seq * seq;
  const int H = hidden, I = intermediate;
  for (int l = n_layers - 1; l >= lowest; --l) {
    const pg_vit_layer& L = layers[l];
    const pg_vit_saved_layer& s = saved[l];
    const pg_vit_layer_bwd& B = bwd[l];
    const bool train = B.d_w_qkv != nullptr;   // every layer in [lowest, layers) is trainable or above a trainable one

    // ---- MLP block: x2 = x1 + fc2(quick_gelu(fc1(LN2(x1))))
    if (l == n_layers - 1 && cast_to_bf16(w.g, SRC_F32, w.g16, rows * H, st)) return 1;   // below, LN backward leaves g16
    {
      GemmProblem p{};                                                    // dU = (dX2 . W2) o quick_gelu'(U), fused epilogue
      p.M = (int)rows; p.N = I; p.K = H;
      p.a = w.g16; p.lda = H; p.w = B.w_fc2_t; p.ldw = H;
      p.out = w.t16; p.ldo = I; p.bias = nullptr; p.epi = EPI_BF16_DGELU; p.operand_bf16 = 1; p.aux = s.u;
      if (gemm_f16(p, sms, st)) return 1;
    }
    if (train) {
      if (wgrad(w.g16, SRC_BF16, H, H, s.h, SRC_F16, I, I, rows, B.d_w_fc2, w, sms, st)) return 1;
      if (column_sum_accumulate(w.g, SRC_F32, H, B.d_b_fc2, rows, H, st)) return 1;
      if (wgrad(w.t16, SRC_BF16, I, I, s.xn2, SRC_F16, H, H, rows, B.d_w_fc1, w, sms, st)) return 1;
      if (column_sum_accumulate(w.t16, SRC_BF16, I, B.d_b_fc1, rows, I, st)) return 1;
    }
    if (dgrad(w.t16, B.w_fc1_t, w.t32, rows, H, I, sms, st)) return 1;                         // dXn2 = dU . W1
    if (layernorm_backward(w.t32, s.x1, L.ln2_g, w.g, 1, train ? B.d_ln2_g : nullptr, train ? B.d_ln2_b : nullptr, w.g16,
                           rows, H, eps, sms, st))
      return 1;                                                                                // g = dX1 (+ bf16 copy)

    // ---- attention block: x1 = x0 + out_proj(attention(qkv(LN1(x0))))
    if (dgrad(w.g16, B.w_o_t, w.t32, rows, H, H, sms, st)) return 1;                           // dAO = dX1 . Wo
    if (train) {
      if (wgrad(w.g16, SRC_BF16, H, H, s.ao, SRC_F16, H, H, rows, B.d_w_o, w, sms, st)) return 1;
      if (column_sum_accumulate(w.g, SRC_F32, H, B.d_b_o, rows, H, st)) return 1;
    }
    if (attention_delta(w.t32, s.ao, w.delta, w.do_bf, n_seq, seq, heads, sms, st)) return 1;
    if (cast_to_bf16(s.qkv, SRC_F16, w.qkv_bf, rows * 3 * H, st)) return 1;
    if (attention_backward_masked(s.qkv, w.qkv_bf, w.do_bf, s.lse2, w.delta, w.t16, reinterpret_cast<const long long*>(mask),
                                  causal, n_seq, seq, heads, st))
      return 1;
    if (train) {
      if (wgrad(w.t16, SRC_BF16, 3 * H, 3 * H, s.xn1, SRC_F16, H, H, rows, B.d_w_qkv, w, sms, st)) return 1;
      if (column_sum_accumulate(w.t16, SRC_BF16, 3 * H, B.d_b_qkv, rows, 3 * H, st)) return 1;
    }
    if (dgrad(w.t16, B.w_qkv_t, w.t32, rows, H, 3 * H, sms, st)) return 1;                     // dXn1 = dqkv . Wqkv
    if (layernorm_backward(w.t32, s.x0, L.ln1_g, w.g, 1, train ? B.d_ln1_g : nullptr, train ? B.d_ln1_b : nullptr, w.g16,
                           rows, H, eps, sms, st))
      return 1;                                                                                // g = dX0 (+ bf16 copy)
    if (train && events && events[l]) {   // layer l's gradient bucket is final for this call
      cudaError_t e = cudaEventRecord(reinterpret_cast<cudaEvent_t>(events[l]), st);
      if (e != cudaSuccess) { set_last_error("%s: cudaEventRecord(layer %d): %s", name, l, cudaGetErrorString(e)); return 1; }
    }
  }
  return 0;
}

// Checks every layer's pg_vit_layer_bwd (gradients all set or all NULL, transposed weights present); returns the lowest
// trainable layer (n_layers if none), or -1 with last_error set.
int check_layer_grads(const pg_vit_layer_bwd* bwd, int n_layers, const char* name) {
  int lowest = n_layers;
  for (int l = 0; l < n_layers; ++l) {
    const pg_vit_layer_bwd& B = bwd[l];
    const bool any = B.d_ln1_g || B.d_ln1_b || B.d_w_qkv || B.d_b_qkv || B.d_w_o || B.d_b_o || B.d_ln2_g || B.d_ln2_b ||
                     B.d_w_fc1 || B.d_b_fc1 || B.d_w_fc2 || B.d_b_fc2;
    const bool all = B.d_ln1_g && B.d_ln1_b && B.d_w_qkv && B.d_b_qkv && B.d_w_o && B.d_b_o && B.d_ln2_g && B.d_ln2_b &&
                     B.d_w_fc1 && B.d_b_fc1 && B.d_w_fc2 && B.d_b_fc2;
    if (any && !all) { set_last_error("%s: layer %d gradients must be all set or all NULL", name, l); return -1; }
    if (any && l < lowest) lowest = l;
    if (!B.w_qkv_t || !B.w_o_t || !B.w_fc1_t || !B.w_fc2_t) { set_last_error("%s: layer %d lacks transposed weights", name, l); return -1; }
  }
  return lowest;
}

// pg_vit_backward (d_emb: gradient of the token mean) and pg_vit_backward_cls (d_cls: gradient of the CLS rows).
int vit_backward(pg_vit* h, const pg_vit_saved* sv, const float* d_emb, const float* d_cls, int32_t n_views,
                 const pg_vit_grads* gr, void* workspace, size_t workspace_bytes, void* stream_, const char* name) {
  if (!h || !sv || !sv->layers_host || !(d_emb || d_cls) || !gr || !gr->layers_host || !workspace) {
    set_last_error("%s: null argument", name);
    return 1;
  }
  if (n_views <= 0) return 0;
  const int sms = sm_count();
  if (sms < 0) return 1;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream_);
  const pg_vit_config& c = h->cfg;
  const long rows = (long)n_views * h->tokens;
  const int np = h->grid_patches * h->grid_patches;
  const int H = c.hidden;
  if (reinterpret_cast<uintptr_t>(workspace) & 255) { set_last_error("%s: workspace must be 256-byte aligned", name); return 1; }
  const BwdWs w = carve_bwd(h, n_views, workspace);
  if (workspace_bytes < w.total) { set_last_error("%s: workspace %zu < required %zu", name, workspace_bytes, w.total); return 1; }

  const bool emb_train = gr->d_patch_w || gr->d_class_emb || gr->d_pos_emb || gr->d_pre_ln_g || gr->d_pre_ln_b;
  if (emb_train && !(gr->d_patch_w && gr->d_class_emb && gr->d_pos_emb && gr->d_pre_ln_g && gr->d_pre_ln_b)) {
    set_last_error("%s: embedding gradients must be all set or all NULL", name);
    return 1;
  }
  const int lowest_layer = check_layer_grads(gr->layers_host, c.layers, name);
  if (lowest_layer < 0) return 1;
  const int lowest = emb_train ? 0 : lowest_layer;   // the backward stops below the lowest layer that needs a gradient

  if (d_emb) {
    // d last_hidden_state = d_emb / tokens for every token (backward of the token mean, super_guessr.py:397-398)
    if (token_mean_backward(d_emb, w.g, n_views, h->tokens, H, st)) return 1;
  } else {
    // d last_hidden_state = d_cls at token 0 of every view, zero elsewhere (CLIPVisionTransformer's pooled CLS row)
    const size_t row_bytes = (size_t)H * sizeof(float);
    cudaError_t e = cudaMemsetAsync(w.g, 0, (size_t)rows * row_bytes, st);
    if (e == cudaSuccess)
      e = cudaMemcpy2DAsync(w.g, (size_t)h->tokens * row_bytes, d_cls, row_bytes, row_bytes, n_views, cudaMemcpyDeviceToDevice, st);
    if (e != cudaSuccess) { set_last_error("%s: CLS seed: %s", name, cudaGetErrorString(e)); return 1; }
  }

  if (encoder_layers_backward(h->layers.data(), sv->layers_host, gr->layers_host, c.layers, lowest, H, c.heads,
                              c.intermediate, c.ln_eps, n_views, h->tokens, nullptr, 0, gr->layer_done_events, w, sms, st,
                              name))
    return 1;

  if (emb_train) {
    // pre_layrnorm backward: g = d(pre-LN output) -> t32 = dE
    if (layernorm_backward(w.g, sv->e, h->w.pre_ln_g, w.t32, 0, gr->d_pre_ln_g, gr->d_pre_ln_b, nullptr, rows, H, c.ln_eps,
                           sms, st))
      return 1;
    if (embed_backward(w.t32, gr->d_pos_emb, gr->d_class_emb, n_views, h->tokens, H, st)) return 1;
    // patch_embedding.weight [hidden, patch_k_pad] += dE[patch tokens]^T . im2col
    if (wgrad(w.t32, SRC_F32, H, H, sv->im2col, SRC_F16, c.patch_k_pad, c.patch_k_pad, (long)n_views * np, gr->d_patch_w, w,
              sms, st, np, h->tokens, 1))
      return 1;
    if (gr->layer_done_events && gr->layer_done_events[c.layers]) {
      cudaError_t e = cudaEventRecord(reinterpret_cast<cudaEvent_t>(gr->layer_done_events[c.layers]), st);
      if (e != cudaSuccess) { set_last_error("%s: cudaEventRecord(embeddings): %s", name, cudaGetErrorString(e)); return 1; }
    }
  }
  return 0;
}

}  // namespace

extern "C" {

int pg_vit_forward_train(pg_vit* h, const void* pixels, int32_t pixels_f16, int32_t n_views, const pg_vit_saved* sv,
                         float* emb_out, void* stream_) {
  if (!h || !pixels || !sv || !sv->layers_host || !sv->im2col || !sv->e || !sv->x_out || !emb_out) {
    set_last_error("pg_vit_forward_train: null argument");
    return 1;
  }
  if (n_views <= 0) return 0;
  const int sms = sm_count();
  if (sms < 0) return 1;
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  const pg_vit_config& c = h->cfg;
  const long rows = (long)n_views * h->tokens;
  const int np = h->grid_patches * h->grid_patches;
  for (int l = 0; l < c.layers; ++l) {
    const pg_vit_saved_layer& s = sv->layers_host[l];
    if (!s.x0 || !s.xn1 || !s.qkv || !s.lse2 || !s.ao || !s.x1 || !s.xn2 || !s.u || !s.h) {
      set_last_error("pg_vit_forward_train: layer %d has a null save buffer", l);
      return 1;
    }
  }
  float* x = sv->layers_host[0].x0;
  if (im2col(pixels, pixels_f16, sv->im2col, n_views, c.image_size, c.patch_size, c.patch_k_pad, sms, stream)) return 1;
  {
    GemmProblem p{};
    p.M = n_views * np; p.N = c.hidden; p.K = c.patch_k_pad;
    p.a = sv->im2col; p.lda = c.patch_k_pad; p.w = h->w.patch_w; p.ldw = c.patch_k_pad;
    p.out = x; p.ldo = c.hidden; p.bias = nullptr; p.epi = EPI_F32_ROWMAP;
    p.rowmap_div = np; p.rowmap_mul = h->tokens; p.rowmap_add = 1;
    if (gemm_f16(p, sms, stream)) return 1;
  }
  if (embed_preln(x, h->w.class_emb, h->w.pos_emb, h->w.pre_ln_g, h->w.pre_ln_b, rows, h->tokens, c.hidden, c.ln_eps, sms,
                  stream, sv->e))
    return 1;
  if (encoder_layers_train(h->layers.data(), sv->layers_host, sv->x_out, c.layers, c.hidden, c.heads, c.intermediate,
                           c.ln_eps, n_views, h->tokens, nullptr, 0, sms, stream))
    return 1;
  return token_mean(sv->x_out, emb_out, n_views, h->tokens, c.hidden, stream);
}

size_t pg_vit_backward_workspace_bytes(const pg_vit* h, int32_t n_views) {
  if (!h || n_views <= 0) return 0;
  return carve_bwd(h, n_views, nullptr).total;
}

int pg_vit_backward(pg_vit* h, const pg_vit_saved* sv, const float* d_emb, int32_t n_views, const pg_vit_grads* gr,
                    void* workspace, size_t workspace_bytes, void* stream) {
  if (!d_emb) { set_last_error("pg_vit_backward: null argument"); return 1; }
  return vit_backward(h, sv, d_emb, nullptr, n_views, gr, workspace, workspace_bytes, stream, "pg_vit_backward");
}

int pg_vit_backward_cls(pg_vit* h, const pg_vit_saved* sv, const float* d_cls, int32_t n_views, const pg_vit_grads* gr,
                        void* workspace, size_t workspace_bytes, void* stream) {
  if (!d_cls) { set_last_error("pg_vit_backward_cls: null argument"); return 1; }
  return vit_backward(h, sv, nullptr, d_cls, n_views, gr, workspace, workspace_bytes, stream, "pg_vit_backward_cls");
}

// ---------------------------------------------------------------------------------------------- CLIPModel training step
int pg_text_forward_train(pg_text* h, const int64_t* input_ids, const int64_t* attention_mask, int32_t n, int32_t S,
                          const pg_text_saved* sv, float* pooled_out, void* stream_) {
  if (!h || !input_ids || !sv || !sv->layers_host || !sv->x_final || !pooled_out) {
    set_last_error("pg_text_forward_train: null argument");
    return 1;
  }
  if (n <= 0) return 0;
  const pg_text_config& c = h->cfg;
  if (S < 1 || S > c.max_positions) {
    set_last_error("pg_text_forward_train: sequence length %d not in [1, %d] (max_position_embeddings)", S, c.max_positions);
    return 1;
  }
  if (n > 65535) { set_last_error("pg_text_forward_train: n %d > 65535 captions per call", n); return 1; }
  for (int l = 0; l < c.layers; ++l) {
    const pg_vit_saved_layer& s = sv->layers_host[l];
    if (!s.x0 || !s.xn1 || !s.qkv || !s.lse2 || !s.ao || !s.x1 || !s.xn2 || !s.u || !s.h) {
      set_last_error("pg_text_forward_train: layer %d has a null save buffer", l);
      return 1;
    }
  }
  const int sms = sm_count();
  if (sms < 0) return 1;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream_);
  const long rows = (long)n * S;
  const long long* ids = reinterpret_cast<const long long*>(input_ids);
  if (text_embed(ids, h->w.token_emb, h->w.pos_emb, sv->layers_host[0].x0, rows, S, c.hidden, c.vocab, sms, st)) return 1;
  if (encoder_layers_train(h->layers.data(), sv->layers_host, sv->x_final, c.layers, c.hidden, c.heads, c.intermediate,
                           c.ln_eps, n, S, attention_mask, 1, sms, st))
    return 1;
  return rows_layernorm_f32(sv->x_final, pooled_out, h->w.final_ln_g, h->w.final_ln_b, n, c.hidden, c.ln_eps, ids, S, sms, st);
}

static size_t text_bwd_carve(const pg_text* h, int n, int S, void* ws, BwdWs* w, float** part) {
  const pg_text_config& c = h->cfg;
  Carver cv(ws);
  *w = carve_encoder_bwd(n, S, c.hidden, c.heads, c.intermediate, 0, cv);
  *part = reinterpret_cast<float*>(cv.take((size_t)n * 2 * c.hidden * sizeof(float)));
  return cv.off;
}

size_t pg_text_backward_workspace_bytes(const pg_text* h, int32_t n, int32_t S) {
  if (!h || n <= 0 || S <= 0) return 0;
  BwdWs w;
  float* part;
  return text_bwd_carve(h, n, S, nullptr, &w, &part);
}

int pg_text_backward(pg_text* h, const pg_text_saved* sv, const int64_t* input_ids, const int64_t* attention_mask,
                     const float* d_pooled, int32_t n, int32_t S, const pg_text_grads* gr, void* workspace,
                     size_t workspace_bytes, void* stream_) {
  if (!h || !sv || !sv->layers_host || !sv->x_final || !input_ids || !d_pooled || !gr || !gr->layers_host || !workspace) {
    set_last_error("pg_text_backward: null argument");
    return 1;
  }
  if (n <= 0) return 0;
  const pg_text_config& c = h->cfg;
  if (S < 1 || S > c.max_positions) { set_last_error("pg_text_backward: sequence length %d not in [1, %d]", S, c.max_positions); return 1; }
  if (!gr->d_token_emb || !gr->d_pos_emb || !gr->d_final_ln_g || !gr->d_final_ln_b) {
    set_last_error("pg_text_backward: every text-tower gradient is required (the pretraining step trains all of them)");
    return 1;
  }
  if (check_layer_grads(gr->layers_host, c.layers, "pg_text_backward") < 0) return 1;
  for (int l = 0; l < c.layers; ++l)   // all set or all NULL per layer (checked above)
    if (!gr->layers_host[l].d_w_qkv) { set_last_error("pg_text_backward: encoder layer %d has no gradients", l); return 1; }
  const int sms = sm_count();
  if (sms < 0) return 1;
  if (reinterpret_cast<uintptr_t>(workspace) & 255) { set_last_error("pg_text_backward: workspace must be 256-byte aligned"); return 1; }
  BwdWs w;
  float* part;
  const size_t need = text_bwd_carve(h, n, S, workspace, &w, &part);
  if (workspace_bytes < need) { set_last_error("pg_text_backward: workspace %zu < required %zu", workspace_bytes, need); return 1; }
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream_);
  const long rows = (long)n * S;
  const int H = c.hidden;
  const long long* ids = reinterpret_cast<const long long*>(input_ids);

  // final_layer_norm backward on the pooled rows only: d(last layer output) is zero on every other row
  cudaError_t e = cudaMemsetAsync(w.g, 0, (size_t)rows * H * sizeof(float), st);
  if (e != cudaSuccess) { set_last_error("pg_text_backward: memset: %s", cudaGetErrorString(e)); return 1; }
  if (text_pool_ln_backward(sv->x_final, d_pooled, h->w.final_ln_g, ids, n, S, H, c.ln_eps, w.g, part, gr->d_final_ln_g,
                            gr->d_final_ln_b, st))
    return 1;
  if (encoder_layers_backward(h->layers.data(), sv->layers_host, gr->layers_host, c.layers, 0, H, c.heads, c.intermediate,
                              c.ln_eps, n, S, attention_mask, 1, nullptr, w, sms, st, "pg_text_backward"))
    return 1;
  // embeddings = token_embedding[ids] + position_embedding[:S]
  if (embed_backward(w.g, gr->d_pos_emb, nullptr, n, S, H, st)) return 1;
  return token_embedding_grad(ids, w.g, rows, H, c.vocab, gr->d_token_emb, st);
}

size_t pg_clip_loss_grad_workspace_bytes(int32_t n, int32_t P) {
  if (n <= 0 || P <= 0) return 0;
  return clip_loss_grad_workspace_bytes(n, P);
}

int pg_clip_loss_grad(const float* img, const float* txt, int32_t n, int32_t P, const float* logit_scale, double grad_scale,
                      void* workspace, size_t workspace_bytes, float* loss, float* d_img, float* d_txt, float* d_logit_scale,
                      float* logits_per_image, float* logits_per_text, void* stream) {
  if (!img || !txt || !logit_scale || !workspace || !loss || !d_img || !d_txt || !d_logit_scale) {
    set_last_error("pg_clip_loss_grad: null argument");
    return 1;
  }
  return clip_loss_grad(img, txt, n, P, logit_scale, grad_scale, workspace, workspace_bytes, loss, d_img, d_txt, d_logit_scale,
                        logits_per_image, logits_per_text, reinterpret_cast<cudaStream_t>(stream));
}

int pg_layernorm_f32(const float* x, float* y, const float* gamma, const float* beta, int64_t rows, int32_t hidden, float eps,
                     void* stream) {
  if (!x || !y || !gamma || !beta) { set_last_error("pg_layernorm_f32: null argument"); return 1; }
  if (rows <= 0) return 0;
  const int sms = sm_count();
  if (sms < 0) return 1;
  return rows_layernorm_f32(x, y, gamma, beta, rows, hidden, eps, nullptr, 0, sms, reinterpret_cast<cudaStream_t>(stream));
}

// ---------------------------------------------------------------------------------------------- building blocks
int pg_gemm_ex(const void* a, int32_t lda, const void* w, int32_t ldw, void* out, int32_t ldo, const float* bias,
               const float* resid, int32_t M, int32_t N, int32_t K, int32_t epilogue, int32_t operand_bf16, void* stream) {
  if (!a || !w || !out) { set_last_error("pg_gemm_ex: null argument"); return 1; }
  if (epilogue < 0 || epilogue > PG_EPI_F32_BIAS) { set_last_error("pg_gemm_ex: bad epilogue %d", epilogue); return 1; }
  const int sms = sm_count();
  if (sms < 0) return 1;
  GemmProblem p{};
  p.M = M; p.N = N; p.K = K; p.a = a; p.lda = lda; p.w = w; p.ldw = ldw; p.out = out; p.ldo = ldo; p.bias = bias;
  p.epi = epilogue; p.operand_bf16 = operand_bf16 ? 1 : 0; p.resid = resid;
  return gemm_f16(p, sms, reinterpret_cast<cudaStream_t>(stream));
}

int pg_gemm_tn(const void* a, int32_t lda, const void* w, int32_t ldw, float* out, int32_t ldo, int32_t M, int32_t N,
               int32_t K, int32_t accumulate, int32_t operand_bf16, void* stream) {
  if (!a || !w || !out) { set_last_error("pg_gemm_tn: null argument"); return 1; }
  const int sms = sm_count();
  if (sms < 0) return 1;
  GemmProblem p{};
  p.M = M; p.N = N; p.K = K; p.a = a; p.lda = lda; p.w = w; p.ldw = ldw; p.out = out; p.ldo = ldo; p.bias = nullptr;
  p.epi = accumulate ? EPI_F32_BIAS_RESID : EPI_F32_BIAS; p.operand_bf16 = operand_bf16 ? 1 : 0; p.mn_major = 1;
  return gemm_f16(p, sms, reinterpret_cast<cudaStream_t>(stream));
}

int pg_attention_f16_lse(const void* qkv, void* out, float* lse2, int32_t n_views, int32_t seq, int32_t heads, void* stream) {
  if (!qkv || !out || !lse2 || seq <= 0 || heads <= 0) { set_last_error("pg_attention_f16_lse: bad argument"); return 1; }
  return attention_f16(qkv, out, n_views, seq, heads, reinterpret_cast<cudaStream_t>(stream), lse2);
}

size_t pg_attention_backward_workspace_bytes(int32_t n_views, int32_t seq, int32_t heads) {
  if (n_views <= 0 || seq <= 0 || heads <= 0) return 0;
  const size_t rows = (size_t)n_views * seq, hidden = (size_t)heads * 64;
  Carver c(nullptr);
  c.take(rows * 3 * hidden * 2);   // qkv bf16
  c.take(rows * hidden * 2);       // dO bf16
  c.take((size_t)n_views * heads * seq * 4);
  return c.off;
}

int pg_attention_backward(const void* qkv, const void* out, const float* d_out, const float* lse2, void* dqkv_bf16,
                          int32_t n_views, int32_t seq, int32_t heads, void* workspace, size_t workspace_bytes,
                          void* stream_) {
  if (!qkv || !out || !d_out || !lse2 || !dqkv_bf16 || !workspace) { set_last_error("pg_attention_backward: null argument"); return 1; }
  if (n_views <= 0) return 0;
  if (workspace_bytes < pg_attention_backward_workspace_bytes(n_views, seq, heads) ||
      (reinterpret_cast<uintptr_t>(workspace) & 255)) {
    set_last_error("pg_attention_backward: workspace too small or not 256-byte aligned");
    return 1;
  }
  const int sms = sm_count();
  if (sms < 0) return 1;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream_);
  const size_t rows = (size_t)n_views * seq, hidden = (size_t)heads * 64;
  Carver c(workspace);
  void* qkv_bf = c.take(rows * 3 * hidden * 2);
  void* do_bf = c.take(rows * hidden * 2);
  float* delta = reinterpret_cast<float*>(c.take((size_t)n_views * heads * seq * 4));
  if (attention_delta(d_out, out, delta, do_bf, n_views, seq, heads, sms, st)) return 1;
  if (cast_to_bf16(qkv, SRC_F16, qkv_bf, (long)(rows * 3 * hidden), st)) return 1;
  return attention_backward(qkv, qkv_bf, do_bf, lse2, delta, dqkv_bf16, n_views, seq, heads, st);
}

int pg_attention_f16_masked_lse(const void* qkv, void* out, float* lse2, const int64_t* mask, int32_t causal, int32_t n_views,
                                int32_t seq, int32_t heads, void* stream) {
  if (!qkv || !out || !lse2 || seq <= 0 || heads <= 0) { set_last_error("pg_attention_f16_masked_lse: bad argument"); return 1; }
  return attention_f16_masked(qkv, out, reinterpret_cast<const long long*>(mask), causal, n_views, seq, heads,
                              reinterpret_cast<cudaStream_t>(stream), lse2);
}

int pg_attention_backward_masked(const void* qkv, const void* out, const float* d_out, const float* lse2, const int64_t* mask,
                                 int32_t causal, void* dqkv_bf16, int32_t n_views, int32_t seq, int32_t heads, void* workspace,
                                 size_t workspace_bytes, void* stream_) {
  if (!qkv || !out || !d_out || !lse2 || !dqkv_bf16 || !workspace) {
    set_last_error("pg_attention_backward_masked: null argument");
    return 1;
  }
  if (n_views <= 0) return 0;
  if (workspace_bytes < pg_attention_backward_workspace_bytes(n_views, seq, heads) ||
      (reinterpret_cast<uintptr_t>(workspace) & 255)) {
    set_last_error("pg_attention_backward_masked: workspace too small or not 256-byte aligned");
    return 1;
  }
  const int sms = sm_count();
  if (sms < 0) return 1;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream_);
  const size_t rows = (size_t)n_views * seq, hidden = (size_t)heads * 64;
  Carver c(workspace);
  void* qkv_bf = c.take(rows * 3 * hidden * 2);
  void* do_bf = c.take(rows * hidden * 2);
  float* delta = reinterpret_cast<float*>(c.take((size_t)n_views * heads * seq * 4));
  if (attention_delta(d_out, out, delta, do_bf, n_views, seq, heads, sms, st)) return 1;
  if (cast_to_bf16(qkv, SRC_F16, qkv_bf, (long)(rows * 3 * hidden), st)) return 1;
  return attention_backward_masked(qkv, qkv_bf, do_bf, lse2, delta, dqkv_bf16, reinterpret_cast<const long long*>(mask), causal,
                                   n_views, seq, heads, st);
}

int pg_layernorm_backward(const float* dy, const float* x, const float* gamma, float* dx, int32_t accumulate, float* dgamma,
                          float* dbeta, void* dx_bf16, int64_t rows, int32_t hidden, float eps, void* stream) {
  if (!dy || !x || !gamma || !dx) { set_last_error("pg_layernorm_backward: null argument"); return 1; }
  const int sms = sm_count();
  if (sms < 0) return 1;
  return layernorm_backward(dy, x, gamma, dx, accumulate, dgamma, dbeta, dx_bf16, rows, hidden, eps, sms,
                            reinterpret_cast<cudaStream_t>(stream));
}

int pg_dgelu_bf16(const float* dh, const void* u, void* du, int64_t n, void* stream) {
  if (!dh || !u || !du) { set_last_error("pg_dgelu_bf16: null argument"); return 1; }
  return dgelu_bf16(dh, u, du, n, reinterpret_cast<cudaStream_t>(stream));
}

int pg_transpose_to_bf16(const void* src, int32_t src_type, int64_t lds, void* out, int64_t ldo, int64_t rows, int32_t cols,
                         void* stream) {
  if (!src || !out) { set_last_error("pg_transpose_to_bf16: null argument"); return 1; }
  return transpose_to_bf16(src, src_type, lds, out, ldo, rows, cols, 0, 0, 0, reinterpret_cast<cudaStream_t>(stream));
}

int pg_column_sum_accumulate(const void* x, int32_t src_type, int64_t ldx, float* out, int64_t rows, int32_t cols,
                             void* stream) {
  if (!x || !out) { set_last_error("pg_column_sum_accumulate: null argument"); return 1; }
  return column_sum_accumulate(x, src_type, ldx, out, rows, cols, reinterpret_cast<cudaStream_t>(stream));
}

int pg_token_mean_backward(const float* d_emb, float* g, int32_t n_views, int32_t tokens, int32_t hidden, void* stream) {
  if (!d_emb || !g) { set_last_error("pg_token_mean_backward: null argument"); return 1; }
  return token_mean_backward(d_emb, g, n_views, tokens, hidden, reinterpret_cast<cudaStream_t>(stream));
}

int pg_embed_backward(const float* d_e, float* dpos, float* dcls, int32_t n_views, int32_t tokens, int32_t hidden,
                      void* stream) {
  if (!d_e || !dpos) { set_last_error("pg_embed_backward: null argument"); return 1; }
  return embed_backward(d_e, dpos, dcls, n_views, tokens, hidden, reinterpret_cast<cudaStream_t>(stream));
}

int pg_text_pool_ln_backward(const float* x, const float* d_pooled, const float* gamma, const int64_t* ids, int32_t n,
                             int32_t S, int32_t hidden, float eps, float* g, float* part, float* dgamma, float* dbeta,
                             void* stream) {
  if (!x || !d_pooled || !gamma || !ids || !g || !part || !dgamma || !dbeta) {
    set_last_error("pg_text_pool_ln_backward: null argument");
    return 1;
  }
  return text_pool_ln_backward(x, d_pooled, gamma, reinterpret_cast<const long long*>(ids), n, S, hidden, eps, g, part, dgamma,
                               dbeta, reinterpret_cast<cudaStream_t>(stream));
}

int pg_token_embedding_grad(const int64_t* ids, const float* dx, int64_t rows, int32_t hidden, int32_t vocab, float* dtok,
                            void* stream) {
  if (!ids || !dx || !dtok) { set_last_error("pg_token_embedding_grad: null argument"); return 1; }
  return token_embedding_grad(reinterpret_cast<const long long*>(ids), dx, rows, hidden, vocab, dtok,
                              reinterpret_cast<cudaStream_t>(stream));
}

}  // extern "C"
