// C ABI (include/pigeon_b200.h) over the kernels in this directory.  Host-side orchestration only:
// argument checks, workspace carving and the launch sequence of the vision tower.
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

#include <stdlib.h>

#include <atomic>
#include <new>
#include <vector>

#include "../../include/pigeon_b200.h"
#include "attention.h"
#include "gemm.h"
#include "head.h"
#include "preprocess.h"
#include "pretrain.h"
#include "refiner.h"
#include "tma_host.h"
#include "train.h"
#include "vit_handle.h"
#include "vit_misc.h"

using namespace pg;

namespace pg {

static int g_sm_count = 0;
int sm_count() {
  if (g_sm_count <= 0) {
    int dev = 0, n = 0;
    if (cudaGetDevice(&dev) != cudaSuccess ||
        cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) {
      set_last_error("no usable CUDA device (cudaDeviceGetAttribute failed)");
      return -1;
    }
    g_sm_count = n;
  }
  return g_sm_count;
}

// Pre-LN CLIPEncoderLayer stack with the LayerNorm kernels (HF modeling_clip.py 4.23.1 CLIPEncoderLayer.forward):
//   x += out_proj(attn(layer_norm1(x)));  x += fc2(quick_gelu(fc1(layer_norm2(x))))
// on x f32 [n_seq * seq, hidden]; xn / u are the fp16 scratch of vit_carve.  The vision tower passes mask = NULL and
// causal = 0 (plain attention_f16); the text tower its attention_mask and causal = 1.
int encoder_layers(const pg_vit_layer* layers, int n_layers, int hidden, int heads, int intermediate, float eps, float* x,
                   void* xn, void* u, int n_seq, int seq, const int64_t* mask, int causal, int sms, cudaStream_t stream) {
  const long rows = (long)n_seq * seq;
  for (int l = 0; l < n_layers; ++l) {
    const pg_vit_layer& L = layers[l];
    if (layernorm_f16(x, xn, L.ln1_g, L.ln1_b, rows, hidden, eps, sms, stream)) return 1;
    GemmProblem p{};
    p.M = (int)rows; p.N = 3 * hidden; p.K = hidden;
    p.a = xn; p.lda = hidden; p.w = L.w_qkv; p.ldw = hidden;
    p.out = u; p.ldo = 3 * hidden; p.bias = L.b_qkv; p.epi = EPI_F16_BIAS;
    if (gemm_f16(p, sms, stream)) return 1;
    if (attention_f16_masked(u, xn, reinterpret_cast<const long long*>(mask), causal, n_seq, seq, heads, stream)) return 1;
    p = GemmProblem{};
    p.M = (int)rows; p.N = hidden; p.K = hidden;
    p.a = xn; p.lda = hidden; p.w = L.w_o; p.ldw = hidden;
    p.out = x; p.ldo = hidden; p.bias = L.b_o; p.epi = EPI_F32_BIAS_RESID;
    if (gemm_f16(p, sms, stream)) return 1;
    if (layernorm_f16(x, xn, L.ln2_g, L.ln2_b, rows, hidden, eps, sms, stream)) return 1;
    p = GemmProblem{};
    p.M = (int)rows; p.N = intermediate; p.K = hidden;
    p.a = xn; p.lda = hidden; p.w = L.w_fc1; p.ldw = hidden;
    p.out = u; p.ldo = intermediate; p.bias = L.b_fc1; p.epi = EPI_F16_BIAS_QGELU;
    if (gemm_f16(p, sms, stream)) return 1;
    p = GemmProblem{};
    p.M = (int)rows; p.N = hidden; p.K = intermediate;
    p.a = u; p.lda = intermediate; p.w = L.w_fc2; p.ldw = intermediate;
    p.out = x; p.ldo = hidden; p.bias = L.b_fc2; p.epi = EPI_F32_BIAS_RESID;
    if (gemm_f16(p, sms, stream)) return 1;
  }
  return 0;
}

}  // namespace pg

extern "C" {

int pg_abi_version(void) { return PG_ABI_VERSION; }
const char* pg_last_error(void) { return last_error(); }
int pg_device_sm_count(void) { return sm_count(); }

// ---------------------------------------------------------------------------------------------- ViT
int pg_vit_create(const pg_vit_config* cfg, const pg_vit_weights* w, pg_vit** out) {
  if (!cfg || !w || !out) { set_last_error("pg_vit_create: null argument"); return 1; }
  if (cfg->hidden % 256 || cfg->intermediate % 256) { set_last_error("pg_vit_create: hidden/intermediate must be multiples of 256"); return 1; }
  if (cfg->heads <= 0 || cfg->hidden != cfg->heads * 64) { set_last_error("pg_vit_create: head_dim must be 64"); return 1; }
  if (cfg->patch_size <= 0 || cfg->image_size % cfg->patch_size) { set_last_error("pg_vit_create: image_size %% patch_size != 0"); return 1; }
  if (cfg->patch_k_pad % 64 || cfg->patch_k_pad < 3 * cfg->patch_size * cfg->patch_size) { set_last_error("pg_vit_create: bad patch_k_pad"); return 1; }
  if (cfg->layers <= 0 || !w->layers_host) { set_last_error("pg_vit_create: no layers"); return 1; }
  pg_vit* h = new (std::nothrow) pg_vit();
  if (!h) { set_last_error("pg_vit_create: out of host memory"); return 1; }
  h->cfg = *cfg;
  h->w = *w;
  h->layers.assign(w->layers_host, w->layers_host + cfg->layers);
  h->w.layers_host = h->layers.data();
  h->grid_patches = cfg->image_size / cfg->patch_size;
  h->tokens = h->grid_patches * h->grid_patches + 1;
  *out = h;
  return 0;
}

void pg_vit_destroy(pg_vit* h) { delete h; }

static bool vit_ln_folded(const pg_vit* h) {
  for (const pg_vit_layer& L : h->layers)
    if (!L.w_qkv_ln || !L.b_qkv_ln || !L.cs_qkv || !L.w_fc1_ln || !L.b_fc1_ln || !L.cs_fc1) return false;
  return true;
}

static size_t vit_carve(const pg_vit* h, int n_views, void* ws, float** x, void** xn, void** u, void** x16 = nullptr,
                        float** stats = nullptr) {
  const size_t rows = (size_t)n_views * h->tokens;
  const int wide = h->cfg.intermediate > 3 * h->cfg.hidden ? h->cfg.intermediate : 3 * h->cfg.hidden;
  size_t u_elems = rows * (size_t)wide;
  const size_t im2col_elems = (size_t)n_views * h->grid_patches * h->grid_patches * h->cfg.patch_k_pad;
  if (im2col_elems > u_elems) u_elems = im2col_elems;
  Carver c(ws);
  *x = reinterpret_cast<float*>(c.take(rows * h->cfg.hidden * sizeof(float)));  // residual stream, fp32
  *xn = c.take(rows * h->cfg.hidden * 2);  // LayerNorm output / attention output (fp16), time-shared
  *u = c.take(u_elems * 2);                // im2col | qkv | fc1 activations (fp16), time-shared
  if (vit_ln_folded(h)) {                  // LayerNorm folded into the GEMMs: raw fp16 residual row + its moments
    void* p16 = c.take(rows * h->cfg.hidden * 2);
    float* st = reinterpret_cast<float*>(c.take(rows * (h->cfg.hidden / 128) * 2 * sizeof(float)));
    if (x16) *x16 = p16;
    if (stats) *stats = st;
  }
  return c.off;
}

size_t pg_vit_workspace_bytes(const pg_vit* h, int32_t n_views) {
  if (!h || n_views <= 0) return 0;
  float* x; void* xn; void* u;
  return vit_carve(h, n_views, nullptr, &x, &xn, &u);
}

static int vit_forward(pg_vit* h, const void* pixels, int32_t pixels_f16, int32_t n_views, void* workspace,
                       size_t workspace_bytes, float* emb_out, float* hidden_out, float* cls_out, void* stream_) {
  if (!h || !pixels || !workspace || !emb_out) { set_last_error("pg_vit_forward: null argument"); return 1; }
  if (n_views <= 0) return 0;
  const int sms = sm_count();
  if (sms < 0) return 1;
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  float* x; void* xn; void* u; void* x16 = nullptr; float* stats = nullptr;
  const size_t need = vit_carve(h, n_views, workspace, &x, &xn, &u, &x16, &stats);
  const bool folded = vit_ln_folded(h);
  if (workspace_bytes < need) { set_last_error("pg_vit_forward: workspace %zu < required %zu", workspace_bytes, need); return 1; }
  if (reinterpret_cast<uintptr_t>(workspace) & 255) { set_last_error("pg_vit_forward: workspace must be 256-byte aligned"); return 1; }
  const pg_vit_config& c = h->cfg;
  const long rows = (long)n_views * h->tokens;
  const int np = h->grid_patches * h->grid_patches;

  // patch embedding: im2col -> GEMM whose epilogue scatters row (view, patch) to token (view, 1 + patch)
  if (im2col(pixels, pixels_f16, u, n_views, c.image_size, c.patch_size, c.patch_k_pad, sms, stream)) return 1;
  {
    GemmProblem p{};
    p.M = n_views * np; p.N = c.hidden; p.K = c.patch_k_pad;
    p.a = u; p.lda = c.patch_k_pad; p.w = h->w.patch_w; p.ldw = c.patch_k_pad;
    p.out = x; p.ldo = c.hidden; p.bias = nullptr; p.epi = EPI_F32_ROWMAP;
    p.rowmap_div = np; p.rowmap_mul = h->tokens; p.rowmap_add = 1;
    if (gemm_f16(p, sms, stream)) return 1;
  }
  if (embed_preln(x, h->w.class_emb, h->w.pos_emb, h->w.pre_ln_g, h->w.pre_ln_b, rows, h->tokens, c.hidden, c.ln_eps,
                  sms, stream, nullptr, folded ? x16 : nullptr, folded ? stats : nullptr))
    return 1;

  // LayerNorm folded into the GEMMs either side of it (5 launches per layer, no normalised copy in HBM): the residual
  // epilogues leave the raw fp16 row and its (sum, sum of squares) behind, the consumers apply rstd * (acc - mu * colsum).
  for (int l = 0; folded && l < c.layers; ++l) {
    const pg_vit_layer& L = h->layers[l];
    GemmProblem p{};
    p.M = (int)rows; p.N = 3 * c.hidden; p.K = c.hidden;
    p.a = x16; p.lda = c.hidden; p.w = L.w_qkv_ln; p.ldw = c.hidden;
    p.out = u; p.ldo = 3 * c.hidden; p.bias = L.b_qkv_ln; p.epi = EPI_F16_LN_BIAS;
    p.stats = stats; p.colsum = L.cs_qkv; p.ln_eps = c.ln_eps;
    if (gemm_f16(p, sms, stream)) return 1;
    if (attention_f16(u, xn, n_views, h->tokens, c.heads, stream)) return 1;
    p = GemmProblem{};
    p.M = (int)rows; p.N = c.hidden; p.K = c.hidden;
    p.a = xn; p.lda = c.hidden; p.w = L.w_o; p.ldw = c.hidden;
    p.out = x; p.ldo = c.hidden; p.bias = L.b_o; p.epi = EPI_F32_BIAS_RESID_STATS;
    p.aux = x16; p.stats = stats;
    if (gemm_f16(p, sms, stream)) return 1;
    p = GemmProblem{};
    p.M = (int)rows; p.N = c.intermediate; p.K = c.hidden;
    p.a = x16; p.lda = c.hidden; p.w = L.w_fc1_ln; p.ldw = c.hidden;
    p.out = u; p.ldo = c.intermediate; p.bias = L.b_fc1_ln; p.epi = EPI_F16_LN_BIAS_QGELU;
    p.stats = stats; p.colsum = L.cs_fc1; p.ln_eps = c.ln_eps;
    if (gemm_f16(p, sms, stream)) return 1;
    p = GemmProblem{};
    p.M = (int)rows; p.N = c.hidden; p.K = c.intermediate;
    p.a = u; p.lda = c.intermediate; p.w = L.w_fc2; p.ldw = c.intermediate;
    p.out = x; p.ldo = c.hidden; p.bias = L.b_fc2;
    if (l + 1 < c.layers) { p.epi = EPI_F32_BIAS_RESID_STATS; p.aux = x16; p.stats = stats; }
    else p.epi = EPI_F32_BIAS_RESID;
    if (gemm_f16(p, sms, stream)) return 1;
  }

  if (!folded && encoder_layers(h->layers.data(), c.layers, c.hidden, c.heads, c.intermediate, c.ln_eps, x, xn, u, n_views,
                                h->tokens, nullptr, 0, sms, stream))
    return 1;
  if (token_mean(x, emb_out, n_views, h->tokens, c.hidden, stream)) return 1;
  if (hidden_out) {
    cudaError_t e = cudaMemcpyAsync(hidden_out, x, (size_t)rows * c.hidden * sizeof(float), cudaMemcpyDeviceToDevice, stream);
    if (e != cudaSuccess) { set_last_error("pg_vit_forward: hidden copy: %s", cudaGetErrorString(e)); return 1; }
  }
  if (cls_out) {   // row 0 of every view: one strided copy out of the residual stream
    const size_t row_bytes = (size_t)c.hidden * sizeof(float);
    cudaError_t e = cudaMemcpy2DAsync(cls_out, row_bytes, x, (size_t)h->tokens * row_bytes, row_bytes, n_views,
                                      cudaMemcpyDeviceToDevice, stream);
    if (e != cudaSuccess) { set_last_error("pg_vit_forward_cls: CLS copy: %s", cudaGetErrorString(e)); return 1; }
  }
  return 0;
}

int pg_vit_forward(pg_vit* h, const void* pixels, int32_t pixels_f16, int32_t n_views, void* workspace,
                   size_t workspace_bytes, float* emb_out, float* hidden_out, void* stream) {
  return vit_forward(h, pixels, pixels_f16, n_views, workspace, workspace_bytes, emb_out, hidden_out, nullptr, stream);
}

int pg_vit_forward_cls(pg_vit* h, const void* pixels, int32_t pixels_f16, int32_t n_views, void* workspace,
                       size_t workspace_bytes, float* emb_out, float* hidden_out, float* cls_out, void* stream) {
  if (!cls_out) { set_last_error("pg_vit_forward_cls: null cls_out"); return 1; }
  return vit_forward(h, pixels, pixels_f16, n_views, workspace, workspace_bytes, emb_out, hidden_out, cls_out, stream);
}

// ---------------------------------------------------------------------------------------------- head
int pg_head_pack_weight(const float* w, void* w3_out, int32_t C, int32_t D, void* stream) {
  if (!w || !w3_out || C <= 0 || D <= 0) { set_last_error("pg_head_pack_weight: bad argument"); return 1; }
  return weight_split(w, w3_out, C, D, reinterpret_cast<cudaStream_t>(stream));
}

size_t pg_head_workspace_bytes(int32_t B, int32_t D) {
  if (B <= 0 || D <= 0) return 0;
  return align_up((size_t)B * 3 * D * 2, 1024);
}

// Process-wide switch like pg_refiner_set_schedule; PG_HEAD_FUSED=1 only sets the initial value, once.
static std::atomic<int> g_head_fused{-1};
static bool head_fused_on() {
  int v = g_head_fused.load(std::memory_order_relaxed);
  if (v < 0) {
    const char* e = getenv("PG_HEAD_FUSED");
    v = (e && e[0] == '1') ? 1 : 0;
    g_head_fused.store(v, std::memory_order_relaxed);
  }
  return v == 1;
}
int pg_head_set_fused(int32_t on) {
  g_head_fused.store(on ? 1 : 0, std::memory_order_relaxed);
  return 0;
}

int pg_head_forward(const float* emb, int32_t B, int32_t V, int32_t D, const void* w3, const float* bias,
                    const double* centroids, int32_t C, int32_t k, void* workspace, size_t workspace_bytes,
                    float* pooled, float* logits, float* probs, int64_t* pred_cell, double* pred_lnglat,
                    float* topk_val, int64_t* topk_idx, void* stream_) {
  if (B < 0) { set_last_error("pg_head_forward: negative batch B=%d", B); return 1; }
  // An empty batch has nothing to read or write, and zero-byte buffers may well be NULL (torch.empty(0).data_ptr() is 0),
  // so it returns before the pointer checks (tests/test_gpu_head.py::test_head_empty_batch).
  if (B == 0) return 0;
  if (!emb || !w3 || !centroids || !workspace || !pooled || !logits || !probs || !pred_cell || !pred_lnglat ||
      !topk_val || !topk_idx) { set_last_error("pg_head_forward: null argument"); return 1; }
  if (V <= 0 || D % 8 || C <= 0 || k <= 0 || k > C) { set_last_error("pg_head_forward: bad shape B=%d V=%d D=%d C=%d k=%d", B, V, D, C, k); return 1; }
  if (workspace_bytes < pg_head_workspace_bytes(B, D)) { set_last_error("pg_head_forward: workspace too small"); return 1; }
  const int sms = sm_count();
  if (sms < 0) return 1;
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  // pg_head_set_fused(1): one kernel (view mean + split -> wgmma GEMM -> bias -> softmax / arg-max / top-k) whenever the
  // shape allows; the default is the three-kernel sequence, which is faster at the batch sizes of this path (DESIGN.md 5.4)
  if (head_fused_on() && head_fused_supported(B, V, D, C, k) && (reinterpret_cast<uintptr_t>(emb) & 15) == 0)
    return head_fused_forward(emb, B, V, D, w3, bias, centroids, C, k, workspace, pooled, logits, probs,
                              reinterpret_cast<long long*>(pred_cell), pred_lnglat, topk_val,
                              reinterpret_cast<long long*>(topk_idx), stream);
  if (view_mean_split(emb, pooled, workspace, B, V, D, stream)) return 1;
  GemmProblem p{};
  p.M = B; p.N = C; p.K = 3 * D;
  p.a = workspace; p.lda = 3 * D; p.w = w3; p.ldw = 3 * D;
  p.out = logits; p.ldo = C; p.bias = bias; p.epi = EPI_F32_BIAS;
  if (gemm_f16(p, sms, stream)) return 1;
  return softmax_topk(logits, probs, reinterpret_cast<long long*>(pred_cell), pred_lnglat, topk_val,
                      reinterpret_cast<long long*>(topk_idx), centroids, B, C, k, stream);
}

int pg_head_loss(const float* logits, int32_t B, int32_t C, int32_t mode, const int64_t* labels_idx, const float* soft,
                 const double* labels_lnglat, const double* centroids, double smoothing_km, double* per_sample,
                 double* loss_out, void* stream) {
  if (!logits || !per_sample || !loss_out || B <= 0 || C <= 0) { set_last_error("pg_head_loss: bad argument"); return 1; }
  return ce_loss(logits, B, C, mode, reinterpret_cast<const long long*>(labels_idx), soft, labels_lnglat, centroids,
                 smoothing_km, per_sample, loss_out, nullptr, 1.0, reinterpret_cast<cudaStream_t>(stream));
}

size_t pg_preprocess_workspace_bytes(const pg_image* images, int32_t n, int32_t size) {
  return preprocess_workspace_bytes(images, nullptr, n, size);
}

int pg_preprocess_clip(const pg_image* images, int32_t n, int32_t size, const float* mean, const float* stdv,
                       void* workspace, size_t workspace_bytes, void* out, int32_t out_f16, void* stream) {
  return preprocess_clip(images, nullptr, n, size, mean, stdv, workspace, workspace_bytes, out, out_f16,
                         reinterpret_cast<cudaStream_t>(stream));
}

size_t pg_preprocess_window_workspace_bytes(const pg_image* images, const pg_window* windows, int32_t n, int32_t size) {
  if (!windows) { set_last_error("pg_preprocess_window_workspace_bytes: windows is NULL"); return 0; }
  return preprocess_workspace_bytes(images, windows, n, size);
}

int pg_preprocess_clip_window(const pg_image* images, const pg_window* windows, int32_t n, int32_t size,
                              const float* mean, const float* stdv, void* workspace, size_t workspace_bytes, void* out,
                              int32_t out_f16, void* stream) {
  if (!windows) { set_last_error("pg_preprocess_clip_window: windows is NULL"); return 1; }
  return preprocess_clip(images, windows, n, size, mean, stdv, workspace, workspace_bytes, out, out_f16,
                         reinterpret_cast<cudaStream_t>(stream));
}

int pg_head_loss_grad(const float* logits, int32_t B, int32_t C, int32_t mode, const int64_t* labels_idx,
                      const float* soft, const double* labels_lnglat, const double* centroids, double smoothing_km,
                      double grad_scale, double* per_sample, double* loss_out, float* dlogits, void* stream) {
  if (!logits || !per_sample || !loss_out || !dlogits || B <= 0 || C <= 0) {
    set_last_error("pg_head_loss_grad: bad argument");
    return 1;
  }
  return ce_loss(logits, B, C, mode, reinterpret_cast<const long long*>(labels_idx), soft, labels_lnglat, centroids,
                 smoothing_km, per_sample, loss_out, dlogits, grad_scale, reinterpret_cast<cudaStream_t>(stream));
}

int pg_head_backward(const float* dlogits, const float* pooled, const float* w, int32_t B, int32_t C, int32_t D,
                     int32_t accumulate, float* dw, float* db, float* dpooled, void* stream) {
  if (!dlogits || B <= 0 || C <= 0 || D <= 0) { set_last_error("pg_head_backward: bad argument"); return 1; }
  if ((dw && !pooled) || (dpooled && !w)) { set_last_error("pg_head_backward: missing operand"); return 1; }
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  // dW[c, d] = sum_b dlogits[b, c] * pooled[b, d];  db[c] = sum_b dlogits[b, c];  dpooled = dlogits . W
  if (dw && sgemm_f32(true, dlogits, pooled, dw, C, D, B, accumulate ? 1.f : 0.f, st)) return 1;
  if (db && column_sum_f32(dlogits, db, B, C, accumulate ? 1.f : 0.f, st)) return 1;
  if (dpooled && sgemm_f32(false, dlogits, w, dpooled, B, D, C, 0.f, st)) return 1;
  return 0;
}

int pg_adamw_step(float* param, const float* grad, float* exp_avg, float* exp_avg_sq, int64_t n, double lr,
                  double beta1, double beta2, double eps, double weight_decay, int64_t step, double grad_scale,
                  void* stream) {
  if (!param || !grad || !exp_avg || !exp_avg_sq || n <= 0 || step < 1) {
    set_last_error("pg_adamw_step: bad argument");
    return 1;
  }
  return adamw_step(param, grad, exp_avg, exp_avg_sq, n, lr, beta1, beta2, eps, weight_decay, step, grad_scale,
                    reinterpret_cast<cudaStream_t>(stream));
}

// ---------------------------------------------------------------------------------------------- CLIP pretraining step
size_t pg_grad_norm_clip_workspace_bytes(int64_t n) { return grad_norm_clip_workspace_bytes(n); }

int pg_grad_norm_clip(const float* grad, int64_t n, double grad_scale, double max_norm, float* total_norm, float* clip_coef,
                      void* workspace, size_t workspace_bytes, void* stream) {
  if (!grad || n <= 0 || !total_norm || !clip_coef || !workspace || !(max_norm > 0.0)) {
    set_last_error("pg_grad_norm_clip: bad argument");
    return 1;
  }
  return grad_norm_clip(grad, n, grad_scale, max_norm, total_norm, clip_coef, workspace, workspace_bytes,
                        reinterpret_cast<cudaStream_t>(stream));
}

int pg_adamw_hf_step(float* param, const float* grad, float* exp_avg, float* exp_avg_sq, int64_t n, double lr,
                     double beta1, double beta2, double eps, double weight_decay, int64_t step, double grad_scale,
                     const float* clip_coef, void* stream) {
  if (!param || !grad || !exp_avg || !exp_avg_sq || n <= 0 || step < 1) {
    set_last_error("pg_adamw_hf_step: bad argument");
    return 1;
  }
  return adamw_hf_step(param, grad, exp_avg, exp_avg_sq, n, lr, beta1, beta2, eps, weight_decay, step, grad_scale,
                       clip_coef, reinterpret_cast<cudaStream_t>(stream));
}

// ---------------------------------------------------------------------------------------------- refiner
size_t pg_refiner_workspace_bytes(int64_t B, int32_t topk, int32_t D, int32_t num_cells) {
  if (B <= 0 || topk <= 0 || D <= 0 || num_cells <= 0) return 0;
  Carver c(nullptr);
  c.take((size_t)B * D * 4);         // pooled queries
  c.take((size_t)B * topk * 4);      // best_logit
  c.take((size_t)B * topk * 2 * 4);  // best_lnglat
  c.take((size_t)B * topk * 4);      // best_proto
  c.take(refiner_sort_workspace_bytes(num_cells, (long)B * topk));  // counting sort of the pairs by geocell
  return c.off;
}

static RefinerBank to_bank(const pg_refiner_bank* bank) {
  RefinerBank rb;
  rb.num_cells = bank->num_cells; rb.dim = bank->dim;
  rb.cell_off = reinterpret_cast<const long long*>(bank->cell_off);
  rb.proto_emb = bank->proto_emb; rb.proto_lnglat = bank->proto_lnglat; rb.proto_count = bank->proto_count;
  rb.member_off = reinterpret_cast<const long long*>(bank->member_off);
  rb.member_idx = reinterpret_cast<const long long*>(bank->member_idx);
  rb.data_emb = bank->data_emb; rb.data_lnglat = bank->data_lnglat;
  rb.proto_sqnorm = bank->proto_sqnorm;
  return rb;
}

// Which scan the schedule and the call shape select: 1 query-major, 2 cell-major (v3), 3 tile scan (v4), 4 slab scan (v5).
static int pick_scan(int sched, int64_t B, int32_t topk, const pg_refiner_bank* bank) {
  const bool slab_ok = bank->proto_sqnorm && bank->num_protos > 0;
  if (sched == 1 || sched == 2) return sched;
  if (sched == 3) return bank->proto_sqnorm ? 3 : 2;
  if (sched == 4) return slab_ok ? 4 : 2;
  if ((long)B * topk < 2L * bank->num_cells) return 1;   // small batches: the sort would dominate
  // a slab is 64 prototypes of ONE geocell and a CTA tile 512: only banks with large geocells fill them
  const long cells = bank->live_cells > 0 ? bank->live_cells : bank->num_cells;
  if (slab_ok && bank->num_protos >= 256L * cells) return 4;
  return 2;
}

// Scan schedule of pg_refiner_forward: 0 = automatic (cell-major when geocells are shared by >= 2 pairs on average),
// 1 = query-major, 2 = cell-major (v3), 3 = tile scan (v4), 4 = slab scan (v5; what automatic picks for banks with large
// geocells).  Process-wide A/B switch (pg_refiner_set_schedule); the environment variable
// PG_REFINER_QUERY_MAJOR=1 only sets the initial value, once.
static std::atomic<int> g_refiner_schedule{-1};
static int refiner_schedule() {
  int v = g_refiner_schedule.load(std::memory_order_relaxed);
  if (v < 0) {
    const char* e = getenv("PG_REFINER_QUERY_MAJOR");
    v = (e && e[0] == '1') ? 1 : 0;
    g_refiner_schedule.store(v, std::memory_order_relaxed);
  }
  return v;
}

int pg_refiner_set_schedule(int32_t mode) {
  if (mode < 0 || mode > 4) { set_last_error("pg_refiner_set_schedule: mode %d not in {0, 1, 2, 3, 4}", mode); return 1; }
  g_refiner_schedule.store(mode, std::memory_order_relaxed);
  return 0;
}

int pg_refiner_forward(const pg_refiner_bank* bank, const float* emb, int64_t B, int32_t V, const double* init_lnglat,
                       const int64_t* cand_idx, const float* cand_prob, int32_t cand_stride, int32_t topk,
                       float temperature, double max_refinement_km, void* workspace, size_t workspace_bytes,
                       float* out_lnglat, int64_t* out_cell, float* best_logit, float* best_lnglat,
                       int32_t* best_proto, int32_t* choice, void* stream_) {
  if (!bank || !emb || !init_lnglat || !cand_idx || !cand_prob || !workspace || !out_lnglat || !out_cell) {
    set_last_error("pg_refiner_forward: null argument"); return 1;
  }
  if (B <= 0) return 0;
  // mirrors the reference assert at models/proto_refiner.py:135-137
  if (topk <= 0 || topk > cand_stride) { set_last_error("pg_refiner_forward: \"topk\" (%d) must be <= number of candidates (%d)", topk, cand_stride); return 1; }
  if (V <= 0 || bank->dim % 128 || bank->dim > 1024) { set_last_error("pg_refiner_forward: bad V=%d / dim=%d", V, bank->dim); return 1; }
  if (workspace_bytes < pg_refiner_workspace_bytes(B, topk, bank->dim, bank->num_cells)) { set_last_error("pg_refiner_forward: workspace too small"); return 1; }
  const int sms = sm_count();
  if (sms < 0) return 1;
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  Carver c(workspace);
  float* q = reinterpret_cast<float*>(c.take((size_t)B * bank->dim * 4));
  float* bl = reinterpret_cast<float*>(c.take((size_t)B * topk * 4));
  float* bll = reinterpret_cast<float*>(c.take((size_t)B * topk * 2 * 4));
  int* bp = reinterpret_cast<int*>(c.take((size_t)B * topk * 4));
  void* sort_ws = c.take(refiner_sort_workspace_bytes(bank->num_cells, (long)B * topk));
  if (best_logit) bl = best_logit;
  if (best_lnglat) bll = best_lnglat;
  if (best_proto) bp = best_proto;
  const RefinerBank rb = to_bank(bank);
  if (refiner_pool(emb, q, B, V, bank->dim, stream)) return 1;
  // cell-major (each touched prototype segment read once) as soon as cells are shared by several pairs on average;
  // the query-major kernel (one warp per pair) for small batches where the sort would dominate
  const int scan = pick_scan(refiner_schedule(), B, topk, bank);
  const long long* cand = reinterpret_cast<const long long*>(cand_idx);
  if (scan == 4) {
    if (refiner_scan_slabs(rb, bank->num_protos, q, cand, cand_stride, B, topk, sort_ws, bl, bll, bp, sms, stream)) return 1;
  } else if (scan == 3) {
    if (refiner_scan_tiles(rb, q, cand, cand_stride, B, topk, sort_ws, bl, bll, bp, sms, stream)) return 1;
  } else if (scan == 2) {
    if (refiner_scan_cell_major(rb, q, cand, cand_stride, B, topk, sort_ws, bl, bll, bp, sms, stream)) return 1;
  } else {
    if (refiner_scan(rb, q, cand, cand_stride, B, topk, bl, bll, bp, sms, stream)) return 1;
  }
  return refiner_finalize(bl, bll, reinterpret_cast<const long long*>(cand_idx), cand_prob, cand_stride, init_lnglat, B,
                          topk, temperature, max_refinement_km, out_lnglat, reinterpret_cast<long long*>(out_cell),
                          choice, stream);
}

// Cell-sharded retrieval (SURVEY.md 8e-ii): a rank whose bank holds only some geocells (the others empty) scans all queries
// against ITS cells; pairs whose geocell it does not hold come back as "empty cell" (-100000).  After the per-pair partials
// of all ranks are merged by owner, pg_refiner_finalize runs the temperature softmax / gate / arg-max on the merged values.
int pg_refiner_scan(const pg_refiner_bank* bank, const float* emb, int64_t B, int32_t V, const int64_t* cand_idx,
                    int32_t cand_stride, int32_t topk, void* workspace, size_t workspace_bytes, float* best_logit,
                    float* best_lnglat, int32_t* best_proto, void* stream_) {
  if (!bank || !emb || !cand_idx || !workspace || !best_logit || !best_lnglat || !best_proto) {
    set_last_error("pg_refiner_scan: null argument"); return 1;
  }
  if (B <= 0) return 0;
  if (topk <= 0 || topk > cand_stride) { set_last_error("pg_refiner_scan: \"topk\" (%d) must be <= number of candidates (%d)", topk, cand_stride); return 1; }
  if (V <= 0 || bank->dim % 128 || bank->dim > 1024) { set_last_error("pg_refiner_scan: bad V=%d / dim=%d", V, bank->dim); return 1; }
  if (workspace_bytes < pg_refiner_workspace_bytes(B, topk, bank->dim, bank->num_cells)) { set_last_error("pg_refiner_scan: workspace too small"); return 1; }
  const int sms = sm_count();
  if (sms < 0) return 1;
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  Carver c(workspace);
  float* q = reinterpret_cast<float*>(c.take((size_t)B * bank->dim * 4));
  c.take((size_t)B * topk * 4);
  c.take((size_t)B * topk * 2 * 4);
  c.take((size_t)B * topk * 4);
  void* sort_ws = c.take(refiner_sort_workspace_bytes(bank->num_cells, (long)B * topk));
  const RefinerBank rb = to_bank(bank);
  if (refiner_pool(emb, q, B, V, bank->dim, stream)) return 1;
  const int scan = pick_scan(refiner_schedule(), B, topk, bank);
  const long long* cand = reinterpret_cast<const long long*>(cand_idx);
  if (scan == 4)
    return refiner_scan_slabs(rb, bank->num_protos, q, cand, cand_stride, B, topk, sort_ws, best_logit, best_lnglat,
                              best_proto, sms, stream);
  if (scan == 3)
    return refiner_scan_tiles(rb, q, cand, cand_stride, B, topk, sort_ws, best_logit, best_lnglat, best_proto, sms, stream);
  if (scan == 2)
    return refiner_scan_cell_major(rb, q, cand, cand_stride, B, topk, sort_ws, best_logit, best_lnglat, best_proto, sms,
                                   stream);
  return refiner_scan(rb, q, cand, cand_stride, B, topk, best_logit, best_lnglat, best_proto, sms, stream);
}

int pg_refiner_bank_sqnorm(const float* proto_emb, int64_t P, int32_t D, float* sqnorm_out, void* stream) {
  if (!proto_emb || !sqnorm_out || P < 0 || D <= 0) { set_last_error("pg_refiner_bank_sqnorm: bad argument"); return 1; }
  const int sms = sm_count();
  if (sms < 0) return 1;
  return refiner_bank_sqnorm(proto_emb, P, D, sqnorm_out, sms, reinterpret_cast<cudaStream_t>(stream));
}

int pg_refiner_finalize(const float* best_logit, const float* best_lnglat, const double* init_lnglat,
                        const int64_t* cand_idx, const float* cand_prob, int32_t cand_stride, int64_t B, int32_t topk,
                        float temperature, double max_refinement_km, float* out_lnglat, int64_t* out_cell, int32_t* choice,
                        void* stream) {
  if (!best_logit || !best_lnglat || !init_lnglat || !cand_idx || !cand_prob || !out_lnglat || !out_cell) {
    set_last_error("pg_refiner_finalize: null argument"); return 1;
  }
  if (B <= 0) return 0;
  if (topk <= 0 || topk > cand_stride) { set_last_error("pg_refiner_finalize: bad topk %d / stride %d", topk, cand_stride); return 1; }
  return refiner_finalize(best_logit, best_lnglat, reinterpret_cast<const long long*>(cand_idx), cand_prob, cand_stride,
                          init_lnglat, B, topk, temperature, max_refinement_km, out_lnglat,
                          reinterpret_cast<long long*>(out_cell), choice, reinterpret_cast<cudaStream_t>(stream));
}

int pg_bank_build(const float* data_views, int64_t N, int32_t V, int32_t D, const int64_t* member_off,
                  const int64_t* member_idx, int64_t P, float* data_mean_out, float* proto_emb_out, void* stream) {
  if (!data_views || !member_off || !member_idx || !data_mean_out || !proto_emb_out || N <= 0 || V <= 0 || D <= 0 || P < 0) {
    set_last_error("pg_bank_build: bad argument"); return 1;
  }
  const int sms = sm_count();
  if (sms < 0) return 1;
  return bank_build(data_views, N, V, D, reinterpret_cast<const long long*>(member_off),
                    reinterpret_cast<const long long*>(member_idx), P, data_mean_out, proto_emb_out, sms,
                    reinterpret_cast<cudaStream_t>(stream));
}

// ---------------------------------------------------------------------------------------------- profiler
void pg_profile_begin(void) { prof_begin(); }
int pg_profile_end(void) { return prof_end(); }
void pg_profile_read(const char** names, float* ms, int32_t* counts, int32_t n) { prof_read(names, ms, counts, n); }

// ---------------------------------------------------------------------------------------------- blocks
int pg_gemm_f16(const void* a, int32_t lda, const void* w, int32_t ldw, void* out, int32_t ldo, const float* bias,
                int32_t M, int32_t N, int32_t K, int32_t epilogue, void* stream) {
  if (!a || !w || !out) { set_last_error("pg_gemm_f16: null argument"); return 1; }
  if (epilogue < 0 || epilogue > PG_EPI_F32_BIAS) { set_last_error("pg_gemm_f16: bad epilogue %d", epilogue); return 1; }
  const int sms = sm_count();
  if (sms < 0) return 1;
  GemmProblem p{};
  p.M = M; p.N = N; p.K = K; p.a = a; p.lda = lda; p.w = w; p.ldw = ldw; p.out = out; p.ldo = ldo; p.bias = bias;
  p.epi = epilogue;
  return gemm_f16(p, sms, reinterpret_cast<cudaStream_t>(stream));
}

int pg_gemm_set_schedule(int32_t mode) { return gemm_set_schedule(mode); }

static_assert(PG_EPI_F16_BIAS == EPI_F16_BIAS && PG_EPI_F32_BIAS == EPI_F32_BIAS && PG_EPI_F32_ROWMAP == EPI_F32_ROWMAP &&
              PG_EPI_BF16_DGELU == EPI_BF16_DGELU && PG_EPI_F16_BIAS_QGELU_SAVE == EPI_F16_BIAS_QGELU_SAVE &&
              PG_EPI_F32_BIAS_RESID_STATS == EPI_F32_BIAS_RESID_STATS && PG_EPI_F16_LN_BIAS == EPI_F16_LN_BIAS &&
              PG_EPI_F16_LN_BIAS_QGELU == EPI_F16_LN_BIAS_QGELU, "PG_EPI_* mirror pg::GemmEpilogue");

int pg_gemm_problem_run(const pg_gemm_problem* q, void* stream) {
  if (!q || !q->a || !q->w || !q->out) { set_last_error("pg_gemm_problem_run: null argument"); return 1; }
  const int sms = sm_count();
  if (sms < 0) return 1;
  GemmProblem p{};
  p.M = q->M; p.N = q->N; p.K = q->K; p.a = q->a; p.lda = q->lda; p.w = q->w; p.ldw = q->ldw; p.out = q->out; p.ldo = q->ldo;
  p.bias = q->bias; p.epi = q->epilogue;
  p.rowmap_div = q->rowmap_div; p.rowmap_mul = q->rowmap_mul; p.rowmap_add = q->rowmap_add;
  p.operand_bf16 = q->operand_bf16 ? 1 : 0; p.resid = q->resid; p.aux = q->aux; p.mn_major = q->mn_major ? 1 : 0;
  p.stats = q->stats; p.colsum = q->colsum; p.ln_eps = q->ln_eps;
  return gemm_f16(p, sms, reinterpret_cast<cudaStream_t>(stream));
}

int pg_layernorm_f16(const float* x, void* y, const float* gamma, const float* beta, int64_t rows, int32_t hidden,
                     float eps, void* stream) {
  if (!x || !y || !gamma || !beta) { set_last_error("pg_layernorm_f16: null argument"); return 1; }
  const int sms = sm_count();
  if (sms < 0) return 1;
  return layernorm_f16(x, y, gamma, beta, rows, hidden, eps, sms, reinterpret_cast<cudaStream_t>(stream));
}

int pg_attention_f16(const void* qkv, void* out, int32_t n_views, int32_t seq, int32_t heads, void* stream) {
  if (!qkv || !out) { set_last_error("pg_attention_f16: null argument"); return 1; }
  return attention_f16(qkv, out, n_views, seq, heads, reinterpret_cast<cudaStream_t>(stream));
}

int pg_attention_f16_masked(const void* qkv, void* out, const int64_t* mask, int32_t causal, int32_t n_views, int32_t seq,
                            int32_t heads, void* stream) {
  if (!qkv || !out) { set_last_error("pg_attention_f16_masked: null argument"); return 1; }
  return attention_f16_masked(qkv, out, reinterpret_cast<const long long*>(mask), causal, n_views, seq, heads,
                              reinterpret_cast<cudaStream_t>(stream));
}

int pg_attention_f16_variant(const void* qkv, void* out, float* lse2, int32_t n_views, int32_t seq, int32_t heads,
                             int32_t variant, int32_t poly, void* stream) {
  if (!qkv || !out) { set_last_error("pg_attention_f16_variant: null argument"); return 1; }
  if (variant < 0 || variant > 3) { set_last_error("pg_attention_f16_variant: variant %d not in {0, 1, 2, 3}", variant); return 1; }
  (void)poly;   // one kernel on sm_90a: every variant number of the ABI runs it
  return attention_f16(qkv, out, n_views, seq, heads, reinterpret_cast<cudaStream_t>(stream), lse2);
}

}  // extern "C"
