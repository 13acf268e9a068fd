// C ABI of the CLIP text tower, the projections and the image-text logits (include/pigeon_b200.h): argument checks,
// workspace carving and the launch sequence of HF CLIPTextTransformer.forward (transformers 4.23.1 modeling_clip.py):
//   token + position embedding -> encoder layers (causal + attention_mask) -> final_layer_norm -> pooled row.
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

#include <new>
#include <vector>

#include "../../include/pigeon_b200.h"
#include "clip.h"
#include "gemm.h"
#include "tma_host.h"
#include "vit_handle.h"
#include "vit_misc.h"

using namespace pg;

namespace {

size_t text_carve(const pg_text* h, int n, int S, void* ws, float** x, void** xn, void** u) {
  const size_t rows = (size_t)n * S;
  const int wide = h->cfg.intermediate > 3 * h->cfg.hidden ? h->cfg.intermediate : 3 * h->cfg.hidden;
  Carver c(ws);
  *x = reinterpret_cast<float*>(c.take(rows * h->cfg.hidden * sizeof(float)));  // residual stream, fp32
  *xn = c.take(rows * h->cfg.hidden * 2);                                      // LayerNorm / attention output (fp16)
  *u = c.take(rows * (size_t)wide * 2);                                        // qkv | fc1 activations (fp16)
  return c.off;
}

}  // namespace

extern "C" {

int pg_text_create(const pg_text_config* cfg, const pg_text_weights* w, pg_text** out) {
  if (!cfg || !w || !out) { set_last_error("pg_text_create: null argument"); return 1; }
  if (cfg->hidden <= 0 || cfg->hidden % 256 || cfg->intermediate <= 0 || cfg->intermediate % 256) {
    set_last_error("pg_text_create: hidden/intermediate must be multiples of 256"); return 1;
  }
  if (cfg->heads <= 0 || cfg->hidden != cfg->heads * 64) { set_last_error("pg_text_create: head_dim must be 64"); return 1; }
  if (cfg->vocab <= 0 || cfg->max_positions <= 0) { set_last_error("pg_text_create: bad vocab / max_positions"); return 1; }
  if (cfg->layers <= 0 || !w->layers_host) { set_last_error("pg_text_create: no layers"); return 1; }
  if (!w->token_emb || !w->pos_emb || !w->final_ln_g || !w->final_ln_b) { set_last_error("pg_text_create: missing weights"); return 1; }
  pg_text* h = new (std::nothrow) pg_text();
  if (!h) { set_last_error("pg_text_create: out of host memory"); return 1; }
  h->cfg = *cfg;
  h->w = *w;
  h->layers.assign(w->layers_host, w->layers_host + cfg->layers);
  h->w.layers_host = h->layers.data();
  *out = h;
  return 0;
}

void pg_text_destroy(pg_text* h) { delete h; }

size_t pg_text_workspace_bytes(const pg_text* h, int32_t n, int32_t S) {
  if (!h || n <= 0 || S <= 0) return 0;
  float* x; void* xn; void* u;
  return text_carve(h, n, S, nullptr, &x, &xn, &u);
}

int pg_text_forward(pg_text* h, const int64_t* input_ids, const int64_t* attention_mask, int32_t n, int32_t S,
                    void* workspace, size_t workspace_bytes, float* pooled_out, float* hidden_out, void* stream_) {
  if (!h || !input_ids || !workspace || !pooled_out) { set_last_error("pg_text_forward: null argument"); return 1; }
  if (n <= 0) return 0;
  const pg_text_config& c = h->cfg;
  if (S < 1 || S > c.max_positions) {
    set_last_error("pg_text_forward: sequence length %d not in [1, %d] (max_position_embeddings)", S, c.max_positions);
    return 1;
  }
  if (n > 65535) { set_last_error("pg_text_forward: n %d > 65535 captions per call", n); return 1; }
  const int sms = sm_count();
  if (sms < 0) return 1;
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  float* x; void* xn; void* u;
  const size_t need = text_carve(h, n, S, workspace, &x, &xn, &u);
  if (workspace_bytes < need) { set_last_error("pg_text_forward: workspace %zu < required %zu", workspace_bytes, need); return 1; }
  if (reinterpret_cast<uintptr_t>(workspace) & 255) { set_last_error("pg_text_forward: workspace must be 256-byte aligned"); return 1; }
  const long rows = (long)n * S;
  const long long* ids = reinterpret_cast<const long long*>(input_ids);
  if (text_embed(ids, h->w.token_emb, h->w.pos_emb, x, rows, S, c.hidden, c.vocab, sms, stream)) return 1;
  if (encoder_layers(h->layers.data(), c.layers, c.hidden, c.heads, c.intermediate, c.ln_eps, x, xn, u, n, S,
                     attention_mask, 1, sms, stream))
    return 1;
  if (rows_layernorm_f32(x, pooled_out, h->w.final_ln_g, h->w.final_ln_b, n, c.hidden, c.ln_eps, ids, S, sms, stream))
    return 1;
  if (hidden_out &&
      rows_layernorm_f32(x, hidden_out, h->w.final_ln_g, h->w.final_ln_b, rows, c.hidden, c.ln_eps, nullptr, 0, sms, stream))
    return 1;
  return 0;
}

size_t pg_clip_project_workspace_bytes(int32_t n, int32_t D) {
  if (n <= 0 || D <= 0) return 0;
  return align_up((size_t)n * 3 * D * 2, 1024);
}

int pg_clip_project(const float* x, int32_t n, int32_t D, const float* ln_g, const float* ln_b, float ln_eps, const void* w3,
                    int32_t P, void* workspace, size_t workspace_bytes, float* out, void* stream_) {
  if (!x || !w3 || !workspace || !out) { set_last_error("pg_clip_project: null argument"); return 1; }
  if (n <= 0) return 0;
  if (D <= 0 || P <= 0) { set_last_error("pg_clip_project: bad shape D=%d P=%d", D, P); return 1; }
  if (workspace_bytes < pg_clip_project_workspace_bytes(n, D)) { set_last_error("pg_clip_project: workspace too small"); return 1; }
  const int sms = sm_count();
  if (sms < 0) return 1;
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (ln_split3(x, workspace, ln_g, ln_b, n, D, ln_eps, sms, stream)) return 1;
  GemmProblem p{};
  p.M = n; p.N = P; p.K = 3 * D;
  p.a = workspace; p.lda = 3 * D; p.w = w3; p.ldw = 3 * D;
  p.out = out; p.ldo = P; p.bias = nullptr; p.epi = EPI_F32_BIAS;
  return gemm_f16(p, sms, stream);
}

int pg_clip_logits(const float* img, int32_t Ni, const float* txt, int32_t Nt, int32_t P, float logit_scale,
                   float* logits_per_image, float* logits_per_text, float* probs, int64_t* pred, float* loss, void* stream) {
  if (!img || !txt || !logits_per_image) { set_last_error("pg_clip_logits: null argument"); return 1; }
  return clip_logits(img, Ni, txt, Nt, P, logit_scale, logits_per_image, logits_per_text, probs,
                     reinterpret_cast<long long*>(pred), loss, reinterpret_cast<cudaStream_t>(stream));
}

}  // extern "C"
