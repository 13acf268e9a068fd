// Shared by capi.cu and vit_train_capi.cu: the tower handle, workspace carving, SM-count cache.
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

#include <vector>

#include "../../include/pigeon_b200.h"
#include "tma_host.h"

struct pg_vit {
  pg_vit_config cfg;
  pg_vit_weights w;
  std::vector<pg_vit_layer> layers;
  int tokens;
  int grid_patches;
};

struct pg_text {
  pg_text_config cfg;
  pg_text_weights w;
  std::vector<pg_vit_layer> layers;
};

namespace pg {

int sm_count();   // cached cudaDevAttrMultiProcessorCount of the current device, -1 (and last_error) on failure

// The pre-LN encoder-layer stack with LayerNorm kernels (capi.cu), shared by the vision tower (mask NULL, causal 0) and the
// text tower (attention_mask, causal 1).  x f32 [n_seq * seq, hidden]; xn fp16 [rows, hidden]; u fp16 [rows, max(3 hidden,
// intermediate)].
int encoder_layers(const pg_vit_layer* layers, int n_layers, int hidden, int heads, int intermediate, float eps, float* x,
                   void* xn, void* u, int n_seq, int seq, const int64_t* mask, int causal, int sms, cudaStream_t stream);

inline size_t align_up(size_t x, size_t a) { return (x + a - 1) / a * a; }

struct Carver {
  uint8_t* base;
  size_t off = 0;
  explicit Carver(void* p) : base(reinterpret_cast<uint8_t*>(p)) {}
  void* take(size_t bytes) {
    void* p = base ? base + off : nullptr;
    off += align_up(bytes, 1024);
    return p;
  }
};

}  // namespace pg
