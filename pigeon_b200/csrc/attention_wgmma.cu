// Multi-head self-attention core for the CLIP vision tower on sm_90a (wgmma + TMA + mbarrier).
//
//   out[v, s, h*64 + :] = softmax_s'( q[v,s,h,:] . k[v,s',h,:] / sqrt(64) ) @ v[v,s',h,:]
//
// Restates the attention core of HF CLIPAttention.forward (bmm -> fp32 softmax -> bmm; no mask, no
// dropout in eval) that the reference reaches through models/clip_embedder.py:63 and
// models/super_guessr.py:395.  head_dim is fixed to 64 (ViT-L/14: 16 heads x 64).
//
// Input  qkv : fp16 [n_views * S, 3 * hidden]   row = (view, token); cols = [q | k | v], head-major inside
// Output out : fp16 [n_views * S, hidden]
//
// One CTA (one warpgroup, 128 threads) per (q-tile of 64 rows, head, view); 40 KB of shared memory, so several CTAs share
// an SM and cover each other's TMA and softmax latency.  Single pass, flash-style, KV blocks of 64:
//   thread 0 keeps the K/V tiles (64 x 64 halves, 128B swizzle) of the NEXT block in flight through a 2-slot ring;
//   S_j = Q K_j^T            wgmma m64n64k16, both operands K-major in shared memory, fp32 accumulator in registers;
//   online softmax           on the accumulator fragment (a row lives in the four lanes of a quad): running maximum m and
//                            row sum l, O and l rescaled when m rises, P_j = exp2(S_j c - m c) packed to fp16 in place —
//                            the accumulator fragment of S is exactly the A-operand fragment of the next MMA;
//   O += P_j V_j             wgmma with A from registers and V as an MN-major shared-memory operand.
// Final O / l -> fp16 through shared memory (16-byte coalesced stores).
//
// kMasked = true is the text tower's variant (HF CLIPTextTransformer: causal mask plus the padding `attention_mask`,
// modeling_clip.py 4.23.1 `_build_causal_attention_mask` / `_expand_mask`): key j is admissible for query i only if
// j <= i (causal) and mask[view, j] != 0, applied on the S fragment where the ragged-tail test sits.  A causal q-tile stops
// at its diagonal KV block.  Block 0 holds key 0, which every row admits as long as mask[view, 0] != 0 (CLIP's BOS):
// the running maximum is then finite after the first block and the rescale ex2((m - n) c) never sees -inf - -inf.
#include "attention.h"
#include "prof.h"
#include "ptx.cuh"
#include "tma_host.h"

#include <atomic>

namespace pg {

namespace {

constexpr int kHeadDim = 64;
constexpr int kBlockQ = 64;
constexpr int kBlockKV = 64;
constexpr int kTileBytes = 64 * kHeadDim * 2;    // 8 KB: Q, K_j or V_j
constexpr int kThreads = 128;
constexpr int kOutLdBytes = 144;                 // O staging rows (128 B of fp16 + 16 B pad against bank conflicts)
constexpr int kSmemBytes = 5 * kTileBytes + 1024 + 64;

struct AttnArgs {
  int seq;      // tokens per view (577)
  int hidden;   // heads * 64
  __half* out;  // [n_views*seq, hidden]
  float scale_log2;  // (1/sqrt(64)) * log2(e)
  float* lse2;       // optional [n_views * heads, seq]: log2-domain log-sum-exp of the scaled logits (for the backward pass)
  const long long* mask;   // kMasked: optional [n_views, seq], 0 = key excluded
  int causal;              // kMasked: key j admissible for query i only if j <= i
};

__device__ __forceinline__ float ex2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

template <bool kMasked>
__global__ void __launch_bounds__(kThreads, 4)
attention_kernel(const __grid_constant__ CUtensorMap tmap_qkv, const AttnArgs args) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* smem_q = smem;
  uint8_t* smem_kv = smem + kTileBytes;    // slot s: K at 2 s, V at 2 s + 1 (tiles)
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + 5 * kTileBytes);
  uint64_t* q_full = bars;
  uint64_t* kv_full = bars + 1;            // [2]

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int q_tile = blockIdx.x, head = blockIdx.y, view = blockIdx.z;
  const int S = args.seq;
  int nb = (S + kBlockKV - 1) / kBlockKV;                       // KV blocks (10 for S = 577)
  if constexpr (kMasked) {
    if (args.causal && q_tile + 1 < nb) nb = q_tile + 1;        // kBlockQ == kBlockKV: the diagonal block is q_tile
  }
  const int row0 = view * S;                                    // first row of this view in qkv / out
  const int q_col = head * kHeadDim, k_col = args.hidden + q_col, v_col = 2 * args.hidden + q_col;

  auto load_kv = [&](int j) {   // thread 0 only
    const int slot = j & 1;
    mbar_arrive_expect_tx(&kv_full[slot], 2 * kTileBytes);
    tma_load_3d(smem_kv + (2 * slot) * kTileBytes, &tmap_qkv, &kv_full[slot], k_col, j * kBlockKV, view);
    tma_load_3d(smem_kv + (2 * slot + 1) * kTileBytes, &tmap_qkv, &kv_full[slot], v_col, j * kBlockKV, view);
  };

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmap_qkv);
    mbar_init(q_full, 1);
    mbar_init(&kv_full[0], 1);
    mbar_init(&kv_full[1], 1);
    fence_mbar_init();
    mbar_arrive_expect_tx(q_full, kTileBytes);
    tma_load_3d(smem_q, &tmap_qkv, q_full, q_col, q_tile * kBlockQ, view);
    load_kv(0);
  }
  __syncthreads();

  const float c = args.scale_log2;
  const uint32_t q_addr = smem_u32(smem_q);
  float o[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) o[i] = 0.f;
  float m0 = -INFINITY, m1 = -INFINITY;   // running maxima of this thread's two rows (raw logit units)
  float l0 = 0.f, l1 = 0.f;               // this thread's share of the two row sums
  mbar_wait(q_full, 0);

  for (int j = 0; j < nb; ++j) {
    const int slot = j & 1;
    // slot (j + 1) & 1 held block j - 1: every warp passed the barrier that ends iteration j - 1
    if (threadIdx.x == 0 && j + 1 < nb) load_kv(j + 1);
    mbar_wait(&kv_full[slot], (j >> 1) & 1);
    const uint32_t k_addr = smem_u32(smem_kv + (2 * slot) * kTileBytes);
    const uint32_t v_addr = k_addr + kTileBytes;

    float s[32];
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < kHeadDim / 16; ++k)
      wgmma_ss_n64_f16<0, 0>(s, make_smem_desc(q_addr + k * 32, 16, 1024), make_smem_desc(k_addr + k * 32, 16, 1024), k != 0);
    wgmma_commit();
    wgmma_wait<0>();

    // kv columns past the view (last block only) drop out of the maximum and get P = 0; their K / V rows are zeros (the
    // tensor map is per view, so TMA zero-fills past the last token and no other view's data enters this one's MMAs)
    if constexpr (kMasked) {
      // rows 16 warp + lane / 4 (s[4g], s[4g + 1]) and that + 8 (s[4g + 2], s[4g + 3]) of the q-tile
      const int q0 = q_tile * kBlockQ + 16 * warp + (lane >> 2);
      const long long* mrow = args.mask ? args.mask + (size_t)view * S : nullptr;
#pragma unroll
      for (int i = 0; i < 32; ++i) {
        const int kv = j * kBlockKV + 8 * (i >> 2) + 2 * (lane & 3) + (i & 1);
        bool ok = kv < S;
        if (args.causal) ok = ok && kv <= q0 + 8 * ((i >> 1) & 1);
        if (mrow) ok = ok && __ldg(mrow + kv) != 0;
        if (!ok) s[i] = -INFINITY;
      }
    } else {
      const int valid = S - j * kBlockKV;
      if (valid < kBlockKV) {
#pragma unroll
        for (int i = 0; i < 32; ++i) {
          const int col = 8 * (i >> 2) + 2 * (lane & 3) + (i & 1);
          if (col >= valid) s[i] = -INFINITY;
        }
      }
    }
    float b0 = -INFINITY, b1 = -INFINITY;
#pragma unroll
    for (int g = 0; g < 8; ++g) {
      b0 = fmaxf(b0, fmaxf(s[4 * g], s[4 * g + 1]));
      b1 = fmaxf(b1, fmaxf(s[4 * g + 2], s[4 * g + 3]));
    }
    b0 = fmaxf(b0, __shfl_xor_sync(0xffffffffu, b0, 1));
    b0 = fmaxf(b0, __shfl_xor_sync(0xffffffffu, b0, 2));
    b1 = fmaxf(b1, __shfl_xor_sync(0xffffffffu, b1, 1));
    b1 = fmaxf(b1, __shfl_xor_sync(0xffffffffu, b1, 2));
    const float n0 = fmaxf(m0, b0), n1 = fmaxf(m1, b1);   // finite: every block has at least one valid column
    const float a0 = ex2((m0 - n0) * c), a1 = ex2((m1 - n1) * c);
    m0 = n0; m1 = n1;
    l0 *= a0; l1 *= a1;
#pragma unroll
    for (int g = 0; g < 8; ++g) {
      o[4 * g] *= a0; o[4 * g + 1] *= a0;
      o[4 * g + 2] *= a1; o[4 * g + 3] *= a1;
    }
    const float mc0 = m0 * c, mc1 = m1 * c;
    uint32_t p[4][4];   // A fragments of P: one per 16 kv columns
#pragma unroll
    for (int g = 0; g < 8; ++g) {
      const float p00 = ex2(fmaf(s[4 * g], c, -mc0)), p01 = ex2(fmaf(s[4 * g + 1], c, -mc0));
      const float p10 = ex2(fmaf(s[4 * g + 2], c, -mc1)), p11 = ex2(fmaf(s[4 * g + 3], c, -mc1));
      l0 += p00 + p01;
      l1 += p10 + p11;
      p[g >> 1][2 * (g & 1)] = pack_half2(p00, p01);
      p[g >> 1][2 * (g & 1) + 1] = pack_half2(p10, p11);
    }

    wgmma_fence();
#pragma unroll
    for (int k = 0; k < kBlockKV / 16; ++k)   // V tile: row = kv index (128 B of head_dim), 16 kv rows per step
      wgmma_rs_n64_f16<1>(o, p[k], make_smem_desc(v_addr + k * 16 * 128, 1024, 1024), 1);
    wgmma_commit();
    wgmma_wait<0>();
    __syncthreads();   // both tiles of this slot are consumed: it may be refilled
  }

  // epilogue: O / l -> fp16 -> shared (over Q and the first K tile) -> global
  l0 += __shfl_xor_sync(0xffffffffu, l0, 1);
  l0 += __shfl_xor_sync(0xffffffffu, l0, 2);
  l1 += __shfl_xor_sync(0xffffffffu, l1, 1);
  l1 += __shfl_xor_sync(0xffffffffu, l1, 2);
  const float inv0 = 1.0f / l0, inv1 = 1.0f / l1;
  const int r_loc = 16 * warp + (lane >> 2);
  if (args.lse2 != nullptr && (lane & 3) == 0) {
    float* lse = args.lse2 + ((size_t)view * (args.hidden / kHeadDim) + head) * S;
    const int q0 = q_tile * kBlockQ + r_loc;
    if (q0 < S) lse[q0] = m0 * c + log2f(l0);
    if (q0 + 8 < S) lse[q0 + 8] = m1 * c + log2f(l1);
  }
  const uint32_t st = smem_u32(smem);
#pragma unroll
  for (int g = 0; g < 8; ++g) {
    const uint32_t off = (uint32_t)r_loc * kOutLdBytes + g * 16 + (lane & 3) * 4;
    asm volatile("st.shared.b32 [%0], %1;" ::"r"(st + off), "r"(pack_half2(o[4 * g] * inv0, o[4 * g + 1] * inv0)) : "memory");
    asm volatile("st.shared.b32 [%0], %1;" ::"r"(st + off + 8 * kOutLdBytes), "r"(pack_half2(o[4 * g + 2] * inv1, o[4 * g + 3] * inv1)) : "memory");
  }
  __syncthreads();
#pragma unroll
  for (int i = 0; i < (kBlockQ * 8) / kThreads; ++i) {
    const int piece = threadIdx.x + i * kThreads, r = piece >> 3, c16 = piece & 7;
    const int q_row = q_tile * kBlockQ + r;
    if (q_row < S)
      *reinterpret_cast<uint4*>(args.out + (size_t)(row0 + q_row) * args.hidden + q_col + c16 * 8) = lds_u4(st + r * kOutLdBytes + c16 * 16);
  }
}

template <bool kMasked>
int launch_attention(const void* qkv, void* out, int n_views, int seq, int heads, cudaStream_t stream, float* lse2,
                     const long long* mask, int causal, const char* name) {
  if (n_views <= 0) return 0;
  if (n_views > 65535) { set_last_error("attention: n_views %d > 65535 (grid.z)", n_views); return 1; }
  const int hidden = heads * kHeadDim;
  CUtensorMap tm;
  if (make_tmap_f16_3d(&tm, qkv, n_views, seq, 3 * hidden, 3 * hidden, kBlockKV, kHeadDim)) return 1;
  static std::atomic<int> attr_set_dev[64];   // per instantiation and device (the attribute is per context)
  int dev = 0;
  cudaGetDevice(&dev);
  if (dev < 0 || dev >= 64) dev = 0;
  if (!attr_set_dev[dev].load(std::memory_order_acquire)) {
    cudaError_t e = cudaFuncSetAttribute(attention_kernel<kMasked>, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemBytes);
    if (e != cudaSuccess) { set_last_error("attention: cudaFuncSetAttribute: %s", cudaGetErrorString(e)); return 1; }
    attr_set_dev[dev].store(1, std::memory_order_release);
  }
  AttnArgs a;
  a.seq = seq;
  a.hidden = hidden;
  a.out = reinterpret_cast<__half*>(out);
  a.scale_log2 = 0.125f * 1.4426950408889634f;
  a.lse2 = lse2;
  a.mask = mask;
  a.causal = causal;
  dim3 grid((seq + kBlockQ - 1) / kBlockQ, heads, n_views);
  ProfScope prof(name, stream);
  attention_kernel<kMasked><<<grid, kThreads, kSmemBytes, stream>>>(tm, a);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) { set_last_error("attention launch: %s", cudaGetErrorString(e)); return 1; }
  return 0;
}

}  // namespace

int attention_f16(const void* qkv, void* out, int n_views, int seq, int heads, cudaStream_t stream, float* lse2) {
  return launch_attention<false>(qkv, out, n_views, seq, heads, stream, lse2, nullptr, 0, "attention");
}

int attention_f16_masked(const void* qkv, void* out, const long long* mask, int causal, int n_views, int seq, int heads,
                         cudaStream_t stream, float* lse2) {
  if (!mask && !causal) return attention_f16(qkv, out, n_views, seq, heads, stream, lse2);
  return launch_attention<true>(qkv, out, n_views, seq, heads, stream, lse2, mask, causal ? 1 : 0, "attention_masked");
}

}  // namespace pg
