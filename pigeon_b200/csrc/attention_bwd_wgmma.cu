// Backward of the multi-head attention core on sm_90a (wgmma + TMA + mbarrier), head_dim 64 — part of the fine-tune
// step (what autograd runs for HF CLIPAttention in reference training/train_eval_loop.py:216).
//
//   S = scale Q K^T,  P = softmax(S),  O = P V          (forward, attention_wgmma.cu; it keeps lse2 = log2 sum exp)
//   dV = P^T dO,  dP = dO V^T,  dS = P o (dP - delta),  delta = rowsum(dO o O),  dQ = scale dS K,  dK = scale dS^T Q
//
// Two launches of one kernel template, each "row tile" of 64 rows owning its accumulators in registers for the whole loop,
// so that no atomics and no transposes are needed and every MMA uses an operand form the forward kernel already uses:
//   MODE_DQ   CTA = (64 query rows, head, view), loops over KV blocks of 64:
//             S = Q K_j^T (f16), dP = dO V_j^T (bf16)  ->  dS  ->  dQ += dS K_j        (dS: register A operand, K_j: MN-major B)
//   MODE_DKV  CTA = (64 key/value rows, head, view), loops over query blocks of 64:
//             S^T = K Q_j^T (f16), dP^T = V dO_j^T (bf16)  ->  P^T, dS^T  ->  dV += P^T dO_j,  dK += dS^T Q_j
// The logits are recomputed from the SAME fp16 q/k the forward used (so P is reproduced exactly); everything that carries
// gradient magnitude (dO, dS, and the q/k/v copies they multiply) is bf16 — gradients underflow fp16's range.
//
// One warpgroup (128 threads) per CTA; thread 0 keeps the three 64 x 64 tiles of the NEXT block in flight through a 2-slot
// TMA ring.  P / dS are formed on the accumulator fragments of S / dP, which are the A-operand fragments of the next MMA.
//
// kMasked = true is the text tower's variant: the admissibility predicate of the masked forward (key j admissible for query i
// only if j <= i when causal, and mask[view, j] != 0) zeroes P and dS on the recomputed S / S^T fragments.  With causal
// masking a dQ row tile stops at its diagonal KV block and a dK/dV row tile starts at its diagonal query block
// (kRows == kBlk, so the diagonal block index is the tile index).
#include <cuda_bf16.h>

#include "attention.h"
#include "prof.h"
#include "ptx.cuh"
#include "tma_host.h"

namespace pg {

namespace {

constexpr int kHeadDim = 64;
constexpr int kRows = 64;                              // row tile
constexpr int kBlk = 64;                               // column block
constexpr int kTileBytes = 64 * kHeadDim * 2;          // 8 KB
constexpr int kSlotBytes = 3 * kTileBytes;
constexpr int kThreads = 128;
constexpr int kSmemBytes = 2 * kTileBytes + 2 * kSlotBytes + 2 * kBlk * 4 + 64 + 1024;

enum { MODE_DQ = 0, MODE_DKV = 1 };

struct BwdArgs {
  int seq, hidden;
  const float* lse2;    // [n_views * heads, seq]
  const float* delta;   // [n_views * heads, seq]
  __nv_bfloat16* dqkv;  // [n_views * seq, 3 * hidden]
  float scale;          // 1 / sqrt(64)
  float scale_log2;     // scale * log2(e)
  const long long* mask;   // kMasked: optional [n_views, seq], 0 = key excluded
  int causal;              // kMasked: key j admissible for query i only if j <= i
};

__device__ __forceinline__ float ex2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ uint32_t pack_bf16x2(float lo, float hi) {
  __nv_bfloat162 v = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&v);
}

template <int MODE, bool kMasked>
__global__ void __launch_bounds__(kThreads, 2)
attention_bwd_kernel(const __grid_constant__ CUtensorMap tmap_f16, const __grid_constant__ CUtensorMap tmap_bf16,
                     const __grid_constant__ CUtensorMap tmap_do, const BwdArgs args) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* smem_r16 = smem;                              // row tile, fp16 (Q | K)
  uint8_t* smem_rbf = smem + kTileBytes;                 // row tile, bf16 (dO | V)
  uint8_t* smem_st = smem + 2 * kTileBytes;              // ring: [C16 | Cbf1 | Cbf2] per slot
  float* cbuf = reinterpret_cast<float*>(smem_st + 2 * kSlotBytes);   // MODE_DKV: [lse2 | delta] of a query block
  uint64_t* bars = reinterpret_cast<uint64_t*>(cbuf + 2 * kBlk);
  uint64_t* r_full = bars;
  uint64_t* full_bar = bars + 1;             // [2]

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int tile = blockIdx.x, head = blockIdx.y, view = blockIdx.z;
  const int S = args.seq;
  const int heads = args.hidden / kHeadDim;
  int j0 = 0, nb = (S + kBlk - 1) / kBlk;   // column blocks [j0, nb)
  if constexpr (kMasked) {
    if (args.causal) {
      if (MODE == MODE_DQ) nb = tile + 1;
      else j0 = tile;
    }
  }
  const int row0 = view * S;
  const int q_col = head * kHeadDim, k_col = args.hidden + q_col, v_col = 2 * args.hidden + q_col;

  auto load_block = [&](int j) {   // thread 0 only
    const int slot = (j - j0) & 1;
    uint8_t* st = smem_st + slot * kSlotBytes;
    const int c_row = j * kBlk;
    mbar_arrive_expect_tx(&full_bar[slot], kSlotBytes);
    if (MODE == MODE_DQ) {
      tma_load_3d(st, &tmap_f16, &full_bar[slot], k_col, c_row, view);                       // K_j  fp16  (S)
      tma_load_3d(st + kTileBytes, &tmap_bf16, &full_bar[slot], v_col, c_row, view);         // V_j  bf16  (dP)
      tma_load_3d(st + 2 * kTileBytes, &tmap_bf16, &full_bar[slot], k_col, c_row, view);     // K_j  bf16  (dQ)
    } else {
      tma_load_3d(st, &tmap_f16, &full_bar[slot], q_col, c_row, view);                       // Q_j  fp16  (S^T)
      tma_load_3d(st + kTileBytes, &tmap_do, &full_bar[slot], q_col, c_row, view);           // dO_j bf16  (dP^T, dV)
      tma_load_3d(st + 2 * kTileBytes, &tmap_bf16, &full_bar[slot], q_col, c_row, view);     // Q_j  bf16  (dK)
    }
  };

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmap_f16);
    tma_prefetch_desc(&tmap_bf16);
    tma_prefetch_desc(&tmap_do);
    mbar_init(r_full, 1);
    mbar_init(&full_bar[0], 1);
    mbar_init(&full_bar[1], 1);
    fence_mbar_init();
    const int r_row = tile * kRows;
    mbar_arrive_expect_tx(r_full, 2 * kTileBytes);
    if (MODE == MODE_DQ) {
      tma_load_3d(smem_r16, &tmap_f16, r_full, q_col, r_row, view);
      tma_load_3d(smem_rbf, &tmap_do, r_full, q_col, r_row, view);
    } else {
      tma_load_3d(smem_r16, &tmap_f16, r_full, k_col, r_row, view);
      tma_load_3d(smem_rbf, &tmap_bf16, r_full, v_col, r_row, view);
    }
    load_block(j0);
  }
  __syncthreads();

  // this thread's two rows of the row tile (accumulator fragment layout) and its column pairs 8 g + 2 (lane & 3) + {0, 1}
  const int r_a = tile * kRows + 16 * warp + (lane >> 2), r_b = r_a + 8;
  const bool va = r_a < S, vb = r_b < S;
  const float c = args.scale_log2, scale = args.scale;
  const size_t stat0 = ((size_t)view * heads + head) * S;
  float lse_a = 0.f, lse_b = 0.f, dl_a = 0.f, dl_b = 0.f;
  if (MODE == MODE_DQ) {
    if (va) { lse_a = args.lse2[stat0 + r_a]; dl_a = args.delta[stat0 + r_a]; }
    if (vb) { lse_b = args.lse2[stat0 + r_b]; dl_b = args.delta[stat0 + r_b]; }
  }
  const uint32_t r16_addr = smem_u32(smem_r16), rbf_addr = smem_u32(smem_rbf);
  float acc1[32], acc2[32];   // dQ | dV, dK
#pragma unroll
  for (int i = 0; i < 32; ++i) acc1[i] = acc2[i] = 0.f;
  // kMasked: admissibility of this thread's two rows as keys (MODE_DKV)
  bool key_a = true, key_b = true;
  if constexpr (kMasked) {
    if (MODE == MODE_DKV && args.mask) {
      key_a = va && __ldg(args.mask + (size_t)view * S + r_a) != 0;
      key_b = vb && __ldg(args.mask + (size_t)view * S + r_b) != 0;
    }
  }
  mbar_wait(r_full, 0);

  for (int j = j0; j < nb; ++j) {
    const int slot = (j - j0) & 1;
    if (threadIdx.x == 0 && j + 1 < nb) load_block(j + 1);   // slot (j + 1) & 1 was released by the barrier ending j - 1
    if (MODE == MODE_DKV) {
      // per-column statistics of this query block (columns past the view are masked below)
      const int qi = j * kBlk + (threadIdx.x & 63);
      cbuf[threadIdx.x] = qi < S ? (threadIdx.x < 64 ? args.lse2[stat0 + qi] : args.delta[stat0 + qi]) : 0.f;
      __syncthreads();
    }
    mbar_wait(&full_bar[slot], ((j - j0) >> 1) & 1);
    const uint32_t c16 = smem_u32(smem_st + slot * kSlotBytes), cb1 = c16 + kTileBytes, cb2 = cb1 + kTileBytes;

    float sv[32], dv[32];
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < kHeadDim / 16; ++k)
      wgmma_ss_n64_f16<0, 0>(sv, make_smem_desc(r16_addr + k * 32, 16, 1024), make_smem_desc(c16 + k * 32, 16, 1024), k != 0);
#pragma unroll
    for (int k = 0; k < kHeadDim / 16; ++k)
      wgmma_ss_n64_bf16<0, 0>(dv, make_smem_desc(rbf_addr + k * 32, 16, 1024), make_smem_desc(cb1 + k * 32, 16, 1024), k != 0);
    wgmma_commit();
    wgmma_wait<0>();

    uint32_t pk_p[4][4], pk_ds[4][4];   // A fragments, one per 16 columns of the block
#pragma unroll
    for (int g = 0; g < 8; ++g) {
      float pv[4], ds[4];
#pragma unroll
      for (int e = 0; e < 4; ++e) {   // e & 1: column of the pair; e >> 1: row a / row b
        const int col = j * kBlk + 8 * g + 2 * (lane & 3) + (e & 1);   // index inside the view of this column
        bool ok = ((e >> 1) ? vb : va) && col < S;
        if constexpr (kMasked) {
          const int row = (e >> 1) ? r_b : r_a;
          if (MODE == MODE_DQ) {       // row = query, col = key
            if (args.causal) ok = ok && col <= row;
            if (args.mask) ok = ok && __ldg(args.mask + (size_t)view * S + col) != 0;
          } else {                     // row = key, col = query
            if (args.causal) ok = ok && row <= col;
            ok = ok && ((e >> 1) ? key_b : key_a);
          }
        }
        float lse, dl;
        if (MODE == MODE_DQ) { lse = (e >> 1) ? lse_b : lse_a; dl = (e >> 1) ? dl_b : dl_a; }
        else { lse = cbuf[col - j * kBlk]; dl = cbuf[kBlk + col - j * kBlk]; }
        const float p = ok ? ex2(fmaf(sv[4 * g + e], c, -lse)) : 0.f;
        pv[e] = p;
        ds[e] = ok ? p * (dv[4 * g + e] - dl) * scale : 0.f;
      }
      pk_p[g >> 1][2 * (g & 1)] = pack_bf16x2(pv[0], pv[1]);
      pk_p[g >> 1][2 * (g & 1) + 1] = pack_bf16x2(pv[2], pv[3]);
      pk_ds[g >> 1][2 * (g & 1)] = pack_bf16x2(ds[0], ds[1]);
      pk_ds[g >> 1][2 * (g & 1) + 1] = pack_bf16x2(ds[2], ds[3]);
    }

    wgmma_fence();
    if (MODE == MODE_DQ) {
#pragma unroll
      for (int k = 0; k < kBlk / 16; ++k)      // dQ += dS K_j : contraction over the block's kv rows
        wgmma_rs_n64_bf16<1>(acc1, pk_ds[k], make_smem_desc(cb2 + k * 16 * 128, 1024, 1024), 1);
    } else {
#pragma unroll
      for (int k = 0; k < kBlk / 16; ++k)      // dV += P^T dO_j : contraction over the block's query rows
        wgmma_rs_n64_bf16<1>(acc1, pk_p[k], make_smem_desc(cb1 + k * 16 * 128, 1024, 1024), 1);
#pragma unroll
      for (int k = 0; k < kBlk / 16; ++k)      // dK += dS^T Q_j
        wgmma_rs_n64_bf16<1>(acc2, pk_ds[k], make_smem_desc(cb2 + k * 16 * 128, 1024, 1024), 1);
    }
    wgmma_commit();
    wgmma_wait<0>();
    __syncthreads();   // the slot and cbuf are consumed
  }

  // epilogue: accumulators -> bf16 -> dqkv
  constexpr int kNumAcc = (MODE == MODE_DQ) ? 1 : 2;
#pragma unroll
  for (int a = 0; a < kNumAcc; ++a) {
    // MODE_DQ: acc1 = dQ -> q section;  MODE_DKV: acc1 = dV -> v section, acc2 = dK -> k section
    const int out_col = (MODE == MODE_DQ) ? q_col : (a == 0 ? v_col : k_col);
    const float* acc = (a == 0) ? acc1 : acc2;
    __nv_bfloat16* oa = args.dqkv + (size_t)(row0 + r_a) * (3 * args.hidden) + out_col + 2 * (lane & 3);
    __nv_bfloat16* ob = oa + (size_t)8 * (3 * args.hidden);
#pragma unroll
    for (int g = 0; g < 8; ++g) {
      if (va) *reinterpret_cast<uint32_t*>(oa + 8 * g) = pack_bf16x2(acc[4 * g], acc[4 * g + 1]);
      if (vb) *reinterpret_cast<uint32_t*>(ob + 8 * g) = pack_bf16x2(acc[4 * g + 2], acc[4 * g + 3]);
    }
  }
}

template <int MODE, bool kMasked = false>
int launch_bwd(const CUtensorMap& t16, const CUtensorMap& tbf, const CUtensorMap& tdo, const BwdArgs& a, int n_views,
               int heads, cudaStream_t stream) {
  auto kern = attention_bwd_kernel<MODE, kMasked>;
  cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemBytes);
  if (e != cudaSuccess) { set_last_error("attention_backward: cudaFuncSetAttribute: %s", cudaGetErrorString(e)); return 1; }
  dim3 grid((a.seq + kRows - 1) / kRows, heads, n_views);
  ProfScope prof(MODE == MODE_DQ ? (kMasked ? "attention_bwd_dq_masked" : "attention_bwd_dq")
                                 : (kMasked ? "attention_bwd_dkv_masked" : "attention_bwd_dkv"), stream);
  kern<<<grid, kThreads, kSmemBytes, stream>>>(t16, tbf, tdo, a);
  e = cudaGetLastError();
  if (e != cudaSuccess) { set_last_error("attention_backward launch: %s", cudaGetErrorString(e)); return 1; }
  return 0;
}

}  // namespace

namespace {

template <bool kMasked>
int run_backward(const void* qkv_f16, const void* qkv_bf16, const void* d_out_bf16, const float* lse2, const float* delta,
                 void* dqkv_bf16, const long long* mask, int causal, int n_views, int seq, int heads, cudaStream_t stream) {
  if (n_views <= 0) return 0;
  if (n_views > 65535) { set_last_error("attention_backward: n_views %d > 65535 (grid.z)", n_views); return 1; }
  const int hidden = heads * kHeadDim;
  CUtensorMap t16, tbf, tdo;   // per view: tiles past a view's last token are zero-filled
  if (make_tmap_f16_3d(&t16, qkv_f16, n_views, seq, 3 * hidden, 3 * hidden, kBlk, kHeadDim)) return 1;
  if (make_tmap_f16_3d(&tbf, qkv_bf16, n_views, seq, 3 * hidden, 3 * hidden, kBlk, kHeadDim)) return 1;
  if (make_tmap_f16_3d(&tdo, d_out_bf16, n_views, seq, hidden, hidden, kBlk, kHeadDim)) return 1;
  BwdArgs a;
  a.seq = seq; a.hidden = hidden; a.lse2 = lse2; a.delta = delta;
  a.dqkv = reinterpret_cast<__nv_bfloat16*>(dqkv_bf16);
  a.scale = 0.125f;
  a.scale_log2 = 0.125f * 1.4426950408889634f;
  a.mask = mask;
  a.causal = causal;
  if (launch_bwd<MODE_DQ, kMasked>(t16, tbf, tdo, a, n_views, heads, stream)) return 1;
  return launch_bwd<MODE_DKV, kMasked>(t16, tbf, tdo, a, n_views, heads, stream);
}

}  // namespace

int attention_backward(const void* qkv_f16, const void* qkv_bf16, const void* d_out_bf16, const float* lse2,
                       const float* delta, void* dqkv_bf16, int n_views, int seq, int heads, cudaStream_t stream) {
  return run_backward<false>(qkv_f16, qkv_bf16, d_out_bf16, lse2, delta, dqkv_bf16, nullptr, 0, n_views, seq, heads, stream);
}

int attention_backward_masked(const void* qkv_f16, const void* qkv_bf16, const void* d_out_bf16, const float* lse2,
                              const float* delta, void* dqkv_bf16, const long long* mask, int causal, int n_views, int seq,
                              int heads, cudaStream_t stream) {
  if (!mask && !causal)
    return attention_backward(qkv_f16, qkv_bf16, d_out_bf16, lse2, delta, dqkv_bf16, n_views, seq, heads, stream);
  return run_backward<true>(qkv_f16, qkv_bf16, d_out_bf16, lse2, delta, dqkv_bf16, mask, causal ? 1 : 0, n_views, seq, heads,
                            stream);
}

}  // namespace pg
