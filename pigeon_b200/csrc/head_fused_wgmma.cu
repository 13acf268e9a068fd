// Geocell head as ONE kernel ("a single TMA-fed GEMM+bias+softmax kernel"): restates reference
// models/super_guessr.py:437 (view mean), :447-448 (cell_layer Linear + softmax), :454-455 (arg-max + centroid), :459 (top-k).
//
// grid = (sample blocks of 128) x (geocell blocks of 128); one output tile per CTA, 256 threads = two warpgroups.
// Per 64-column group g of the embedding:
//   thread 0    TMA of the packed weight [C, 3D] = [Whi | Whi | Wlo]: the tiles Whi_{g+1}, Wlo_{g+1} of the NEXT group
//   all threads A operand, thread = (sample, half of the group): view mean of the fp32 embeddings (torch.mean order), hi / lo
//               split, written straight into the 128-byte-swizzled K-major operand tiles (generic proxy ->
//               fence.proxy.async), so the pooled embedding never travels through HBM as an fp16 operand
//   warpgroups  64 samples each:  acc += hi_g Whi_g^T + lo_g Whi_g^T + hi_g Wlo_g^T   (error-compensated fp16 split, fp32
//               accumulator in registers, wgmma m64n128k16; the dropped lo.Wlo term is O(2^-22))
// then accumulators -> shared tile -> + bias -> logits (coalesced through the shared GEMM epilogue).
// The CTA that finishes a sample block LAST (device-scope ticket per block) turns the block's logit rows, still in L2, into
// probabilities, the arg-max + centroid lookup and the top-k: one warp per sample, first-index ties, NaN ranks first (torch).
#include "head.h"

#include <cuda_fp16.h>
#include <math.h>
#include <stdint.h>

#include "gemm_epilogue.cuh"
#include "prof.h"
#include "ptx.cuh"
#include "tma_host.h"

namespace pg {

namespace {

constexpr int HB_M = 128;
constexpr int HB_N = kEpiTileN;
constexpr int HB_K = 64;              // embedding columns per group = one 128-byte swizzle row of fp16
constexpr int kHeadStages = 2;
constexpr int kHeadABytes = HB_M * HB_K * 2;
constexpr int kHeadWBytes = HB_N * HB_K * 2;
constexpr int kHeadStageBytes = 2 * kHeadABytes + 2 * kHeadWBytes;   // hi, lo | Whi, Wlo
constexpr int kHeadThreads = 256;
constexpr int kHeadTileBytes = kHeadStages * kHeadStageBytes + kAccTileBytes + 4 * kStageWarpBytes;
constexpr int kHeadSmem = kHeadTileBytes + 1024 /*alignment*/ + 256 /*barriers*/;
constexpr int kHeadMaxCells = 6144;   // probability rows of 8 warps reuse the operand stages and the accumulator tile
static_assert(kHeadMaxCells * 8 * 4 <= kHeadTileBytes, "probability rows must fit the reused shared memory");

struct HeadArgs {
  const float* emb;   // [B, V, D]
  int B, V, D, C, k;
  const float* bias;
  const double* centroids;
  float* pooled;
  float* logits;
  float* probs;
  long long* pred_cell;
  double* pred_lnglat;
  float* topk_val;
  long long* topk_idx;
  int* tickets;       // [sample blocks], zero before the launch; left zero by the kernel
};

// "greater" with first-index tie-break; NaN ranks above everything (torch.argmax / topk semantics) — as in head.cu
__device__ __forceinline__ bool head_better(float v, int i, float bv, int bi) {
  const bool vn = isnan(v), bn = isnan(bv);
  if (vn != bn) return vn;
  if (vn && bn) return i < bi;
  return (v > bv) || (v == bv && i < bi);
}

__global__ void __launch_bounds__(kHeadThreads, 1)
head_fused_kernel(const __grid_constant__ CUtensorMap tmap_w, const HeadArgs h) {
  extern __shared__ uint8_t head_smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(head_smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* smem_acc = smem + kHeadStages * kHeadStageBytes;    // fp32 accumulator tile
  uint8_t* smem_stage = smem_acc + kAccTileBytes;              // epilogue staging, 4 warps
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem_stage + 4 * kStageWarpBytes);   // [kHeadStages] weight tiles landed
  int* last_flag = reinterpret_cast<int*>(full_bar + kHeadStages);

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int wg = warp >> 2;
  const int n_blocks = (h.C + HB_N - 1) / HB_N;
  const int m_blk = blockIdx.x / n_blocks, n_blk = blockIdx.x % n_blocks;
  const int groups = h.D / HB_K;

  auto load_w = [&](int g) {   // thread 0 only
    const int stage = g % kHeadStages;
    uint8_t* st = smem + stage * kHeadStageBytes + 2 * kHeadABytes;
    mbar_arrive_expect_tx(&full_bar[stage], 2 * kHeadWBytes);
    tma_load_2d(st, &tmap_w, &full_bar[stage], g * HB_K, n_blk * HB_N);                          // Whi_g
    tma_load_2d(st + kHeadWBytes, &tmap_w, &full_bar[stage], 2 * h.D + g * HB_K, n_blk * HB_N);  // Wlo_g
  };
  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmap_w);
    for (int s = 0; s < kHeadStages; ++s) mbar_init(&full_bar[s], 1);
    fence_mbar_init();
    load_w(0);
  }
  __syncthreads();

  // A operand: this thread's sample row and its 32 of the group's 64 columns
  const int row = threadIdx.x & (HB_M - 1), half = threadIdx.x >> 7;
  const long b = (long)m_blk * HB_M + row;
  const bool live = b < h.B;
  const float vcount = (float)h.V;     // x = s / V like torch.mean (division, not a reciprocal multiply)
  const uint32_t row_off = (uint32_t)(row >> 3) * 1024 + (uint32_t)(row & 7) * 128;
  float acc[HB_N / 2];
  for (int g = 0; g < groups; ++g) {
    const int stage = g % kHeadStages;
    // stage (g + 1) % 2 was read by group g - 1, which every warp has left through the barrier at its end
    if (threadIdx.x == 0 && g + 1 < groups) load_w(g + 1);
    float x[HB_K / 2];
#pragma unroll
    for (int i = 0; i < HB_K / 2; ++i) x[i] = 0.f;
    if (live) {
      for (int v = 0; v < h.V; ++v) {
        const float4* src = reinterpret_cast<const float4*>(h.emb + (b * h.V + v) * h.D + g * HB_K + half * (HB_K / 2));
#pragma unroll
        for (int i = 0; i < HB_K / 8; ++i) {
          const float4 t = __ldg(src + i);
          x[4 * i] += t.x; x[4 * i + 1] += t.y; x[4 * i + 2] += t.z; x[4 * i + 3] += t.w;
        }
      }
#pragma unroll
      for (int i = 0; i < HB_K / 2; ++i) x[i] = x[i] / vcount;
      if (n_blk == 0) {
        float4* dst = reinterpret_cast<float4*>(h.pooled + b * h.D + g * HB_K + half * (HB_K / 2));
#pragma unroll
        for (int i = 0; i < HB_K / 8; ++i) dst[i] = make_float4(x[4 * i], x[4 * i + 1], x[4 * i + 2], x[4 * i + 3]);
      }
    }
    const uint32_t st = smem_u32(smem) + stage * kHeadStageBytes;   // explicit st.shared: `smem` is generic to the compiler
#pragma unroll
    for (int i = 0; i < 4; ++i) {   // 16-byte piece ch of row r sits at piece ch ^ (r & 7)
      const int ch = 4 * half + i;
      uint32_t hi4[4], lo4[4];
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const float a = x[8 * i + 2 * e], c = x[8 * i + 2 * e + 1];
        const __half ah = __float2half_rn(a), ch_ = __float2half_rn(c);
        const __half al = __float2half_rn(a - __half2float(ah)), cl = __float2half_rn(c - __half2float(ch_));
        hi4[e] = (uint32_t)__half_as_ushort(ah) | ((uint32_t)__half_as_ushort(ch_) << 16);
        lo4[e] = (uint32_t)__half_as_ushort(al) | ((uint32_t)__half_as_ushort(cl) << 16);
      }
      const uint32_t off = row_off + (uint32_t)((ch ^ (row & 7)) << 4);
      sts_u4(st + off, make_uint4(hi4[0], hi4[1], hi4[2], hi4[3]));
      sts_u4(st + kHeadABytes + off, make_uint4(lo4[0], lo4[1], lo4[2], lo4[3]));
    }
    fence_proxy_async_smem();   // generic-proxy writes -> visible to the tensor core's async proxy
    __syncthreads();
    mbar_wait(&full_bar[stage], (g / kHeadStages) & 1);
    const uint32_t hi = st + wg * (kHeadABytes / 2);   // this warpgroup's 64 rows
    const uint32_t lo = hi + kHeadABytes;
    const uint32_t whi = st + 2 * kHeadABytes;
    const uint32_t wlo = whi + kHeadWBytes;
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < HB_K / 16; ++k) {
      const uint64_t d_hi = make_smem_desc(hi + k * 32, 16, 1024);
      const uint64_t d_lo = make_smem_desc(lo + k * 32, 16, 1024);
      const uint64_t d_whi = make_smem_desc(whi + k * 32, 16, 1024);
      const uint64_t d_wlo = make_smem_desc(wlo + k * 32, 16, 1024);
      wgmma_ss_n128_f16<0, 0>(acc, d_hi, d_whi, (g | k) != 0);
      wgmma_ss_n128_f16<0, 0>(acc, d_lo, d_whi, 1);
      wgmma_ss_n128_f16<0, 0>(acc, d_hi, d_wlo, 1);
    }
    wgmma_commit();
    wgmma_wait<0>();
    __syncthreads();   // the stage is consumed
  }
  // ------------------------------------------------------------------ epilogue: logits = acc + bias
  store_acc_fragment(smem_u32(smem_acc), 64 * wg, acc, warp & 3, lane);
  __syncthreads();
  if (warp < 4) {
    GemmArgs ga{};
    ga.M = h.B; ga.N = h.C; ga.K = 3 * h.D;
    ga.out = h.logits; ga.ldo = h.C; ga.bias = h.bias;
    ga.rowmap_div = 1; ga.rowmap_mul = 0; ga.rowmap_add = 0;
    ga.vec_ok = (h.C % 4) == 0;
    ga.resid = h.logits;
    epilogue_tile<EPI_F32_BIAS>(ga, smem_u32(smem_acc) + (uint32_t)(warp * 32) * kAccLdBytes, smem_stage + warp * kStageWarpBytes,
                                m_blk * HB_M + warp * 32, n_blk * HB_N, 0, HB_N, lane);
  }

  // ------------------------------------------------------------------ ticket: who completes this sample block?
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) {
    const int old = atomicAdd(&h.tickets[m_blk], 1);
    const int last = old == n_blocks - 1;
    if (last) h.tickets[m_blk] = 0;   // ready for the next launch
    *last_flag = last;
  }
  __syncthreads();
  if (!*last_flag) return;
  __threadfence();

  // ------------------------------------------------------------------ softmax, arg-max + centroid, top-k: warp per sample
  const int cpad = (h.C + 3) & ~3;
  const uint32_t sp = smem_u32(smem) + (uint32_t)warp * cpad * 4;   // this warp's probability row (explicit ld/st.shared)
  for (int r = warp; r < HB_M; r += kHeadThreads / 32) {
    const long b = (long)m_blk * HB_M + r;
    if (b >= h.B) break;
    const float* lr = h.logits + b * h.C;
    float m = -INFINITY;
    for (int c0 = 0; c0 < h.C; c0 += 32 * 8) {   // eight independent L2 reads in flight per lane
      float v[8];
#pragma unroll
      for (int u = 0; u < 8; ++u) { const int c = c0 + u * 32 + lane; v[u] = c < h.C ? __ldcg(lr + c) : -INFINITY; }
#pragma unroll
      for (int u = 0; u < 8; ++u) { const int c = c0 + u * 32 + lane; if (c < h.C) { sts_f1(sp + c * 4, v[u]); m = fmaxf(m, v[u]); } }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    float s = 0.f;
    for (int c = lane; c < h.C; c += 32) { const float e = expf(lds_f1(sp + c * 4) - m); sts_f1(sp + c * 4, e); s += e; }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    for (int c = lane; c < h.C; c += 32) { const float p = lds_f1(sp + c * 4) / s; sts_f1(sp + c * 4, p); h.probs[b * h.C + c] = p; }
    __syncwarp();
    for (int j = 0; j < h.k; ++j) {
      float bv = -INFINITY;
      int bi = 0x7fffffff;
      for (int c = lane; c < h.C; c += 32) {
        const float p = lds_f1(sp + c * 4);
        if (p != -1.f && head_better(p, c, bv, bi)) { bv = p; bi = c; }
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        const float ov = __shfl_xor_sync(0xffffffffu, bv, o);
        const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
        if (head_better(ov, oi, bv, bi)) { bv = ov; bi = oi; }
      }
      if (lane == 0) {
        h.topk_val[b * h.k + j] = bv;
        h.topk_idx[b * h.k + j] = bi;
        if (j == 0) {
          h.pred_cell[b] = bi;
          h.pred_lnglat[2 * b] = h.centroids[2 * (long)bi];
          h.pred_lnglat[2 * b + 1] = h.centroids[2 * (long)bi + 1];
        }
        sts_f1(sp + bi * 4, -1.f);   // probabilities are >= 0, so -1 marks "taken"
      }
      __syncwarp();
    }
  }
}

}  // namespace

bool head_fused_supported(int B, int V, int D, int C, int k) {
  return B > 0 && V > 0 && D % HB_K == 0 && C > 0 && C <= kHeadMaxCells && k > 0 && k <= C;
}

size_t head_fused_workspace_bytes(int B) { return (size_t)((B + HB_M - 1) / HB_M) * sizeof(int); }

int head_fused_forward(const float* emb, int B, int V, int D, const void* w3_f16, const float* bias,
                       const double* centroids, int C, int k, void* tickets, float* pooled, float* logits, float* probs,
                       long long* pred_cell, double* pred_lnglat, float* topk_val, long long* topk_idx,
                       cudaStream_t stream) {
  if (!head_fused_supported(B, V, D, C, k)) { set_last_error("head_fused_forward: unsupported shape B=%d V=%d D=%d C=%d k=%d", B, V, D, C, k); return 1; }
  if (reinterpret_cast<uintptr_t>(emb) & 15) { set_last_error("head_fused_forward: emb must be 16-byte aligned"); return 1; }
  CUtensorMap tw;
  if (make_tmap_f16_2d(&tw, w3_f16, C, 3 * (uint64_t)D, 3 * (uint64_t)D, HB_N, HB_K)) return 1;
  const int m_blocks = (B + HB_M - 1) / HB_M, n_blocks = (C + HB_N - 1) / HB_N;
  cudaError_t e = cudaMemsetAsync(tickets, 0, (size_t)m_blocks * sizeof(int), stream);
  if (e != cudaSuccess) { set_last_error("head_fused_forward: memset: %s", cudaGetErrorString(e)); return 1; }
  e = cudaFuncSetAttribute(head_fused_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kHeadSmem);
  if (e != cudaSuccess) { set_last_error("head_fused_forward: cudaFuncSetAttribute: %s", cudaGetErrorString(e)); return 1; }
  HeadArgs h;
  h.emb = emb; h.B = B; h.V = V; h.D = D; h.C = C; h.k = k; h.bias = bias; h.centroids = centroids;
  h.pooled = pooled; h.logits = logits; h.probs = probs; h.pred_cell = pred_cell; h.pred_lnglat = pred_lnglat;
  h.topk_val = topk_val; h.topk_idx = topk_idx; h.tickets = reinterpret_cast<int*>(tickets);
  ProfScope prof("head_fused", stream);
  head_fused_kernel<<<m_blocks * n_blocks, kHeadThreads, kHeadSmem, stream>>>(tw, h);
  e = cudaGetLastError();
  if (e != cudaSuccess) { set_last_error("head_fused launch: %s", cudaGetErrorString(e)); return 1; }
  return 0;
}

}  // namespace pg
