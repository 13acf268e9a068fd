// Persistent warp-specialised wgmma GEMM for sm_90a:  D[M,N] = A[M,K] * W[N,K]^T  (+ epilogue)
//
//   A : fp16 / bf16 row-major [M, K]  (activations, K contiguous  -> K-major wgmma operand)
//   W : fp16 / bf16 row-major [N, K]  (nn.Linear weight layout    -> K-major wgmma operand)
//   or both with the contraction index outermost (GemmProblem::mn_major): MN-major ("transposed") operands
//   accumulate fp32 in registers, epilogue variants in gemm_epilogue.cuh.
//
// Replaces the cuBLAS sgemm calls behind HF CLIPAttention.{q,k,v,out}_proj / CLIPMLP.{fc1,fc2} and the
// cuDNN patch conv reached from reference models/clip_embedder.py:63 and models/super_guessr.py:395,
// and nn.Linear cell_layer at models/super_guessr.py:447.
//
// CTA = 160 threads, 1 CTA / SM, grid = min(#SM, #tiles), output tile 128 x 128:
//   warps 0..3  one warpgroup: per 64-wide K block 2 x 4 wgmma.mma_async m64n128k16 (two 64-row halves), one group in
//               flight while the next is issued; then the accumulators go through a shared-memory tile to the epilogue
//               (each warp 32 rows: bias / activation / residual -> global)
//   warp 4      TMA producer (one lane): global -> 4-stage smem ring, 128B swizzle; it runs ahead into the next tile
//               while the warpgroup is in its epilogue
// K-major problems run the 128 x 256 kernel of gemm_wide.cuh (fp16-output and fp32 residual epilogues whose output rows
// suit a TMA store) or the ping-pong kernel of gemm_pingpong.cu (same tiles and MMAs as this one, two consumer
// warpgroups), unless pg_gemm_set_schedule(1) selects this one for all of them or (2) the ping-pong kernel; MN-major
// operands always run here.
// launch<EPI> below checks the problem and builds the tensor maps for all three.
#include "gemm.h"
#include "gemm_epilogue.cuh"
#include "gemm_pingpong.h"
#include "gemm_wide.h"
#include "ptx.cuh"
#include "prof.h"
#include "tma_host.h"

#include <atomic>
#include <cstdlib>

namespace pg {

// Process-wide kernel choice (pg_gemm_set_schedule): 0 = automatic, 1 = the single-warpgroup kernel for every problem,
// 2 = the ping-pong kernel for every K-major problem.  It exists so that tests can take the single-warpgroup and the
// ping-pong kernels as the bit-exact references of the kernels that replace them, and a benchmark can compare them in one
// process; it is not a tuning knob.  PG_GEMM_SCHEDULE=1 or 2 only sets the initial value, once.
static std::atomic<int> g_gemm_schedule{-1};
static int gemm_schedule() {
  int v = g_gemm_schedule.load(std::memory_order_relaxed);
  if (v < 0) {
    const char* e = getenv("PG_GEMM_SCHEDULE");
    v = (e && (e[0] == '1' || e[0] == '2')) ? e[0] - '0' : 0;
    g_gemm_schedule.store(v, std::memory_order_relaxed);
  }
  return v;
}

int gemm_set_schedule(int mode) {
  if (mode < 0 || mode > 2) { set_last_error("pg_gemm_set_schedule: mode %d not in {0, 1, 2}", mode); return 1; }
  g_gemm_schedule.store(mode, std::memory_order_relaxed);
  return 0;
}

namespace {

constexpr int BLOCK_M = 128;
constexpr int BLOCK_N = kEpiTileN;
constexpr int BLOCK_K = 64;  // 64 halves = 128 bytes = one swizzle atom row
constexpr int kStages = 4;
constexpr int kNumThreads = 160;
constexpr int kProducerWarp = 4;
constexpr int kABytes = BLOCK_M * BLOCK_K * 2;
constexpr int kBBytes = BLOCK_N * BLOCK_K * 2;
constexpr int kStageBytes = kABytes + kBBytes;
constexpr int kSmemBytes = kStages * kStageBytes + kAccTileBytes + 4 * kStageWarpBytes + 1024 /*align slack*/ + 256 /*barriers*/;

template <int EPI, bool BF16, bool MN>
__global__ void __launch_bounds__(kNumThreads, 1)
gemm_f16_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b,
                const GemmArgs args) {
  extern __shared__ uint8_t smem_raw[];
  // 128B-swizzled tiles need 1024-byte alignment.
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* smem_a = smem;
  uint8_t* smem_b = smem + kStages * kABytes;
  uint8_t* smem_acc = smem + kStages * kStageBytes;        // fp32 accumulator tile
  uint8_t* smem_stage = smem_acc + kAccTileBytes;          // epilogue staging, 4 warps
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem_stage + 4 * kStageWarpBytes);
  uint64_t* full_bar = bars;
  uint64_t* empty_bar = bars + kStages;

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;

  const int m_blocks = (args.M + BLOCK_M - 1) / BLOCK_M;
  const int n_blocks = (args.N + BLOCK_N - 1) / BLOCK_N;
  const int num_tiles = m_blocks * n_blocks;
  const int num_kb = (args.K + BLOCK_K - 1) / BLOCK_K;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmap_a);
    tma_prefetch_desc(&tmap_b);
    for (int s = 0; s < kStages; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], 4);  // one arrive per consumer warp
    }
    fence_mbar_init();
  }
  __syncthreads();

  if (warp == kProducerWarp) {
    // ------------------------------------------------------------------ TMA producer
    if (lane == 0) {
      int stage = 0;
      uint32_t phase = 0;
      for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        const int m_blk = tile / n_blocks, n_blk = tile % n_blocks;
        for (int kb = 0; kb < num_kb; ++kb) {
          mbar_wait(&empty_bar[stage], phase ^ 1);
          mbar_arrive_expect_tx(&full_bar[stage], kStageBytes);
          if (!MN) {
            tma_load_2d(smem_a + stage * kABytes, &tmap_a, &full_bar[stage], kb * BLOCK_K, m_blk * BLOCK_M);
            tma_load_2d(smem_b + stage * kBBytes, &tmap_b, &full_bar[stage], kb * BLOCK_K, n_blk * BLOCK_N);
          } else {
            // operand tiles [64 contraction rows x 64 M/N columns] (128 B per row, swizzled): two per operand
#pragma unroll
            for (int c = 0; c < 2; ++c) {
              tma_load_2d(smem_a + stage * kABytes + c * (kABytes / 2), &tmap_a, &full_bar[stage], m_blk * BLOCK_M + c * 64, kb * BLOCK_K);
              tma_load_2d(smem_b + stage * kBBytes + c * (kBBytes / 2), &tmap_b, &full_bar[stage], n_blk * BLOCK_N + c * 64, kb * BLOCK_K);
            }
          }
          if (++stage == kStages) { stage = 0; phase ^= 1; }
        }
      }
    }
    return;
  }

  // -------------------------------------------------------------------- consumer warpgroup
  int stage = 0;
  uint32_t phase = 0;
  const uint32_t acc_s = smem_u32(smem_acc);
  for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
    const int m_blk = tile / n_blocks, n_blk = tile % n_blocks;
    float acc[2][BLOCK_N / 2];
    int prev_stage = -1;
    for (int kb = 0; kb < num_kb; ++kb) {
      mbar_wait(&full_bar[stage], phase);
      const uint32_t a_addr = smem_u32(smem_a + stage * kABytes);
      const uint32_t b_addr = smem_u32(smem_b + stage * kBBytes);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < BLOCK_K / 16; ++k) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {   // rows [64 h, 64 h + 64) of the tile
          uint64_t a_desc, b_desc;
          if (!MN) {
            a_desc = make_smem_desc(a_addr + h * (kABytes / 2) + k * 32, 16, 1024);
            b_desc = make_smem_desc(b_addr + k * 32, 16, 1024);
          } else {   // 16 contraction rows of 128 B per step; the second 64 columns of W are kBBytes / 2 further
            a_desc = make_smem_desc(a_addr + h * (kABytes / 2) + k * 16 * 128, kABytes / 2, 1024);
            b_desc = make_smem_desc(b_addr + k * 16 * 128, kBBytes / 2, 1024);
          }
          if (BF16) wgmma_ss_n128_bf16<MN, MN>(acc[h], a_desc, b_desc, (kb | k) != 0);
          else      wgmma_ss_n128_f16<MN, MN>(acc[h], a_desc, b_desc, (kb | k) != 0);
        }
      }
      wgmma_commit();
      if (prev_stage >= 0) {   // the previous K block's MMAs have retired: hand its smem slot back to the producer
        wgmma_wait<1>();
        if (lane == 0) mbar_arrive(&empty_bar[prev_stage]);
      }
      prev_stage = stage;
      if (++stage == kStages) { stage = 0; phase ^= 1; }
    }
    wgmma_wait<0>();
    if (lane == 0) mbar_arrive(&empty_bar[prev_stage]);

    // accumulators -> shared tile -> epilogue (gemm_epilogue.cuh): warp w takes rows [32 w, 32 w + 32)
    store_acc_fragment(acc_s, 0, acc[0], warp, lane);
    store_acc_fragment(acc_s, 64, acc[1], warp, lane);
    named_barrier<1>(128);
    epilogue_tile<EPI>(args, acc_s + (uint32_t)(warp * 32) * kAccLdBytes, smem_stage + warp * kStageWarpBytes,
                       m_blk * BLOCK_M + warp * 32, n_blk * BLOCK_N, 0, BLOCK_N, lane);
    named_barrier<1>(128);   // the tile is free for the next accumulators
  }
}

template <int EPI, bool BF16, bool MN>
int launch_kernel(const CUtensorMap& ta, const CUtensorMap& tb, const GemmArgs& a, int grid, cudaStream_t stream) {
  auto kern = gemm_f16_kernel<EPI, BF16, MN>;
  static std::atomic<int> attr_set[64];   // per template instantiation and device (the attribute is per context)
  int dev = 0;
  cudaGetDevice(&dev);
  if (dev < 0 || dev >= 64) dev = 0;
  if (!attr_set[dev].load(std::memory_order_acquire)) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemBytes);
    if (e != cudaSuccess) { set_last_error("gemm: cudaFuncSetAttribute: %s", cudaGetErrorString(e)); return 1; }
    attr_set[dev].store(1, std::memory_order_release);
  }
  kern<<<grid, kNumThreads, kSmemBytes, stream>>>(ta, tb, a);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) { set_last_error("gemm launch: %s", cudaGetErrorString(e)); return 1; }
  return 0;
}

template <int EPI>
int launch(const GemmProblem& p, int num_sms, cudaStream_t stream) {
  constexpr bool f16_out = EpiTraits<EPI>::kF16Out || EPI == EPI_BF16_DGELU;   // 2-byte output elements
  const int sched = gemm_schedule();
  // The 128 x 256 kernel stores its output (and loads the residual, stores the fp16 copy) with TMA: row pitch a multiple of
  // 16 bytes for the fp16 output and copy (`out`, `resid` and `aux` are 16-byte aligned, checked by gemm_f16 and below).
  // Otherwise the problem takes the ping-pong kernel, which gives the same bits.
  const bool wide = gemm_wide_epilogue(EPI) && !p.mn_major && sched == 0 && p.ldo % 8 == 0;
  const int block_n = wide ? kWideBlockN : BLOCK_N;
  CUtensorMap ta, tb;
  if (p.mn_major) {   // tensors are [K, M] and [K, N]; box = 64 contraction rows x 64 columns
    if (make_tmap_f16_2d(&ta, p.a, p.K, p.M, p.lda, BLOCK_K, 64)) return 1;
    if (make_tmap_f16_2d(&tb, p.w, p.K, p.N, p.ldw, BLOCK_K, 64)) return 1;
  } else {
    if (make_tmap_f16_2d(&ta, p.a, p.M, p.K, p.lda, BLOCK_M, BLOCK_K)) return 1;
    if (make_tmap_f16_2d(&tb, p.w, p.N, p.K, p.ldw, block_n, BLOCK_K)) return 1;
  }
  GemmArgs a;
  a.M = p.M; a.N = p.N; a.K = p.K; a.out = p.out; a.ldo = p.ldo; a.bias = p.bias;
  a.vec_ok = (p.ldo % (f16_out ? 8 : 4)) == 0;
  a.rowmap_div = p.rowmap_div > 0 ? p.rowmap_div : 1; a.rowmap_mul = p.rowmap_mul; a.rowmap_add = p.rowmap_add;
  a.operand_bf16 = p.operand_bf16 ? 1 : 0;   // A and W of one type: wgmma has no bf16 x fp16 form
  a.resid = p.resid ? p.resid : reinterpret_cast<const float*>(p.out);
  a.aux = p.aux;
  a.mn_major = p.mn_major ? 1 : 0;
  if ((EPI == EPI_BF16_DGELU || EPI == EPI_F16_BIAS_QGELU_SAVE || EPI == EPI_F32_BIAS_RESID_STATS) &&
      (!p.aux || (reinterpret_cast<uintptr_t>(p.aux) & 15))) {
    set_last_error("gemm: this epilogue needs a 16-byte aligned aux buffer"); return 1;
  }
  a.stats = p.stats; a.colsum = p.colsum; a.ln_eps = p.ln_eps; a.stats_slots = 0;
  if (EpiTraits<EPI>::kStats) {
    if (!p.stats || (p.N % 128) || !a.vec_ok || (p.ldo % 8)) { set_last_error("gemm: LayerNorm-producer epilogue needs stats, N %% 128 == 0 and ldo %% 8 == 0"); return 1; }
    a.stats_slots = p.N / 128;
  }
  if (EpiTraits<EPI>::kLn) {
    if (!p.stats || !p.colsum || !p.bias || (p.K % 128) || (p.N % 64) || (reinterpret_cast<uintptr_t>(p.colsum) & 15)) {
      set_last_error("gemm: LayerNorm-consumer epilogue needs stats, a bias, a 16-byte aligned colsum, K %% 128 == 0 and N %% 64 == 0"); return 1;
    }
    a.stats_slots = p.K / 128;
  }
  const int m_blocks = (p.M + BLOCK_M - 1) / BLOCK_M, n_blocks = (p.N + block_n - 1) / block_n;
  const int tiles = m_blocks * n_blocks;
  const int grid = tiles < num_sms ? tiles : num_sms;
  static const char* const kNames[] = {"gemm_f16_bias", "gemm_f16_bias_qgelu", "gemm_f32_bias_resid", "gemm_f32_bias", "gemm_f32_rowmap",
                                       "gemm_bf16_dgelu", "gemm_f16_bias_qgelu_save", "gemm_f32_bias_resid_stats", "gemm_f16_ln_bias",
                                       "gemm_f16_ln_bias_qgelu"};
  ProfScope prof(kNames[EPI], stream);
  // fp16-output and residual problems go to the 128 x 256 kernel (gemm_wide.cuh), other K-major ones to the ping-pong kernel
  // (gemm_pingpong.cu); both sum the same products in the same order as gemm_f16_kernel, so the same bits.  MN-major
  // operands (pg_gemm_tn) stay on gemm_f16_kernel.
  if (wide) {
    // [M, N] with row pitch ldo: fp16 in 64 x 64 boxes, fp32 in 64 x 32 boxes (128-byte rows)
    CUtensorMap tout, tres, taux;
    if (EpiTraits<EPI>::kResid) {
      if (make_tmap_f32_2d(&tout, p.out, p.M, p.N, p.ldo, 64, 32)) return 1;
      if (make_tmap_f32_2d(&tres, a.resid, p.M, p.N, p.ldo, 64, 32)) return 1;
      if (EpiTraits<EPI>::kStats) {
        if (make_tmap_f16_2d(&taux, p.aux, p.M, p.N, p.ldo, 64, 64)) return 1;
      } else {
        taux = tout;
      }
    } else {
      if (make_tmap_f16_2d(&tout, p.out, p.M, p.N, p.ldo, 64, 64)) return 1;
      tres = taux = tout;
    }
    return gemm_wide_launch(EPI, p.operand_bf16 != 0, ta, tb, tout, tres, taux, a, grid, stream);
  }
  if (!p.mn_major && sched != 1) return gemm_pingpong_launch(EPI, p.operand_bf16 != 0, ta, tb, a, grid, stream);
  if (p.mn_major) return p.operand_bf16 ? launch_kernel<EPI, true, true>(ta, tb, a, grid, stream) : launch_kernel<EPI, false, true>(ta, tb, a, grid, stream);
  return p.operand_bf16 ? launch_kernel<EPI, true, false>(ta, tb, a, grid, stream) : launch_kernel<EPI, false, false>(ta, tb, a, grid, stream);
}

}  // namespace

int gemm_f16(const GemmProblem& p, int num_sms, cudaStream_t stream) {
  if (p.M <= 0 || p.N <= 0 || p.K <= 0) return 0;
  if ((p.lda % 8) || (p.ldw % 8)) { set_last_error("gemm: lda/ldw must be multiples of 8 halves (TMA 16B stride)"); return 1; }
  if ((reinterpret_cast<uintptr_t>(p.a) | reinterpret_cast<uintptr_t>(p.w) | reinterpret_cast<uintptr_t>(p.out) |
       reinterpret_cast<uintptr_t>(p.bias)) & 15) {
    set_last_error("gemm: pointers must be 16-byte aligned"); return 1;
  }
  // the epilogues read the residual with 16-byte and the LayerNorm moments with 8-byte vector accesses
  if (reinterpret_cast<uintptr_t>(p.resid) & 15) { set_last_error("gemm: resid must be 16-byte aligned"); return 1; }
  if ((p.epi == EPI_F32_BIAS_RESID_STATS || p.epi == EPI_F16_LN_BIAS || p.epi == EPI_F16_LN_BIAS_QGELU) &&
      (reinterpret_cast<uintptr_t>(p.stats) & 7)) {
    set_last_error("gemm: stats must be 8-byte aligned"); return 1;
  }
  if (p.ldo < p.N) { set_last_error("gemm: ldo %d < N %d", p.ldo, p.N); return 1; }
  if (p.mn_major ? (p.lda < p.M || p.ldw < p.N) : (p.lda < p.K || p.ldw < p.K)) {
    set_last_error("gemm: lda %d / ldw %d shorter than the rows they stride (%s)", p.lda, p.ldw,
                   p.mn_major ? "MN-major: lda >= M, ldw >= N" : "lda >= K, ldw >= K");
    return 1;
  }
  if (num_sms < 1) num_sms = 1;
  // The weight-gradient form takes the shapes pg_gemm_tn documents; its callers transpose and use the K-major form otherwise.
  if (p.mn_major && !(p.N % 256 == 0 && p.M > 128)) { set_last_error("gemm: MN-major operands need N %% 256 == 0 and M > 128"); return 1; }
  switch (p.epi) {
    case EPI_F16_BIAS:              return launch<EPI_F16_BIAS>(p, num_sms, stream);
    case EPI_F16_BIAS_QGELU:        return launch<EPI_F16_BIAS_QGELU>(p, num_sms, stream);
    case EPI_F32_BIAS_RESID:        return launch<EPI_F32_BIAS_RESID>(p, num_sms, stream);
    case EPI_F32_BIAS:              return launch<EPI_F32_BIAS>(p, num_sms, stream);
    case EPI_F32_ROWMAP:            return launch<EPI_F32_ROWMAP>(p, num_sms, stream);
    case EPI_BF16_DGELU:            return launch<EPI_BF16_DGELU>(p, num_sms, stream);
    case EPI_F16_BIAS_QGELU_SAVE:   return launch<EPI_F16_BIAS_QGELU_SAVE>(p, num_sms, stream);
    case EPI_F32_BIAS_RESID_STATS:  return launch<EPI_F32_BIAS_RESID_STATS>(p, num_sms, stream);
    case EPI_F16_LN_BIAS:           return launch<EPI_F16_LN_BIAS>(p, num_sms, stream);
    case EPI_F16_LN_BIAS_QGELU:     return launch<EPI_F16_LN_BIAS_QGELU>(p, num_sms, stream);
    default: set_last_error("gemm: unknown epilogue %d", p.epi); return 1;
  }
}

}  // namespace pg
