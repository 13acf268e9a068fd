// 128 x 256 cooperative wgmma GEMM for sm_90a (K-major operands):  D[M,N] = A[M,K] * W[N,K]^T  (+ epilogue)
//
// The kernel template and its launcher; gemm_wide.cu instantiates the fp16-output epilogues and gemm_wide_resid.cu the
// fp32 residual ones, so each unit compiles (and is checked for spills) on its own.
//
// Runs the fp16-output epilogues that write nothing but the output (qkv and fc1 of the vision tower) and the fp32 residual
// epilogues (out_proj and fc2: EPI_F32_BIAS_RESID, EPI_F32_BIAS_RESID_STATS), see gemm_wide_epilogue.
// The ping-pong kernel (gemm_pingpong.cu) gives each consumer warpgroup its own 128 x 128 tile and issues 2 x 4
// m64n128k16 per 64-wide K block, so every W tile is read from shared memory twice.  Here the two consumer warpgroups share
// one 128 x 256 tile: consumer c owns rows [64 c, 64 c + 64) x 256 columns and issues 4 m64n256k16 per K block.  Per MMA
// FLOP that moves 3/4 of the TMA bytes into shared memory, reads 5/6 of the operand bytes out of it, and fetches 3/4 of
// the bytes from L2.  Every output element is the same k16 steps in the same order as in the other two kernels, and the
// epilogue is epilogue_tile's arithmetic per element, so the outputs are the same bits.
//
// CTA = 384 threads, 1 CTA / SM, grid = min(#SM, #tiles); the CTA's i-th tile is blockIdx.x + i * gridDim.x, row-major
// (m_blk = tile / n_blocks) as in the other kernels:
//   warpgroup 0     producer (24 registers): one lane runs the TMA loads global -> 3-stage ring (A 128 x 64, W 256 x 64,
//                   128B swizzle); for the fp16 output warps 1-3 write each tile's epilogue operands (bias, colsum and
//                   the LayerNorm sums of its rows) into one of two operand buffers, a tile ahead of the consumers
//   warpgroups 1, 2 consumers (240 registers each): both read every stage, so a stage's empty barrier counts their 8 warps
//
// The price is the epilogue overlap that ping-pong buys: both consumers finish a tile together and the tensor cores idle
// during its epilogue.  The epilogue is kept short: it runs on the accumulator fragment in registers, and every global
// access of the tile goes through the TMA unit, issued by one lane of the consumer and asynchronous to the other threads.
//   fp16 output   bias / LayerNorm, quick-GELU, fp16 round to nearest into the consumer's 128B-swizzled staging tile, one
//                 TMA store per 64 x 64 box while the producer already fills the ring for the next tile.  Bias, colsum
//                 and the LayerNorm sums come from the tile's operand buffer, written during the mainloop: the epilogue
//                 does not wait on global memory.
//   fp32 residual the consumer's 64 x 256 part in four 64-column steps.  A step's residual (two 64 x 32 fp32 boxes) comes
//                 in by TMA into one of two step buffers; out = (acc + bias) + resid is written over it and stored by
//                 TMA; the fp16 copy (EPI_F32_BIAS_RESID_STATS) goes through one 64 x 64 fp16 box.  The residual of
//                 steps 0 and 1 is loaded during the tile's mainloop (at its second K block, once the previous tile's
//                 stores have read the buffers), that of step q + 1 at the start of step q as step q - 1's stores drain.
//                 Loads and stores carry the evict_first L2 policy: the residual stream is read and written once and
//                 should not push the A operand out of L2.  The LayerNorm moments are summed in epilogue_tile's order:
//                 a lane pair of the fragment exchanges one fp16 pair, so that each lane holds the 4 consecutive
//                 columns of one of its two rows that epilogue_tile gives one lane.
// The TMA unit clips rows past M and columns past N, and fills the residual's with zeros.
//
// Shared memory (1024 bytes of alignment slack and 256 of mbarriers on top):
//   ring          3 x (16 KB A + 32 KB W)                                                               147 456
//   fp16 output   staging, one per consumer: 64 rows x 256 fp16 columns as four 64 x 64 boxes (8 KB)  2 x 32 768
//                 operand buffers: bias [256], colsum [256] and (s1, s2) [128] fp32                      2 x  3 072
//   fp32 residual one per consumer: 2 step buffers of 64 x 64 fp32 (16 KB) + one 64 x 64 fp16 box        2 x 40 960
// 220 416 and 230 656 bytes of the 232 448 a block may have.
#pragma once
#include "gemm.h"
#include "gemm_epilogue.cuh"
#include "gemm_wide.h"
#include "ptx.cuh"
#include "tma_host.h"

#include <atomic>

namespace pg {

namespace {

constexpr int BLOCK_M = 128;
constexpr int BLOCK_N = kWideBlockN;
constexpr int BLOCK_K = 64;
constexpr int kStages = 3;
constexpr int kNumThreads = 384;
constexpr int kProducerRegs = 24;
constexpr int kConsumerRegs = 240;
static_assert(128 * kProducerRegs + 256 * kConsumerRegs <= 65536, "register budget of one CTA per SM");
constexpr int kABytes = BLOCK_M * BLOCK_K * 2;
constexpr int kBBytes = BLOCK_N * BLOCK_K * 2;
constexpr int kStageBytes = kABytes + kBBytes;
constexpr int kBoxRows = 64, kBoxCols = 64;                // one TMA store: 64 rows x 128 bytes
constexpr int kBoxBytes = kBoxRows * kBoxCols * 2;
constexpr int kOutBytes = (BLOCK_N / kBoxCols) * kBoxBytes;  // one consumer's staging tile
constexpr int kResBoxCols = 32;                              // one fp32 TMA box: 64 rows x 32 columns (128 bytes)
constexpr int kResBoxBytes = kBoxRows * kResBoxCols * 4;
constexpr int kResStepBytes = 2 * kResBoxBytes;             // one 64-column step of the residual / output
constexpr int kResBytes = 2 * kResStepBytes + kBoxBytes;    // one consumer's two step buffers and fp16 box
constexpr int kSteps = BLOCK_N / 64;
// One tile's epilogue operands (fp16 output): bias [256] at 0, colsum [256] at kOpdColsum, the LayerNorm sums (s1, s2) of
// its 128 rows at kOpdLn.
constexpr int kOpdColsum = BLOCK_N * 4, kOpdLn = 2 * BLOCK_N * 4;
constexpr int kOpdBytes = kOpdLn + BLOCK_M * 8;
constexpr int kOpdThreads = 96;   // warps 1-3 of the producer warpgroup write them
template <int EPI>
constexpr int epi_bytes() { return 2 * (EpiTraits<EPI>::kResid ? kResBytes : kOutBytes + kOpdBytes); }
template <int EPI>
constexpr int smem_bytes() { return kStages * kStageBytes + epi_bytes<EPI>() + 1024 /*align slack*/ + 256 /*barriers*/; }
static_assert(smem_bytes<EPI_F32_BIAS_RESID_STATS>() <= 232448 && smem_bytes<EPI_F16_BIAS>() <= 232448,
              "shared memory per block on sm_90");
static_assert(kBoxBytes % 1024 == 0 && kStageBytes % 1024 == 0 && kResBoxBytes % 1024 == 0,
              "128B-swizzled tiles start on 1024-byte boundaries");
constexpr int kConsumerBar = 1;   // + c: the 128 threads of consumer c

// Bias pair of the residual epilogue.  A coherent load (not ld.global.nc, which ptxas may move above a barrier): the
// epilogue's named barriers then keep each step's loads with that step, next to the 128 accumulators.
__device__ __forceinline__ float2 ldg_f2(const float* p) {
  float2 v;
  asm volatile("ld.global.v2.f32 {%0, %1}, [%2];" : "=f"(v.x), "=f"(v.y) : "l"(p));
  return v;
}

__device__ __forceinline__ float2 lds_f2(uint32_t saddr) {
  float2 v;
  asm volatile("ld.shared.v2.f32 {%0, %1}, [%2];" : "=f"(v.x), "=f"(v.y) : "r"(saddr));
  return v;
}
__device__ __forceinline__ void sts_f2(uint32_t saddr, float x, float y) {
  asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(saddr), "f"(x), "f"(y) : "memory");
}

// LayerNorm consumer: out = ln_a * acc + ln_b * colsum + bias, with (ln_a, ln_b) of the A row (= output row) from the
// producer's per-128-column partials, summed as epilogue_tile (gemm_epilogue.cuh) sums them: ln_sums adds up the row's
// partials in order, ln_coeffs turns the two sums into the coefficients.
__device__ __forceinline__ float2 ln_sums(const GemmArgs& args, int row) {
  float s1 = 0.f, s2 = 0.f;
  if (row < args.M) {
    const float2* st = reinterpret_cast<const float2*>(args.stats) + (long)row * args.stats_slots;
    const float2* end = st + args.stats_slots;
#pragma unroll 2
    for (; st < end; ++st) {
      const float2 p = *st;
      s1 += p.x;
      s2 += p.y;
    }
  }
  return make_float2(s1, s2);
}
__device__ __forceinline__ void ln_coeffs(const GemmArgs& args, float s1, float s2, float& ln_a, float& ln_b) {
  const float inv_k = 1.0f / (float)args.K;
  const float mu = s1 * inv_k;
  const float var = fmaxf(s2 * inv_k - mu * mu, 0.f);
  ln_a = rsqrtf(var + args.ln_eps);
  ln_b = -ln_a * mu;
}

// The epilogue operands of one tile (fp16 output) -> its operand buffer at shared address `opd`, by warps 1-3 of the
// producer warpgroup while the consumers still run an earlier tile: warp 3 the bias and colsum of the tile's 256 columns
// (0 past N), warps 1 and 2 the LayerNorm sums (ln_sums) of its rows [0, 64) and [64, 128), one row at a time per lane
// within the producer's 24 registers; the consumers turn them into (ln_a, ln_b) with ln_coeffs.
template <int EPI>
__device__ __forceinline__ void fill_operands(const GemmArgs& args, uint32_t opd, int warp_in_group, int lane, int tile_row0,
                                              int tile_col0) {
  constexpr bool kLn = EpiTraits<EPI>::kLn;
  if (warp_in_group == 3) {
#pragma unroll 2
    for (int i = 0; i < BLOCK_N / 32; ++i) {
      const int j = 32 * i + lane, col = tile_col0 + j;
      float b = 0.f, cs = 0.f;
      if (col < args.N) {
        if (args.bias != nullptr) b = __ldg(args.bias + col);
        if (kLn) cs = __ldg(args.colsum + col);
      }
      sts_f1(opd + 4 * j, b);
      if (kLn) sts_f1(opd + kOpdColsum + 4 * j, cs);
    }
  } else if (kLn) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int r = 64 * (warp_in_group - 1) + 32 * h + lane;
      const float2 s12 = ln_sums(args, tile_row0 + r);
      sts_f2(opd + kOpdLn + 8 * r, s12.x, s12.y);
    }
  }
}

// One consumer warpgroup's epilogue of its 64 x 256 part of the tile.  Thread (warp w, lane l) holds rows r = 16 w + l / 4
// and r + 8 (wgmma.cuh fragment layout), columns 8 j + 2 (l % 4) + {0, 1} for j < 32.  Per element it does exactly what
// epilogue_tile (gemm_epilogue.cuh) does, in the same order.  `opd`: the tile's operand buffer (fill_operands).
template <int EPI>
__device__ __forceinline__ void wide_epilogue(const GemmArgs& args, const float (&acc)[BLOCK_N / 2], uint32_t opd,
                                              const uint8_t* out_tile, const CUtensorMap* tmap_out, int c, int warp_in_group,
                                              int lane, int tile_row0, int tile_col0) {
  constexpr bool kLn = EpiTraits<EPI>::kLn;
  constexpr bool kGelu = (EPI == EPI_F16_BIAS_QGELU || EPI == EPI_F16_LN_BIAS_QGELU);
  const int rbase = 16 * warp_in_group + (lane >> 2);   // this lane's first row within the consumer's 64
  const bool store_lane = (warp_in_group | lane) == 0;
  float ln_a[2] = {1.f, 1.f}, ln_b[2] = {0.f, 0.f};    // of rows rbase + 8 h
  if (kLn) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const float2 s12 = lds_f2(opd + kOpdLn + 8 * (64 * c + rbase + 8 * h));
      ln_coeffs(args, s12.x, s12.y, ln_a[h], ln_b[h]);
    }
  }
  if (store_lane) bulk_wait_group_read<0>();   // the previous tile's stores have read the staging tile
  named_barrier_sync(kConsumerBar + c, 128);
  // 16-byte piece q of staging row r sits at piece slot q ^ (r & 7) (the TMA unit's 128-byte swizzle); rows r and r + 8
  // share r & 7, and the 8 rows of one store instruction hit 8 different slots: no bank conflicts.
  const uint32_t srow = smem_u32(out_tile) + (uint32_t)rbase * 128 + (uint32_t)(lane & 3) * 4;
  const int sw = rbase & 7;
#pragma unroll
  for (int j = 0; j < BLOCK_N / 8; ++j) {
    const uint32_t ocol = opd + (uint32_t)(8 * j + 2 * (lane & 3)) * 4;
    float2 b = make_float2(0.f, 0.f), cs = make_float2(0.f, 0.f);
    if (kLn) {
      cs = lds_f2(ocol + kOpdColsum);
      b = lds_f2(ocol);
    } else if (args.bias != nullptr) {
      b = lds_f2(ocol);
    }
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      float v0 = acc[4 * j + 2 * h], v1 = acc[4 * j + 2 * h + 1];
      if (kLn) {
        v0 = fmaf(ln_a[h], v0, fmaf(ln_b[h], cs.x, b.x));
        v1 = fmaf(ln_a[h], v1, fmaf(ln_b[h], cs.y, b.y));
      } else if (args.bias != nullptr) {
        v0 += b.x;
        v1 += b.y;
      }
      if (kGelu) {
        v0 = quick_gelu(v0);
        v1 = quick_gelu(v1);
      }
      sts_u1(srow + (uint32_t)(j >> 3) * kBoxBytes + (uint32_t)(8 * h) * 128 + (uint32_t)(((j & 7) ^ sw) << 4), pack_half2(v0, v1));
    }
  }
  fence_proxy_async_smem();   // the generic-proxy writes above, before the TMA unit reads them
  named_barrier_sync(kConsumerBar + c, 128);
  if (store_lane && tile_row0 + 64 * c < args.M) {
#pragma unroll
    for (int q = 0; q < BLOCK_N / kBoxCols; ++q)
      if (tile_col0 + q * kBoxCols < args.N)
        tma_store_2d(tmap_out, out_tile + q * kBoxBytes, tile_col0 + q * kBoxCols, tile_row0 + 64 * c);
    bulk_commit_group();
  }
}

// Residual of one 64-column step (global columns [col, col + 64) of the consumer's 64 rows from row0) -> a step buffer, as
// two 64 x 32 fp32 boxes; a box wholly past N is not loaded.  Issued by the consumer's store lane.
__device__ __forceinline__ void load_resid_step(const CUtensorMap* tmap_resid, uint8_t* buf, uint64_t* bar, int col, int row0,
                                                int N, uint64_t pol) {
  const bool two = col + kResBoxCols < N;
  mbar_arrive_expect_tx(bar, two ? 2 * kResBoxBytes : kResBoxBytes);
  tma_load_2d_hint(buf, tmap_resid, bar, col, row0, pol);
  if (two) tma_load_2d_hint(buf + kResBoxBytes, tmap_resid, bar, col + kResBoxCols, row0, pol);
}

// One consumer warpgroup's residual epilogue of its 64 x 256 part of the tile, in four 64-column steps (see the header).
// Per element it does what epilogue_tile does: out = (acc + bias) + resid, the fp16 copy by round to nearest, and per row
// and 128 columns the moments of the fp16 values: lane c16 of epilogue_tile sums the columns 32 ch + 4 c16 + {0..3} over
// ch = 0..3 as (f0 + f1) + (f2 + f3) and fmaf(f0, f0, f1 f1) + fmaf(f2, f2, f3 f3), and the 8 lanes are combined as
// ((p0 + p1) + (p2 + p3)) + ((p4 + p5) + (p6 + p7)).  Here lane l % 4 = t of the fragment holds the columns 8 j + 2 t + {0, 1}
// of rows r and r + 8: lanes t and t ^ 1 swap one fp16 pair, after which lane t holds the 4 columns of c16 = 2 (j % 4) + t / 2
// of row r + 8 (t % 2), and keeps one running sum per j % 4; lanes t and t ^ 2 hold c16 = 2 m and 2 m + 1 of the same row.
// `ebuf` = the consumer's two step buffers and fp16 box; the residual of steps 0 and 1 was loaded during the mainloop.
template <int EPI>
__device__ __forceinline__ void wide_resid_epilogue(const GemmArgs& args, const float (&acc)[BLOCK_N / 2], uint8_t* ebuf,
                                                    uint64_t* res_bar, uint32_t& res_phase, const CUtensorMap* tmap_out,
                                                    const CUtensorMap* tmap_resid, const CUtensorMap* tmap_aux, uint64_t pol,
                                                    int c, int warp_in_group, int lane, int row0, int tile_col0) {
  constexpr bool kStats = EpiTraits<EPI>::kStats;
  const int t = lane & 3;
  const int rbase = 16 * warp_in_group + (lane >> 2);   // this lane's first row within the consumer's 64
  const int sw = rbase & 7;                             // the 128-byte swizzle of rows rbase and rbase + 8
  const bool tile_in_n = tile_col0 + BLOCK_N <= args.N;
  const bool store_lane = (warp_in_group | lane) == 0;
  const uint32_t fbox = smem_u32(ebuf + 2 * kResStepBytes);
  float st_s[4], st_q[4];
#pragma unroll
  for (int q = 0; q < kSteps; ++q) {
    const int col_q = tile_col0 + 64 * q;
    if (col_q >= args.N) break;   // uniform over the warpgroup: the rest of this tile is past N
    const int b = q & 1;
    uint8_t* rbuf = ebuf + b * kResStepBytes;
    if (store_lane && q > 0) {
      bulk_wait_group_read<0>();   // step q - 1's stores have read the fp16 box and step buffer (q + 1) % 2
      if (q + 1 < kSteps && col_q + 64 < args.N)
        load_resid_step(tmap_resid, ebuf + ((q + 1) & 1) * kResStepBytes, &res_bar[(q + 1) & 1], col_q + 64, row0, args.N, pol);
    }
    mbar_wait(&res_bar[b], (res_phase >> b) & 1);
    res_phase ^= 1u << b;
    // fp32 pass: piece (2 (j % 4) + t / 2) of the row in box (j % 8) / 4, 8 bytes in at t % 2; rows r and r + 8 1024 bytes apart
    const uint32_t rrow = smem_u32(rbuf) + (uint32_t)rbase * 128 + (uint32_t)(t & 1) * 8;
    uint32_t h2[8][2];
#pragma unroll
    for (int jj = 0; jj < 8; ++jj) {
      const int j = 8 * q + jj;
      const int col = tile_col0 + 8 * j + 2 * t;
      float2 bv = make_float2(0.f, 0.f);
      if (args.bias != nullptr) {
        if (tile_in_n) {
          bv = ldg_f2(args.bias + col);
        } else {
          if (col < args.N) bv.x = __ldg(args.bias + col);
          if (col + 1 < args.N) bv.y = __ldg(args.bias + col + 1);
        }
      }
      const uint32_t ra = rrow + (uint32_t)(jj >> 2) * kResBoxBytes + (uint32_t)(((2 * (jj & 3) + (t >> 1)) ^ sw) << 4);
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        float v0 = acc[4 * j + 2 * h], v1 = acc[4 * j + 2 * h + 1];
        if (args.bias != nullptr) {
          v0 += bv.x;
          v1 += bv.y;
        }
        const float2 r = lds_f2(ra + 1024 * h);
        v0 += r.x;
        v1 += r.y;
        sts_f2(ra + 1024 * h, v0, v1);
        if (kStats) h2[jj][h] = pack_half2(v0, v1);
      }
    }
    fence_proxy_async_smem();   // the generic-proxy writes above, before the TMA unit reads them
    named_barrier_sync(kConsumerBar + c, 128);   // (and the fp16 box is free: the store lane waited above)
    if (store_lane) {
      tma_store_2d_hint(tmap_out, rbuf, col_q, row0, pol);
      if (col_q + kResBoxCols < args.N) tma_store_2d_hint(tmap_out, rbuf + kResBoxBytes, col_q + kResBoxCols, row0, pol);
      bulk_commit_group();
    }
    if (kStats) {   // N % 128 == 0 (checked at launch): a 256-column tile holds one or two whole 128-column slots
      if ((q & 1) == 0) {
#pragma unroll
        for (int m = 0; m < 4; ++m) st_s[m] = st_q[m] = 0.f;
      }
      const uint32_t frow = fbox + (uint32_t)rbase * 128 + (uint32_t)t * 4;
      const bool odd = (t & 1) != 0;
#pragma unroll
      for (int jj = 0; jj < 8; ++jj) {
        sts_u1(frow + (uint32_t)((jj ^ sw) << 4), h2[jj][0]);
        sts_u1(frow + 1024 + (uint32_t)((jj ^ sw) << 4), h2[jj][1]);
        const uint32_t mine = odd ? h2[jj][1] : h2[jj][0];
        const uint32_t other = __shfl_xor_sync(0xffffffffu, odd ? h2[jj][0] : h2[jj][1], 1);
        const uint32_t lo = odd ? other : mine, hi = odd ? mine : other;
        const float2 f01 = __half22float2(*reinterpret_cast<const __half2*>(&lo));
        const float2 f23 = __half22float2(*reinterpret_cast<const __half2*>(&hi));
        st_s[jj & 3] += (f01.x + f01.y) + (f23.x + f23.y);
        st_q[jj & 3] += fmaf(f01.x, f01.x, f01.y * f01.y) + fmaf(f23.x, f23.x, f23.y * f23.y);
      }
      fence_proxy_async_smem();
      named_barrier_sync(kConsumerBar + c, 128);
      if (store_lane) {
        tma_store_2d_hint(tmap_aux, ebuf + 2 * kResStepBytes, col_q, row0, pol);
        bulk_commit_group();
      }
      if (q & 1) {   // 128 columns complete: combine the 8 column groups of each row, publish
        float u[4], w[4];
#pragma unroll
        for (int m = 0; m < 4; ++m) {
          u[m] = st_s[m] + __shfl_xor_sync(0xffffffffu, st_s[m], 2);
          w[m] = st_q[m] + __shfl_xor_sync(0xffffffffu, st_q[m], 2);
        }
        const int row = row0 + rbase + 8 * (t & 1);
        if (t < 2 && row < args.M)
          reinterpret_cast<float2*>(args.stats)[(long)row * args.stats_slots + (col_q >> 7)] =
              make_float2((u[0] + u[1]) + (u[2] + u[3]), (w[0] + w[1]) + (w[2] + w[3]));
      }
    }
  }
}

template <int EPI, bool BF16>
__global__ void __launch_bounds__(kNumThreads, 1)
gemm_wide_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b,
                 const __grid_constant__ CUtensorMap tmap_out, const __grid_constant__ CUtensorMap tmap_resid,
                 const __grid_constant__ CUtensorMap tmap_aux, const GemmArgs args) {
  constexpr bool kResid = EpiTraits<EPI>::kResid;
  extern __shared__ uint8_t smem_raw[];
  // 128B-swizzled tiles need 1024-byte alignment.
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* smem_a = smem;
  uint8_t* smem_b = smem + kStages * kABytes;
  uint8_t* smem_out = smem + kStages * kStageBytes;   // the consumers' staging tiles / residual buffers
  uint8_t* smem_opd = smem_out + 2 * kOutBytes;       // fp16 output: the two operand buffers
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem_out + epi_bytes<EPI>());
  uint64_t* full_bar = bars;
  uint64_t* empty_bar = bars + kStages;
  uint64_t* res_bar = bars + 2 * kStages;   // + 2 c + b: consumer c's step buffer b is loaded
  uint64_t* opd_full = bars + 2 * kStages;  // + b: operand buffer b is written (fp16 output)
  uint64_t* opd_empty = opd_full + 2;       // + b: both consumers have read it

  const int wg = threadIdx.x >> 7;
  const int warp_in_group = (threadIdx.x >> 5) & 3;
  const int lane = threadIdx.x & 31;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmap_a);
    tma_prefetch_desc(&tmap_b);
    tma_prefetch_desc(&tmap_out);
    if (kResid) {
      tma_prefetch_desc(&tmap_resid);
      if (EpiTraits<EPI>::kStats) tma_prefetch_desc(&tmap_aux);
    }
    for (int s = 0; s < kStages; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], 8);  // one arrive per warp of both consumers
    }
    if (kResid)
      for (int i = 0; i < 4; ++i) mbar_init(&res_bar[i], 1);   // the store lane's arrive.expect_tx
    else
      for (int b = 0; b < 2; ++b) {
        mbar_init(&opd_full[b], kOpdThreads);
        mbar_init(&opd_empty[b], 2);   // the store lane of each consumer
      }
    fence_mbar_init();
  }
  __syncthreads();

  if (wg == 0) {
    // ------------------------------------------------------------------ TMA producer
    setmaxnreg_dec<kProducerRegs>();
    // (the tile counts are computed after setmaxnreg by each role: a value live across it is spilled)
    const int n_blocks = (args.N + BLOCK_N - 1) / BLOCK_N;
    const int num_tiles = (args.M + BLOCK_M - 1) / BLOCK_M * n_blocks;
    const int num_kb = (args.K + BLOCK_K - 1) / BLOCK_K;
    if (threadIdx.x == 0) {
      int stage = 0;
      uint32_t phase = 0;
      for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        const int m_blk = tile / n_blocks, n_blk = tile % n_blocks;
        for (int kb = 0; kb < num_kb; ++kb) {
          mbar_wait(&empty_bar[stage], phase ^ 1);
          mbar_arrive_expect_tx(&full_bar[stage], kStageBytes);
          tma_load_2d(smem_a + stage * kABytes, &tmap_a, &full_bar[stage], kb * BLOCK_K, m_blk * BLOCK_M);
          tma_load_2d(smem_b + stage * kBBytes, &tmap_b, &full_bar[stage], kb * BLOCK_K, n_blk * BLOCK_N);
          if (++stage == kStages) { stage = 0; phase ^= 1; }
        }
      }
    } else if (!kResid && warp_in_group > 0) {
      // the epilogue operands, double-buffered: tile i's are written while the consumers run tile i - 1
      // (shared-window addresses: generic pointers would take two of the 24 registers each)
      const uint32_t opd_s = smem_u32(smem_opd), full_s = smem_u32(opd_full), empty_s = smem_u32(opd_empty);
      for (uint32_t it = 0;; ++it) {
        const int tile = blockIdx.x + it * gridDim.x;
        if (tile >= num_tiles) break;
        const uint32_t b = it & 1;
        mbar_wait(empty_s + 8 * b, ((it >> 1) & 1) ^ 1);
        fill_operands<EPI>(args, opd_s + b * kOpdBytes, warp_in_group, lane, tile / n_blocks * BLOCK_M, tile % n_blocks * BLOCK_N);
        mbar_arrive(full_s + 8 * b);
      }
    }
    return;
  }

  // -------------------------------------------------------------------- consumer warpgroups
  setmaxnreg_inc<kConsumerRegs>();
  const int n_blocks = (args.N + BLOCK_N - 1) / BLOCK_N;
  const int num_tiles = (args.M + BLOCK_M - 1) / BLOCK_M * n_blocks;
  const int num_kb = (args.K + BLOCK_K - 1) / BLOCK_K;
  const int c = wg - 1;
  uint8_t* out_tile = smem_out + c * (kResid ? kResBytes : kOutBytes);   // staging tile / residual buffers
  const bool store_lane = (warp_in_group | lane) == 0;
  const uint64_t pol = kResid ? l2_policy_evict_first() : 0;
  const int resid_kb = num_kb > 1 ? 1 : 0;   // the K block after which steps 0 and 1 of the residual are loaded
  uint32_t res_phase = 0;
  int stage = 0;
  uint32_t phase = 0;
  uint32_t it = 0;   // the CTA's tile count
  for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x, ++it) {
    const int m_blk = tile / n_blocks, n_blk = tile % n_blocks;
    const int row0 = m_blk * BLOCK_M + 64 * c;   // the consumer's first row
    // The first MMA of the tile overwrites the accumulators (scale-d 0); defining them here ends their live range at the
    // previous tile's epilogue.
    float acc[BLOCK_N / 2];
#pragma unroll
    for (int i = 0; i < BLOCK_N / 2; ++i) acc[i] = 0.f;
    int prev_stage = -1;
    for (int kb = 0; kb < num_kb; ++kb) {
      mbar_wait(&full_bar[stage], phase);
      const uint32_t a_addr = smem_u32(smem_a + stage * kABytes + c * (kABytes / 2));   // rows [64 c, 64 c + 64) of the tile
      const uint32_t b_addr = smem_u32(smem_b + stage * kBBytes);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < BLOCK_K / 16; ++k) {
        const uint64_t a_desc = make_smem_desc(a_addr + k * 32, 16, 1024);
        const uint64_t b_desc = make_smem_desc(b_addr + k * 32, 16, 1024);
        if (BF16) wgmma_ss_n256_bf16<0, 0>(acc, a_desc, b_desc, (kb | k) != 0);
        else      wgmma_ss_n256_f16<0, 0>(acc, a_desc, b_desc, (kb | k) != 0);
      }
      wgmma_commit();
      if (prev_stage >= 0) {   // the previous K block's MMAs have retired: this warp is done with its smem slot
        wgmma_wait<1>();
        if (lane == 0) mbar_arrive(&empty_bar[prev_stage]);
      }
      // one K block's MMAs in flight: the store lane waits until the previous tile's stores have read the residual buffers,
      // then loads this tile's first two steps into them
      if (kResid && kb == resid_kb && store_lane && row0 < args.M) {
        bulk_wait_group_read<0>();
#pragma unroll
        for (int q = 0; q < 2; ++q)
          if (n_blk * BLOCK_N + 64 * q < args.N)
            load_resid_step(&tmap_resid, out_tile + q * kResStepBytes, &res_bar[2 * c + q], n_blk * BLOCK_N + 64 * q, row0,
                            args.N, pol);
      }
      prev_stage = stage;
      if (++stage == kStages) { stage = 0; phase ^= 1; }
    }
    wgmma_wait<0>();
    if (lane == 0) mbar_arrive(&empty_bar[prev_stage]);

    if (kResid) {
      if (row0 < args.M)   // uniform over the warpgroup; a consumer wholly past M has nothing to load or store
        wide_resid_epilogue<EPI>(args, acc, out_tile, res_bar + 2 * c, res_phase, &tmap_out, &tmap_resid, &tmap_aux, pol, c,
                                 warp_in_group, lane, row0, n_blk * BLOCK_N);
    } else {
      const int b = it & 1;
      mbar_wait(&opd_full[b], (it >> 1) & 1);   // written during the mainloop, or earlier
      wide_epilogue<EPI>(args, acc, smem_u32(smem_opd + b * kOpdBytes), out_tile, &tmap_out, c, warp_in_group, lane,
                         m_blk * BLOCK_M, n_blk * BLOCK_N);
      if (store_lane) mbar_arrive(&opd_empty[b]);   // after the epilogue's last barrier: the warpgroup is done reading
    }
  }
  if (store_lane) bulk_wait_group<0>();   // the last tile's stores are complete before the CTA exits
}

template <int EPI, bool BF16>
int launch_kernel(const CUtensorMap& ta, const CUtensorMap& tb, const CUtensorMap& tout, const CUtensorMap& tres,
                  const CUtensorMap& taux, const GemmArgs& a, int grid, cudaStream_t stream) {
  constexpr int kSmemBytes = smem_bytes<EPI>();
  auto kern = gemm_wide_kernel<EPI, BF16>;
  static std::atomic<int> attr_set[64];   // per template instantiation and device (the attribute is per context)
  int dev = 0;
  cudaGetDevice(&dev);
  if (dev < 0 || dev >= 64) dev = 0;
  if (!attr_set[dev].load(std::memory_order_acquire)) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemBytes);
    if (e != cudaSuccess) { set_last_error("gemm: cudaFuncSetAttribute: %s", cudaGetErrorString(e)); return 1; }
    attr_set[dev].store(1, std::memory_order_release);
  }
  kern<<<grid, kNumThreads, kSmemBytes, stream>>>(ta, tb, tout, tres, taux, a);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) { set_last_error("gemm launch: %s", cudaGetErrorString(e)); return 1; }
  return 0;
}

template <int EPI>
int launch(bool bf16, const CUtensorMap& ta, const CUtensorMap& tb, const CUtensorMap& tout, const CUtensorMap& tres,
           const CUtensorMap& taux, const GemmArgs& a, int grid, cudaStream_t stream) {
  return bf16 ? launch_kernel<EPI, true>(ta, tb, tout, tres, taux, a, grid, stream)
              : launch_kernel<EPI, false>(ta, tb, tout, tres, taux, a, grid, stream);
}

}  // namespace

// The residual epilogues' launcher (gemm_wide_resid.cu); gemm_wide_launch forwards EPI_F32_BIAS_RESID(_STATS) to it.
int gemm_wide_resid_launch(int epi, bool bf16, const CUtensorMap& ta, const CUtensorMap& tb, const CUtensorMap& tout,
                           const CUtensorMap& tres, const CUtensorMap& taux, const GemmArgs& args, int grid, cudaStream_t stream);

}  // namespace pg
