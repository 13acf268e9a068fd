// Ping-pong persistent wgmma GEMM for sm_90a (K-major operands):  D[M,N] = A[M,K] * W[N,K]^T  (+ epilogue)
//
// Same problem, tile (128 x 128 x 64), operand ring and MMA sequence as gemm_f16_kernel (gemm_wgmma.cu), so the fp32
// accumulators and every output are the same bits; what changes is when the epilogue runs.  There one consumer warpgroup
// finishes a tile's epilogue before it issues the next tile's MMAs, and the tensor cores idle meanwhile.  Here two consumer
// warpgroups take the CTA's tiles in turn, and one runs its epilogue while the other runs its mainloop.
//
// CTA = 384 threads, 1 CTA / SM, grid = min(#SM, #tiles); the CTA's i-th tile is blockIdx.x + i * gridDim.x:
//   warpgroup 0     TMA producer (one lane, 24 registers): global -> 4-stage smem ring, 128B swizzle, tiles in CTA order
//   warpgroups 1, 2 consumers (240 registers each): consumer c takes the tiles with i % 2 == c.  Their mainloops strictly
//                   alternate (named barriers 3 and 4), so they read the ring in the order the producer fills it.
//
// Shared memory (201 984 bytes of the 232 448 a block may have):
//   ring        4 x (16 KB A + 16 KB W)                                      131 072
//   2 x buffer  one per consumer: 128 rows x 64 fp32 columns, rows padded to 68 floats (272 B), 34 816 each
//   slack       1024 (1024-byte alignment of the swizzled ring) + 256 (mbarriers)
// A full padded fp32 tile per consumer (2 x 67.6 KB) does not fit beside the ring, so each consumer drains its tile in two
// 64-column halves through its buffer.  The epilogue's per-warp staging (32 rows x 128 B) lives in the buffer too: a chunk
// is staged at the columns it was just read from, so the staging rows have the buffer's 272-byte pitch, which already keeps
// both the row-per-lane writes and the coalesced row-segment reads free of bank conflicts (no XOR swizzle needed).
// The epilogue (pp_chunk) does per chunk exactly the arithmetic of epilogue_tile (gemm_epilogue.cuh) in the same order;
// the LayerNorm-producer moments are carried across the two halves, so they are summed in the same order too.
#include "gemm.h"
#include "gemm_epilogue.cuh"
#include "gemm_pingpong.h"
#include "ptx.cuh"
#include "tma_host.h"

#include <atomic>

namespace pg {

namespace {

constexpr int BLOCK_M = 128;
constexpr int BLOCK_N = kEpiTileN;
constexpr int BLOCK_K = 64;
constexpr int kStages = 4;
constexpr int kNumThreads = 384;
constexpr int kProducerRegs = 24;
constexpr int kConsumerRegs = 240;
static_assert(128 * kProducerRegs + 256 * kConsumerRegs <= 65536, "register budget of one CTA per SM");
constexpr int kABytes = BLOCK_M * BLOCK_K * 2;
constexpr int kBBytes = BLOCK_N * BLOCK_K * 2;
constexpr int kStageBytes = kABytes + kBBytes;
constexpr int kHalfN = BLOCK_N / 2;
constexpr int kHalfLdBytes = (kHalfN + 4) * 4;
constexpr int kHalfBytes = BLOCK_M * kHalfLdBytes;
constexpr int kSmemBytes = kStages * kStageBytes + 2 * kHalfBytes + 1024 /*align slack*/ + 256 /*barriers*/;
static_assert(kSmemBytes <= 232448, "shared memory per block on sm_90");
constexpr int kConsumerBar = 1;   // + c: the 128 threads of consumer c
constexpr int kOrderBar = 3;      // + c: consumer c may start its next mainloop

// Columns [64 HALF, 64 HALF + 64) of the warpgroup's accumulators (wgmma.cuh fragment layout) -> the consumer's buffer.
template <int HALF>
__device__ __forceinline__ void store_acc_half(uint32_t buf_s, const float (&acc)[2][BLOCK_N / 2], int warp_in_group, int lane) {
#pragma unroll
  for (int blk = 0; blk < 2; ++blk) {
    const uint32_t r0 = buf_s + (uint32_t)(64 * blk + 16 * warp_in_group + (lane >> 2)) * kHalfLdBytes + (uint32_t)(lane & 3) * 8;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int jj = 8 * HALF + j;
      asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(r0 + j * 32), "f"(acc[blk][4 * jj]), "f"(acc[blk][4 * jj + 1]) : "memory");
      asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(r0 + 8 * kHalfLdBytes + j * 32), "f"(acc[blk][4 * jj + 2]),
                   "f"(acc[blk][4 * jj + 3]) : "memory");
    }
  }
}

// State one epilogue warp carries from chunk to chunk of a tile.
struct PpEpiState {
  float4 res[8];                // residual pieces of this chunk
  float st_s[8], st_q[8];       // LayerNorm producer: running (sum, sum of squares) per row piece of this lane
  float ln_a, ln_b;             // LayerNorm consumer: out = ln_a * acc + ln_b * colsum + bias
  uint64_t pol_stream;
};

// One chunk (CHUNK tile columns starting at c0) of one warp's 32 rows, with epilogue_tile's arithmetic per element.  The
// accumulators come from the half buffer (`wbuf` = this warp's first row, `cl` = the chunk's column in the buffer).  Each
// lane streams its row 16 output bytes at a time: read the accumulators, bias / LayerNorm / activation, and write the
// packed piece back over bytes of the row it has already read (the staging); then the coalesced phase as in epilogue_tile.
// EPI_F16_BIAS_QGELU_SAVE keeps both the pre-activation and the output: piece p's 32 bytes hold the two 16-byte pieces.
template <int EPI>
__device__ __forceinline__ void pp_chunk(const GemmArgs& args, PpEpiState& s, uint32_t wbuf, int cl, int c0, int warp_row0,
                                         int tile_col0, int lane) {
  constexpr bool kF16Out = EpiTraits<EPI>::kF16Out;
  constexpr int CHUNK = EpiTraits<EPI>::CHUNK;
  constexpr int kElt = EpiTraits<EPI>::kElt;
  constexpr bool kResid = EpiTraits<EPI>::kResid;
  constexpr bool kStats = EpiTraits<EPI>::kStats;
  constexpr bool kLn = EpiTraits<EPI>::kLn;
  constexpr bool kDgelu = (EPI == EPI_BF16_DGELU);
  constexpr bool kSave = (EPI == EPI_F16_BIAS_QGELU_SAVE);
  constexpr bool kGelu = (EPI == EPI_F16_BIAS_QGELU || EPI == EPI_F16_LN_BIAS_QGELU || kSave);
  constexpr int kPc = kF16Out ? 8 : 4;   // tile columns per 16-byte output piece
  const int sub = lane >> 3, c16 = lane & 7;
  const int col0 = tile_col0 + c0;
  const bool in_n = (col0 + CHUNK <= args.N);
  const bool fast = in_n && args.vec_ok;
  const uint32_t srow = wbuf + (uint32_t)lane * kHalfLdBytes + (uint32_t)cl * 4;   // this lane's row: accumulators, staging
  const uint32_t stage_s = wbuf + (uint32_t)cl * 4;                                   // staging row rr at + rr * kHalfLdBytes
  // this chunk's residual pieces, issued before the streaming pass so that their latency hides behind it
  if (kResid && fast) load_residual<EPI>(args, s.res, warp_row0, col0, lane, s.pol_stream);
  uint2 aux_u[8];
  if (kDgelu && fast) {   // this lane's pre-activation pieces for the coalesced phase, issued before the staging work
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const int grow = warp_row0 + i * 4 + sub;
      aux_u[i] = make_uint2(0u, 0u);
      if (grow < args.M)
        aux_u[i] = *reinterpret_cast<const uint2*>(reinterpret_cast<const __half*>(args.aux) + (long)grow * args.ldo + col0 + c16 * 4);
    }
  }
  // ragged N tail / unaligned rows: this lane's row goes out with per-element stores
  const int row = warp_row0 + lane;
  long orow = row;
  if (EPI == EPI_F32_ROWMAP) orow = (long)args.rowmap_mul * (row / args.rowmap_div) + (row % args.rowmap_div) + args.rowmap_add;
  __syncwarp();
#pragma unroll
  for (int p = 0; p < CHUNK / kPc; ++p) {
    const int pc = col0 + p * kPc;   // global column of v[0]
    float v[kPc];
#pragma unroll
    for (int q = 0; q < kPc / 4; ++q) {
      const float4 t = lds_f4(srow + (uint32_t)(p * kPc + 4 * q) * 4);
      v[4 * q + 0] = t.x; v[4 * q + 1] = t.y; v[4 * q + 2] = t.z; v[4 * q + 3] = t.w;
    }
    if (kLn) {   // LayerNorm folded: rstd * acc + (-rstd * mu) * colsum + bias (N % 64 == 0 and bias != nullptr: checked at launch)
#pragma unroll
      for (int q = 0; q < kPc / 4; ++q) {
        const float4 cs = __ldg(reinterpret_cast<const float4*>(args.colsum + pc) + q);
        const float4 b = __ldg(reinterpret_cast<const float4*>(args.bias + pc) + q);
        v[4 * q + 0] = fmaf(s.ln_a, v[4 * q + 0], fmaf(s.ln_b, cs.x, b.x));
        v[4 * q + 1] = fmaf(s.ln_a, v[4 * q + 1], fmaf(s.ln_b, cs.y, b.y));
        v[4 * q + 2] = fmaf(s.ln_a, v[4 * q + 2], fmaf(s.ln_b, cs.z, b.z));
        v[4 * q + 3] = fmaf(s.ln_a, v[4 * q + 3], fmaf(s.ln_b, cs.w, b.w));
      }
    }
    if (!kLn && args.bias != nullptr) {
      if (in_n) {
#pragma unroll
        for (int q = 0; q < kPc / 4; ++q) {
          const float4 b = __ldg(reinterpret_cast<const float4*>(args.bias + pc) + q);
          v[4 * q + 0] += b.x; v[4 * q + 1] += b.y; v[4 * q + 2] += b.z; v[4 * q + 3] += b.w;
        }
      } else {
#pragma unroll
        for (int i = 0; i < kPc; ++i)
          if (pc + i < args.N) v[i] += __ldg(args.bias + pc + i);
      }
    }
    if (kSave) {   // keep the pre-activation (fp16) for the backward pass
      if (fast) {
        sts_u4(srow + (p << 5), make_uint4(pack_half2(v[0], v[1]), pack_half2(v[2], v[3]), pack_half2(v[4], v[5]), pack_half2(v[6], v[7])));
      } else if (row < args.M) {
        __half* o = reinterpret_cast<__half*>(args.aux) + (long)row * args.ldo + pc;
#pragma unroll
        for (int i = 0; i < kPc; ++i)
          if (pc + i < args.N) o[i] = __float2half_rn(v[i]);
      }
    }
    if (kGelu) {
#pragma unroll
      for (int i = 0; i < kPc; ++i) v[i] = quick_gelu(v[i]);
    }
    if (fast) {
      uint4 pk;
      if (kF16Out) {
        pk = make_uint4(pack_half2(v[0], v[1]), pack_half2(v[2], v[3]), pack_half2(v[4], v[5]), pack_half2(v[6], v[7]));
      } else {
        pk = make_uint4(__float_as_uint(v[0]), __float_as_uint(v[1]), __float_as_uint(v[2]), __float_as_uint(v[3]));
      }
      sts_u4(srow + (kSave ? (p << 5) + 16 : (p << 4)), pk);
    } else if (row < args.M) {
      if (kF16Out) {
        __half* o = reinterpret_cast<__half*>(args.out) + orow * args.ldo + pc;
#pragma unroll
        for (int i = 0; i < kPc; ++i)
          if (pc + i < args.N) o[i] = __float2half_rn(v[i]);
      } else if (kDgelu) {
        __nv_bfloat16* o = reinterpret_cast<__nv_bfloat16*>(args.out) + orow * args.ldo + pc;
        const __half* u = reinterpret_cast<const __half*>(args.aux) + orow * args.ldo + pc;
#pragma unroll
        for (int i = 0; i < kPc; ++i)
          if (pc + i < args.N) o[i] = __float2bfloat16_rn(v[i] * quick_gelu_grad(__half2float(u[i])));
      } else {
        float* o = reinterpret_cast<float*>(args.out) + orow * args.ldo + pc;
#pragma unroll
        for (int i = 0; i < kPc; ++i)
          if (pc + i < args.N) {
            float x = v[i];
            if (kResid) x += args.resid[orow * args.ldo + pc + i];
            o[i] = x;
          }
      }
    }
  }
  if (fast) {
    __syncwarp();
    if (kSave) {   // coalesced store of the pre-activation to aux
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const int rr = i * 4 + sub;
        const int grow = warp_row0 + rr;
        if (grow < args.M)
          *reinterpret_cast<uint4*>(reinterpret_cast<uint8_t*>(args.aux) + ((long)grow * args.ldo + col0) * 2 + c16 * 16) =
              lds_u4(stage_s + rr * kHalfLdBytes + (c16 << 5));
      }
    }
    // ---- coalesced global phase: 8 lanes cover one 128-byte row segment (4 rows per instruction)
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const int rr = i * 4 + sub;
      const int grow = warp_row0 + rr;
      if (grow < args.M) {
        uint4 val = lds_u4(stage_s + rr * kHalfLdBytes + (kSave ? (c16 << 5) + 16 : (c16 << 4)));
        long grow_o = grow;
        if (EPI == EPI_F32_ROWMAP)
          grow_o = (long)args.rowmap_mul * (grow / args.rowmap_div) + (grow % args.rowmap_div) + args.rowmap_add;
        if (kDgelu) {   // 4 fp32 gradients x gelu'(u) -> 4 bf16 (8 bytes per lane, 64 contiguous bytes per row segment)
          const float2 u01 = __half22float2(*reinterpret_cast<const __half2*>(&aux_u[i].x));
          const float2 u23 = __half22float2(*reinterpret_cast<const __half2*>(&aux_u[i].y));
          uint2 o;
          o.x = pack_bf16x2_rn(__uint_as_float(val.x) * quick_gelu_grad(u01.x), __uint_as_float(val.y) * quick_gelu_grad(u01.y));
          o.y = pack_bf16x2_rn(__uint_as_float(val.z) * quick_gelu_grad(u23.x), __uint_as_float(val.w) * quick_gelu_grad(u23.y));
          *reinterpret_cast<uint2*>(reinterpret_cast<uint8_t*>(args.out) + (grow_o * args.ldo + col0) * 2 + c16 * 8) = o;
          continue;
        }
        uint8_t* gp = reinterpret_cast<uint8_t*>(args.out) + (grow_o * args.ldo + col0) * kElt + c16 * 16;
        if (kResid) {
          val.x = __float_as_uint(__uint_as_float(val.x) + s.res[i].x);
          val.y = __float_as_uint(__uint_as_float(val.y) + s.res[i].y);
          val.z = __float_as_uint(__uint_as_float(val.z) + s.res[i].z);
          val.w = __float_as_uint(__uint_as_float(val.w) + s.res[i].w);
          stg_u4_hint(gp, val, s.pol_stream);
        } else {
          *reinterpret_cast<uint4*>(gp) = val;
        }
        if (kStats) {   // fp16 copy of the new residual values (the next GEMM's A operand) and their moments
          const __half2 h01 = __floats2half2_rn(__uint_as_float(val.x), __uint_as_float(val.y));
          const __half2 h23 = __floats2half2_rn(__uint_as_float(val.z), __uint_as_float(val.w));
          uint2 hv;
          hv.x = *reinterpret_cast<const uint32_t*>(&h01);
          hv.y = *reinterpret_cast<const uint32_t*>(&h23);
          stg_u2_hint(reinterpret_cast<uint8_t*>(args.aux) + (grow_o * args.ldo + col0) * 2 + c16 * 8, hv, s.pol_stream);
          const float2 f01 = __half22float2(h01), f23 = __half22float2(h23);
          s.st_s[i] += (f01.x + f01.y) + (f23.x + f23.y);
          s.st_q[i] += fmaf(f01.x, f01.x, f01.y * f01.y) + fmaf(f23.x, f23.x, f23.y * f23.y);
        }
      }
    }
  }
  if (kStats && ((col0 + CHUNK) & 127) == 0) {   // 128 columns complete: combine the 8 lanes of each row, publish
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      float a = s.st_s[i], b = s.st_q[i];
#pragma unroll
      for (int o = 1; o < 8; o <<= 1) {
        a += __shfl_xor_sync(0xffffffffu, a, o);
        b += __shfl_xor_sync(0xffffffffu, b, o);
      }
      const int grow = warp_row0 + i * 4 + sub;
      if (c16 == 0 && grow < args.M)
        reinterpret_cast<float2*>(args.stats)[(long)grow * args.stats_slots + (col0 >> 7)] = make_float2(a, b);
      s.st_s[i] = s.st_q[i] = 0.f;
    }
  }
}

// One consumer warpgroup's epilogue of one tile: warp w takes rows [32 w, 32 w + 32), the two column halves in turn.
template <int EPI>
__device__ __forceinline__ void pp_epilogue(const GemmArgs& args, const float (&acc)[2][BLOCK_N / 2], uint32_t buf_s, int bar_id,
                                            int warp_in_group, int lane, int tile_row0, int tile_col0) {
  constexpr int CHUNK = EpiTraits<EPI>::CHUNK;
  const int warp_row0 = tile_row0 + 32 * warp_in_group;
  const uint32_t wbuf = buf_s + (uint32_t)(32 * warp_in_group) * kHalfLdBytes;
  PpEpiState s;
  s.pol_stream = EpiTraits<EPI>::kResid ? l2_policy_evict_first() : 0;
  s.ln_a = 1.f; s.ln_b = 0.f;
  if (EpiTraits<EPI>::kLn) {   // statistics of this thread's A row (= output row) from the producer's per-128-column partials
    const int row = warp_row0 + lane;
    float s1 = 0.f, s2 = 0.f;
    if (row < args.M) {
      const float2* st = reinterpret_cast<const float2*>(args.stats) + (long)row * args.stats_slots;
      for (int k = 0; k < args.stats_slots; ++k) {
        const float2 p = st[k];
        s1 += p.x;
        s2 += p.y;
      }
    }
    const float inv_k = 1.0f / (float)args.K;
    const float mu = s1 * inv_k;
    const float var = fmaxf(s2 * inv_k - mu * mu, 0.f);
    s.ln_a = rsqrtf(var + args.ln_eps);
    s.ln_b = -s.ln_a * mu;
  }
  if (EpiTraits<EPI>::kStats) {
#pragma unroll
    for (int i = 0; i < 8; ++i) s.st_s[i] = s.st_q[i] = 0.f;
  }

  named_barrier_sync(bar_id, 128);   // the buffer is free: every warp is done with the previous tile
  store_acc_half<0>(buf_s, acc, warp_in_group, lane);
  named_barrier_sync(bar_id, 128);
#pragma unroll 1
  for (int c0 = 0; c0 < kHalfN; c0 += CHUNK) {
    if (tile_col0 + c0 >= args.N) break;   // uniform over the warpgroup: the rest of this tile is past N
    pp_chunk<EPI>(args, s, wbuf, c0, c0, warp_row0, tile_col0, lane);
  }
  if (tile_col0 + kHalfN >= args.N) return;   // uniform over the warpgroup
  named_barrier_sync(bar_id, 128);
  store_acc_half<1>(buf_s, acc, warp_in_group, lane);
  named_barrier_sync(bar_id, 128);
#pragma unroll 1
  for (int c0 = kHalfN; c0 < BLOCK_N; c0 += CHUNK) {
    if (tile_col0 + c0 >= args.N) break;
    pp_chunk<EPI>(args, s, wbuf, c0 - kHalfN, c0, warp_row0, tile_col0, lane);
  }
}

template <int EPI, bool BF16>
__global__ void __launch_bounds__(kNumThreads, 1)
gemm_pingpong_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b,
                     const GemmArgs args) {
  extern __shared__ uint8_t smem_raw[];
  // 128B-swizzled tiles need 1024-byte alignment.
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* smem_a = smem;
  uint8_t* smem_b = smem + kStages * kABytes;
  uint8_t* smem_buf = smem + kStages * kStageBytes;   // the consumers' half-tile buffers
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem_buf + 2 * kHalfBytes);
  uint64_t* full_bar = bars;
  uint64_t* empty_bar = bars + kStages;

  const int wg = threadIdx.x >> 7;
  const int warp_in_group = (threadIdx.x >> 5) & 3;
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
      mbar_init(&empty_bar[s], 4);  // one arrive per warp of the consumer that read the stage
    }
    fence_mbar_init();
  }
  __syncthreads();

  if (wg == 0) {
    // ------------------------------------------------------------------ TMA producer
    setmaxnreg_dec<kProducerRegs>();
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
    }
    return;
  }

  // -------------------------------------------------------------------- consumer warpgroups
  setmaxnreg_inc<kConsumerRegs>();
  const int c = wg - 1;
  const uint32_t buf_s = smem_u32(smem_buf + c * kHalfBytes);
  // ring position of this consumer's first k block: consumer 1 starts after tile 0's num_kb stages
  int stage = (c * num_kb) % kStages;
  uint32_t phase = ((c * num_kb) / kStages) & 1;
  for (int tile = blockIdx.x + c * gridDim.x; tile < num_tiles; tile += 2 * gridDim.x) {
    const int m_blk = tile / n_blocks, n_blk = tile % n_blocks;
    if (tile >= (int)gridDim.x) named_barrier_sync(kOrderBar + c, 256);   // the other consumer has issued the previous tile
    // The first MMA of the tile overwrites the accumulators (scale-d 0); defining them here ends their live range at the
    // previous tile's epilogue instead of carrying all 128 registers through it.
    float acc[2][BLOCK_N / 2];
#pragma unroll
    for (int h = 0; h < 2; ++h)
#pragma unroll
      for (int i = 0; i < BLOCK_N / 2; ++i) acc[h][i] = 0.f;
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
          const uint64_t a_desc = make_smem_desc(a_addr + h * (kABytes / 2) + k * 32, 16, 1024);
          const uint64_t b_desc = make_smem_desc(b_addr + k * 32, 16, 1024);
          if (BF16) wgmma_ss_n128_bf16<0, 0>(acc[h], a_desc, b_desc, (kb | k) != 0);
          else      wgmma_ss_n128_f16<0, 0>(acc[h], a_desc, b_desc, (kb | k) != 0);
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
    // every MMA of this tile is issued: the other consumer may start on the next tile's stages
    if (tile + (int)gridDim.x < num_tiles) named_barrier_arrive(kOrderBar + (c ^ 1), 256);
    wgmma_wait<0>();
    if (lane == 0) mbar_arrive(&empty_bar[prev_stage]);
    // skip the other consumer's num_kb stages
    stage += num_kb;
    phase ^= (uint32_t)(stage / kStages) & 1;
    stage %= kStages;

    pp_epilogue<EPI>(args, acc, buf_s, kConsumerBar + c, warp_in_group, lane, m_blk * BLOCK_M, n_blk * BLOCK_N);
  }
}

template <int EPI, bool BF16>
int launch_kernel(const CUtensorMap& ta, const CUtensorMap& tb, const GemmArgs& a, int grid, cudaStream_t stream) {
  auto kern = gemm_pingpong_kernel<EPI, BF16>;
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
int launch(bool bf16, const CUtensorMap& ta, const CUtensorMap& tb, const GemmArgs& a, int grid, cudaStream_t stream) {
  return bf16 ? launch_kernel<EPI, true>(ta, tb, a, grid, stream) : launch_kernel<EPI, false>(ta, tb, a, grid, stream);
}

}  // namespace

int gemm_pingpong_launch(int epi, bool bf16, const CUtensorMap& ta, const CUtensorMap& tb, const GemmArgs& a, int grid,
                         cudaStream_t stream) {
  switch (epi) {
    case EPI_F16_BIAS:              return launch<EPI_F16_BIAS>(bf16, ta, tb, a, grid, stream);
    case EPI_F16_BIAS_QGELU:        return launch<EPI_F16_BIAS_QGELU>(bf16, ta, tb, a, grid, stream);
    case EPI_F32_BIAS_RESID:        return launch<EPI_F32_BIAS_RESID>(bf16, ta, tb, a, grid, stream);
    case EPI_F32_BIAS:              return launch<EPI_F32_BIAS>(bf16, ta, tb, a, grid, stream);
    case EPI_F32_ROWMAP:            return launch<EPI_F32_ROWMAP>(bf16, ta, tb, a, grid, stream);
    case EPI_BF16_DGELU:            return launch<EPI_BF16_DGELU>(bf16, ta, tb, a, grid, stream);
    case EPI_F16_BIAS_QGELU_SAVE:   return launch<EPI_F16_BIAS_QGELU_SAVE>(bf16, ta, tb, a, grid, stream);
    case EPI_F32_BIAS_RESID_STATS:  return launch<EPI_F32_BIAS_RESID_STATS>(bf16, ta, tb, a, grid, stream);
    case EPI_F16_LN_BIAS:           return launch<EPI_F16_LN_BIAS>(bf16, ta, tb, a, grid, stream);
    case EPI_F16_LN_BIAS_QGELU:     return launch<EPI_F16_LN_BIAS_QGELU>(bf16, ta, tb, a, grid, stream);
    default: set_last_error("gemm: unknown epilogue %d", epi); return 1;
  }
}

}  // namespace pg
