// Shared epilogue of the wgmma kernels (gemm_wgmma.cu, head_fused_wgmma.cu): the warpgroup parks its fp32 accumulator
// fragments in a shared-memory tile (128 rows x 128 columns, rows padded by 4 floats), then each warp takes 32 rows of it
// -> bias / activation / residual -> global.
#pragma once
#include "gemm.h"
#include "ptx.cuh"

#include <cuda_bf16.h>

namespace pg {

constexpr int kStageWarpBytes = 32 * 128;   // per epilogue warp: 32 rows x 128 B, 16-byte pieces XOR-swizzled by (row & 7)
constexpr int kEpiTileN = 128;                       // columns of the accumulator tile
constexpr int kAccLdBytes = (kEpiTileN + 4) * 4;     // padded row: a warp reading one row per lane (16 bytes each) hits no bank twice
constexpr int kAccTileBytes = 128 * kAccLdBytes;

struct GemmArgs {
  int M, N, K;
  void* out;          // fp16 or fp32 [M, ldo]
  int ldo;
  const float* bias;  // [N] or nullptr
  // EPI_F32_ROWMAP: output row = rowmap_mul * (row / rowmap_div) + row % rowmap_div + rowmap_add
  int rowmap_div, rowmap_mul, rowmap_add;
  int vec_ok;  // output rows are 16-byte aligned -> vector stores allowed
  int operand_bf16;    // A and W hold bf16 instead of fp16
  const float* resid;  // residual source of EPI_F32_BIAS_RESID (== out when updating in place)
  void* aux;           // EPI_BF16_DGELU: fc1 pre-activation (fp16, read);  EPI_F16_BIAS_QGELU_SAVE: where to keep it (written)
  int mn_major;        // operands are [K, M] / [K, N] (MN-major wgmma operands), see GemmProblem::mn_major
  float* stats;         // LayerNorm-folded epilogues: float2 [M, stats_slots] partial (sum, sum of squares) per 128 columns
  int stats_slots;      // producer: N / 128; consumer: K / 128
  const float* colsum;  // consumer: fp32 [N] row sums of the folded weight
  float ln_eps;
};

__device__ __forceinline__ float quick_gelu(float v) {
  // HF "quick_gelu": x * sigmoid(1.702 x) = x / (1 + 2^(-1.702 log2(e) x)); ex2.approx + rcp.approx (2 MUFU / element)
  float e;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(-2.4554669595930157f * v));
  return __fdividef(v, 1.0f + e);
}

__device__ __forceinline__ float quick_gelu_grad(float x) {
  // d/dx [x * sigmoid(1.702 x)] = s * (1 + 1.702 x (1 - s))
  float e;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(-2.4554669595930157f * x));
  const float sg = __fdividef(1.0f, 1.0f + e);
  return sg * (1.0f + 1.702f * x * (1.0f - sg));
}
__device__ __forceinline__ uint32_t pack_bf16x2_rn(float lo, float hi) {
  uint32_t r;
  asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(hi), "f"(lo));
  return r;
}

// Accumulator fragment of one m64 wgmma block (wgmma.cuh layout) -> the shared accumulator tile; `blk_row0` = tile row of the
// block's first row, `acc_s` = shared address of the tile.
__device__ __forceinline__ void store_acc_fragment(uint32_t acc_s, int blk_row0, const float (&d)[kEpiTileN / 2], int warp_in_group,
                                                   int lane) {
  const uint32_t r0 = acc_s + (uint32_t)(blk_row0 + 16 * warp_in_group + (lane >> 2)) * kAccLdBytes + (uint32_t)(lane & 3) * 8;
#pragma unroll
  for (int j = 0; j < kEpiTileN / 8; ++j) {
    asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(r0 + j * 32), "f"(d[4 * j]), "f"(d[4 * j + 1]) : "memory");
    asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(r0 + 8 * kAccLdBytes + j * 32), "f"(d[4 * j + 2]), "f"(d[4 * j + 3]) : "memory");
  }
}

// One epilogue warp's share of one output tile: rows [warp_row0, warp_row0 + 32), tile columns [c_begin, c_end).
//   acc_row_s : shared address of this warp's first row (column 0) in the accumulator tile
//   stage     : this warp's private staging buffer (kStageWarpBytes)
// Per chunk of CHUNK columns (128 bytes of output per row): accumulator tile -> registers (thread = row) -> bias / activation ->
// smem staging (32 rows x 128 B, pieces swizzled: conflict-free both ways) -> coalesced global phase in which 8 lanes
// cover one 128-byte row segment (4 rows per instruction).  For the residual epilogue the 16-byte pieces a lane will
// update are fetched ONE CHUNK AHEAD so that their HBM latency hides behind the current chunk's work.
template <int EPI>
struct EpiTraits {
  static constexpr bool kF16Out = (EPI == EPI_F16_BIAS || EPI == EPI_F16_BIAS_QGELU || EPI == EPI_F16_BIAS_QGELU_SAVE ||
                                   EPI == EPI_F16_LN_BIAS || EPI == EPI_F16_LN_BIAS_QGELU);
  static constexpr bool kResid = (EPI == EPI_F32_BIAS_RESID || EPI == EPI_F32_BIAS_RESID_STATS);
  static constexpr bool kStats = (EPI == EPI_F32_BIAS_RESID_STATS);                           // LayerNorm producer
  static constexpr bool kLn = (EPI == EPI_F16_LN_BIAS || EPI == EPI_F16_LN_BIAS_QGELU);       // LayerNorm consumer
  static constexpr int CHUNK = kF16Out ? 64 : 32;
  static constexpr int kElt = kF16Out ? 2 : 4;   // EPI_BF16_DGELU stages fp32 (CHUNK 32) and stores 2-byte elements
};

// L2 eviction policies (createpolicy): the fp32 residual stream (read-modify-write) and
// the fp16 copy are touched once per kernel and are far larger than the 50 MB L2 — marked evict_first so that they do not
// push out the A operand, which the CTAs of one 128-row block share through L2.
__device__ __forceinline__ uint64_t l2_policy_evict_first() {
  uint64_t p;
  asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(p));
  return p;
}
__device__ __forceinline__ uint64_t l2_policy_evict_last() {
  uint64_t p;
  asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(p));
  return p;
}
__device__ __forceinline__ float4 ldg_f4_hint(const void* p, uint64_t pol) {
  float4 v;
  asm volatile("ld.global.L2::cache_hint.v4.f32 {%0, %1, %2, %3}, [%4], %5;"
               : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(p), "l"(pol));
  return v;
}
__device__ __forceinline__ void stg_u4_hint(void* p, uint4 v, uint64_t pol) {
  asm volatile("st.global.L2::cache_hint.v4.b32 [%0], {%1, %2, %3, %4}, %5;" ::"l"(p), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w), "l"(pol)
               : "memory");
}
__device__ __forceinline__ void stg_u2_hint(void* p, uint2 v, uint64_t pol) {
  asm volatile("st.global.L2::cache_hint.v2.b32 [%0], {%1, %2}, %3;" ::"l"(p), "r"(v.x), "r"(v.y), "l"(pol) : "memory");
}

template <int EPI>
__device__ __forceinline__ void load_residual(const GemmArgs& args, float4 (&res)[8], int warp_row0, int col0, int lane,
                                              uint64_t pol) {
  const int sub = lane >> 3, c16 = lane & 7;
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int grow = warp_row0 + i * 4 + sub;
    res[i] = make_float4(0.f, 0.f, 0.f, 0.f);
    if (grow < args.M)
      res[i] = ldg_f4_hint(reinterpret_cast<const uint8_t*>(args.resid) + ((long)grow * args.ldo + col0) * 4 + c16 * 16, pol);
  }
}

template <int EPI>
__device__ __forceinline__ void epilogue_tile(const GemmArgs& args, uint32_t acc_row_s, uint8_t* stage, int warp_row0,
                                              int tile_col0, int c_begin, int c_end, int lane) {
  constexpr bool kF16Out = EpiTraits<EPI>::kF16Out;
  constexpr int CHUNK = EpiTraits<EPI>::CHUNK;
  constexpr int kElt = EpiTraits<EPI>::kElt;
  constexpr bool kResid = EpiTraits<EPI>::kResid;
  constexpr bool kStats = EpiTraits<EPI>::kStats;
  constexpr bool kLn = EpiTraits<EPI>::kLn;
  const int sub = lane >> 3, c16 = lane & 7;
  // the staging buffer through explicit st.shared / ld.shared: `stage` went through integer alignment arithmetic in the
  // callers, so the compiler treats it as a generic pointer and would emit ST.E / LD.E (address-space check per access)
  const uint32_t stage_s = smem_u32(stage);
  float4 res[8], res_next[8];
  const uint64_t pol_stream = kResid ? l2_policy_evict_first() : 0;
  // LayerNorm consumer: statistics of this thread's A row (= output row) from the producer's per-128-column partials
  float ln_a = 1.f, ln_b = 0.f;   // out = ln_a * acc + ln_b * colsum + bias
  if (kLn) {
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
    ln_a = rsqrtf(var + args.ln_eps);
    ln_b = -ln_a * mu;
  }
  // LayerNorm producer: running (sum, sum of squares) of the fp16-rounded new residual values, per row piece of this lane
  float st_s[8], st_q[8];
  if (kStats) {
#pragma unroll
    for (int i = 0; i < 8; ++i) st_s[i] = st_q[i] = 0.f;
  }
  {
    const int col0 = tile_col0 + c_begin;
    if (kResid && args.vec_ok && col0 + CHUNK <= args.N) load_residual<EPI>(args, res, warp_row0, col0, lane, pol_stream);
  }
#pragma unroll 1
  for (int c0 = c_begin; c0 < c_end; c0 += CHUNK) {
    const int col0 = tile_col0 + c0;
    if (col0 >= args.N) break;  // warp-uniform: the rest of this tile is past N
    const bool in_n = (col0 + CHUNK <= args.N);
    const bool fast = in_n && args.vec_ok;
    if (kResid) {  // prefetch the next chunk's residual pieces
      const int ncol0 = col0 + CHUNK;
      if (c0 + CHUNK < c_end && args.vec_ok && ncol0 + CHUNK <= args.N) load_residual<EPI>(args, res_next, warp_row0, ncol0, lane, pol_stream);
    }
    __syncwarp();
    float v[CHUNK];
#pragma unroll
    for (int i = 0; i < CHUNK / 4; ++i) {
      const float4 t = lds_f4(acc_row_s + (uint32_t)lane * kAccLdBytes + (uint32_t)(c0 + 4 * i) * 4);
      v[4 * i + 0] = t.x; v[4 * i + 1] = t.y; v[4 * i + 2] = t.z; v[4 * i + 3] = t.w;
    }
    if (kLn) {   // LayerNorm folded: rstd * acc + (-rstd * mu) * colsum + bias, two FMAs per element
      // (N is a multiple of the chunk and bias != nullptr: checked at launch)
      const float4* c4 = reinterpret_cast<const float4*>(args.colsum + col0);
      const float4* b4 = reinterpret_cast<const float4*>(args.bias + col0);
#pragma unroll
      for (int i = 0; i < CHUNK / 4; ++i) {
        const float4 cs = __ldg(c4 + i);
        const float4 b = __ldg(b4 + i);
        v[4 * i + 0] = fmaf(ln_a, v[4 * i + 0], fmaf(ln_b, cs.x, b.x));
        v[4 * i + 1] = fmaf(ln_a, v[4 * i + 1], fmaf(ln_b, cs.y, b.y));
        v[4 * i + 2] = fmaf(ln_a, v[4 * i + 2], fmaf(ln_b, cs.z, b.z));
        v[4 * i + 3] = fmaf(ln_a, v[4 * i + 3], fmaf(ln_b, cs.w, b.w));
      }
    }
    if (!kLn && args.bias != nullptr) {
      if (in_n) {
        const float4* b4 = reinterpret_cast<const float4*>(args.bias + col0);
#pragma unroll
        for (int i = 0; i < CHUNK / 4; ++i) {
          const float4 b = __ldg(b4 + i);
          v[4 * i + 0] += b.x; v[4 * i + 1] += b.y; v[4 * i + 2] += b.z; v[4 * i + 3] += b.w;
        }
      } else {
#pragma unroll
        for (int i = 0; i < CHUNK; ++i)
          if (col0 + i < args.N) v[i] += __ldg(args.bias + col0 + i);
      }
    }
    constexpr bool kDgelu = (EPI == EPI_BF16_DGELU);
    constexpr bool kSave = (EPI == EPI_F16_BIAS_QGELU_SAVE);
    uint2 aux_u[8];
    if (kDgelu && fast) {   // this lane's pre-activation pieces for the coalesced phase, issued before the staging work
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const int grow = warp_row0 + i * 4 + sub;
        aux_u[i] = make_uint2(0u, 0u);
        if (grow < args.M)
          aux_u[i] = *reinterpret_cast<const uint2*>(reinterpret_cast<const __half*>(args.aux) + (long)grow * args.ldo +
                                                     col0 + c16 * 4);
      }
    }
    if (kSave && fast) {    // keep the pre-activation (fp16) for the backward pass: same staging / coalesced store, to aux
      const uint32_t srow = stage_s + lane * 128;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        uint4 pk;
        pk.x = pack_half2(v[8 * j + 0], v[8 * j + 1]);
        pk.y = pack_half2(v[8 * j + 2], v[8 * j + 3]);
        pk.z = pack_half2(v[8 * j + 4], v[8 * j + 5]);
        pk.w = pack_half2(v[8 * j + 6], v[8 * j + 7]);
        sts_u4(srow + ((j ^ (lane & 7)) << 4), pk);
      }
      __syncwarp();
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const int rr = i * 4 + sub;
        const int grow = warp_row0 + rr;
        if (grow < args.M)
          *reinterpret_cast<uint4*>(reinterpret_cast<uint8_t*>(args.aux) + ((long)grow * args.ldo + col0) * 2 + c16 * 16) =
              lds_u4(stage_s + rr * 128 + ((c16 ^ (rr & 7)) << 4));
      }
      __syncwarp();
    }
    if (EPI == EPI_F16_BIAS_QGELU || EPI == EPI_F16_LN_BIAS_QGELU || kSave) {
      if (kSave && !fast) {   // ragged tail: scalar stores of the pre-activation
        const int row = warp_row0 + lane;
        if (row < args.M) {
          __half* o = reinterpret_cast<__half*>(args.aux) + (long)row * args.ldo + col0;
#pragma unroll
          for (int i = 0; i < CHUNK; ++i)
            if (col0 + i < args.N) o[i] = __float2half_rn(v[i]);
        }
      }
#pragma unroll
      for (int i = 0; i < CHUNK; ++i) v[i] = quick_gelu(v[i]);
    }
    if (fast) {
      // ---- stage this thread's row (128 bytes); 16-byte piece j of row `lane` lives at piece slot j ^ (lane & 7)
      const uint32_t srow = stage_s + lane * 128;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        uint4 pk;
        if (kF16Out) {
          pk.x = pack_half2(v[8 * j + 0], v[8 * j + 1]);
          pk.y = pack_half2(v[8 * j + 2], v[8 * j + 3]);
          pk.z = pack_half2(v[8 * j + 4], v[8 * j + 5]);
          pk.w = pack_half2(v[8 * j + 6], v[8 * j + 7]);
        } else {
          pk.x = __float_as_uint(v[4 * j + 0]);
          pk.y = __float_as_uint(v[4 * j + 1]);
          pk.z = __float_as_uint(v[4 * j + 2]);
          pk.w = __float_as_uint(v[4 * j + 3]);
        }
        sts_u4(srow + ((j ^ (lane & 7)) << 4), pk);
      }
      __syncwarp();
      // ---- coalesced global phase
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const int rr = i * 4 + sub;
        const int grow = warp_row0 + rr;
        if (grow < args.M) {
          uint4 val = lds_u4(stage_s + rr * 128 + ((c16 ^ (rr & 7)) << 4));
          long orow = grow;
          if (EPI == EPI_F32_ROWMAP)
            orow = (long)args.rowmap_mul * (grow / args.rowmap_div) + (grow % args.rowmap_div) + args.rowmap_add;
          if (kDgelu) {   // 4 fp32 gradients x gelu'(u) -> 4 bf16 (8 bytes per lane, 64 contiguous bytes per row segment)
            const float2 u01 = __half22float2(*reinterpret_cast<const __half2*>(&aux_u[i].x));
            const float2 u23 = __half22float2(*reinterpret_cast<const __half2*>(&aux_u[i].y));
            uint2 o;
            o.x = pack_bf16x2_rn(__uint_as_float(val.x) * quick_gelu_grad(u01.x), __uint_as_float(val.y) * quick_gelu_grad(u01.y));
            o.y = pack_bf16x2_rn(__uint_as_float(val.z) * quick_gelu_grad(u23.x), __uint_as_float(val.w) * quick_gelu_grad(u23.y));
            *reinterpret_cast<uint2*>(reinterpret_cast<uint8_t*>(args.out) + (orow * args.ldo + col0) * 2 + c16 * 8) = o;
            continue;
          }
          uint8_t* gp = reinterpret_cast<uint8_t*>(args.out) + (orow * args.ldo + col0) * kElt + c16 * 16;
          if (kResid) {
            val.x = __float_as_uint(__uint_as_float(val.x) + res[i].x);
            val.y = __float_as_uint(__uint_as_float(val.y) + res[i].y);
            val.z = __float_as_uint(__uint_as_float(val.z) + res[i].z);
            val.w = __float_as_uint(__uint_as_float(val.w) + res[i].w);
            stg_u4_hint(gp, val, pol_stream);
          } else {
            *reinterpret_cast<uint4*>(gp) = val;
          }
          if (kStats) {   // fp16 copy of the new residual values (the next GEMM's A operand) and their moments
            const __half2 h01 = __floats2half2_rn(__uint_as_float(val.x), __uint_as_float(val.y));
            const __half2 h23 = __floats2half2_rn(__uint_as_float(val.z), __uint_as_float(val.w));
            uint2 hv;
            hv.x = *reinterpret_cast<const uint32_t*>(&h01);
            hv.y = *reinterpret_cast<const uint32_t*>(&h23);
            stg_u2_hint(reinterpret_cast<uint8_t*>(args.aux) + (orow * args.ldo + col0) * 2 + c16 * 8, hv, pol_stream);
            const float2 f01 = __half22float2(h01), f23 = __half22float2(h23);
            st_s[i] += (f01.x + f01.y) + (f23.x + f23.y);
            st_q[i] += fmaf(f01.x, f01.x, f01.y * f01.y) + fmaf(f23.x, f23.x, f23.y * f23.y);
          }
        }
      }
    } else {
      // ---- ragged N tail / unaligned rows: per-thread scalar stores
      const int row = warp_row0 + lane;
      if (row < args.M) {
        long orow = row;
        if (EPI == EPI_F32_ROWMAP)
          orow = (long)args.rowmap_mul * (row / args.rowmap_div) + (row % args.rowmap_div) + args.rowmap_add;
        if (kF16Out) {
          __half* o = reinterpret_cast<__half*>(args.out) + orow * args.ldo + col0;
#pragma unroll
          for (int i = 0; i < CHUNK; ++i)
            if (col0 + i < args.N) o[i] = __float2half_rn(v[i]);
        } else if (kDgelu) {
          __nv_bfloat16* o = reinterpret_cast<__nv_bfloat16*>(args.out) + orow * args.ldo + col0;
          const __half* u = reinterpret_cast<const __half*>(args.aux) + orow * args.ldo + col0;
#pragma unroll
          for (int i = 0; i < CHUNK; ++i)
            if (col0 + i < args.N) o[i] = __float2bfloat16_rn(v[i] * quick_gelu_grad(__half2float(u[i])));
        } else {
          float* o = reinterpret_cast<float*>(args.out) + orow * args.ldo + col0;
#pragma unroll
          for (int i = 0; i < CHUNK; ++i)
            if (col0 + i < args.N) {
              float x = v[i];
              if (kResid) x += args.resid[orow * args.ldo + col0 + i];
              o[i] = x;
            }
        }
      }
    }
    if (kResid) {
#pragma unroll
      for (int i = 0; i < 8; ++i) res[i] = res_next[i];
    }
    if (kStats && ((col0 + CHUNK) & 127) == 0) {   // 128 columns complete: combine the 8 lanes of each row, publish
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        float a = st_s[i], b = st_q[i];
#pragma unroll
        for (int o = 1; o < 8; o <<= 1) {
          a += __shfl_xor_sync(0xffffffffu, a, o);
          b += __shfl_xor_sync(0xffffffffu, b, o);
        }
        const int grow = warp_row0 + i * 4 + sub;
        if (c16 == 0 && grow < args.M)
          reinterpret_cast<float2*>(args.stats)[(long)grow * args.stats_slots + (col0 >> 7)] = make_float2(a, b);
        st_s[i] = st_q[i] = 0.f;
      }
    }
  }
}

}  // namespace pg
