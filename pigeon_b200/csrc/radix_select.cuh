// Exact selection of the k-th smallest of n non-negative fp64 values by one CTA, shared by optics.cu (core distances)
// and geo_metrics.cu (median km error).
//
// Radix select on the uint64 bit pattern (for non-negative doubles, bit order is value order), most significant digit
// first: bits 53-63, 42-52, 31-41, 20-30, 9-19, 0-8.  `bits(j)` returns the pattern of value j for j in [0, n); each pass
// calls it once per j, so a caller can recompute values instead of storing them.  When the selected digit holds one
// candidate, one more pass fetches its remaining bits.  Histograms use shared-memory integer atomics only, so the
// result is exact and deterministic.
#pragma once
#include <stdint.h>

namespace pg {

// Every thread of the CTA must call this with the same n and k (1 <= k <= n); all of them get the selected pattern.
template <int THREADS, class Bits>
__device__ uint64_t radix_select_kth(int64_t n, uint32_t k, Bits bits) {
  __shared__ uint32_t hist[2048];
  __shared__ uint64_t s_prefix;
  __shared__ uint32_t s_k, s_cnt;
  if (threadIdx.x == 0) { s_prefix = 0; s_k = k; }
  int hi_shift = 64;
  for (int pass = 0; pass < 6; ++pass) {
    const int width = pass < 5 ? 11 : 9, shift = hi_shift - width;
    const uint32_t bins = 1u << width;
    for (uint32_t t = threadIdx.x; t < bins; t += THREADS) hist[t] = 0;
    __syncthreads();
    const uint64_t prefix = s_prefix;
    for (int64_t j = threadIdx.x; j < n; j += THREADS) {
      const uint64_t v = bits(j);
      if (hi_shift == 64 || (v >> hi_shift) == (prefix >> hi_shift)) atomicAdd(&hist[(v >> shift) & (bins - 1)], 1u);
    }
    __syncthreads();
    if (threadIdx.x < 32) {
      const uint32_t lane = threadIdx.x, per = bins / 32, kk = s_k;
      uint32_t sum = 0;
      for (uint32_t t = 0; t < per; ++t) sum += hist[lane * per + t];
      uint32_t incl = sum;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const uint32_t y = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= uint32_t(o)) incl += y;
      }
      const uint32_t excl = incl - sum;
      if (excl < kk && kk <= incl) {
        uint32_t acc = excl, d = lane * per;
        while (acc + hist[d] < kk) acc += hist[d++];
        s_prefix = prefix | (uint64_t(d) << shift);
        s_k = kk - acc;
        s_cnt = hist[d];
      }
    }
    __syncthreads();
    hi_shift = shift;
    if (s_cnt == 1 && shift > 0) {  // one candidate left: fetch its remaining bits
      const uint64_t pre = s_prefix;
      __syncthreads();  // every thread holds the prefix before the one match overwrites it
      for (int64_t j = threadIdx.x; j < n; j += THREADS) {
        const uint64_t v = bits(j);
        if ((v >> shift) == (pre >> shift)) s_prefix = v;
      }
      __syncthreads();
      break;
    }
  }
  const uint64_t out = s_prefix;
  __syncthreads();  // a second call in the same kernel may reset s_prefix only after every thread has read it
  return out;
}

}  // namespace pg
