// Non-interlaced PNG decoding on the GPU, byte-identical to Pillow's `Image.open(f).convert('RGB')`.  Four stages:
//   host      chunk walk (pg_png_parse): signature, IHDR, PLTE, the run of consecutive IDAT chunks, and every chunk
//             Pillow reads on the way (CRCs before the first IDAT, text limits, tRNS layout), so that a file whose
//             parse status is OK is one Pillow opens, loads and converts without an exception;
//   kernel 1  png_inflate_kernel: zlib / DEFLATE (RFC 1950 / 1951), one warp per stream over a persistent grid that
//             takes streams in order of decreasing compressed size.  The warp first gathers the stream's IDAT payloads
//             into one contiguous buffer (the chunk boundaries may fall anywhere), then its 32 lanes decode the same
//             symbols in lockstep from a 64-bit bit buffer through two-level tables in the warp's shared memory (so no
//             broadcast is needed), lane 0 stores literals and the whole warp copies matches; finally the warp checks
//             the Adler-32 with a parallel reduction.  The warp builds each dynamic block's tables together;
//   kernel 2  png_unfilter_kernel: in-place reconstruction of filter types 0-4, one CTA per image, its threads on
//             consecutive rows in a column skew (thread t works on column tile k - t at step k);
//   kernel 3  png_rgb_kernel: one thread per output pixel: bit unpacking, palette lookup, grey replication, alpha
//             drop and Pillow's 16-bit rules, into the caller's pg_image destinations.
// Per-image status: a stream that zlib would reject, that Pillow might read differently (more decompressed data than
// the rows plus PNG_SLACK, bytes after the Adler-32), or a filter type above 4 gives a non-OK status and the image is
// left unwritten; the caller decodes it on the host.  Every read is bounded by the image's own chunks and stream,
// every write by its own buffers and destination.
#include <cuda_runtime.h>
#include <stdarg.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <numeric>
#include <vector>

#include "../../include/pigeon_b200.h"
#include "prof.h"
#include "tma_host.h"

namespace pg {
namespace {

// ------------------------------------------------------------------------------------------------------------------
// Inflate: two-level Huffman tables (zlib inflate_table / libdeflate layout) and the warp decoder
// ------------------------------------------------------------------------------------------------------------------

constexpr int LIT_ROOT = 10, DIST_ROOT = 8, CLEN_ROOT = 7;
// Root tables plus subtables.  A complete code set needs at most zlib's ENOUGH for these roots (1332 and 400 entries);
// the builder refuses a layout past the capacity instead of overrunning it.
constexpr int LIT_ENTRIES = 1536, DIST_ENTRIES = 512, CLEN_ENTRIES = 1 << CLEN_ROOT;
constexpr long long PNG_SLACK = 4096;           // decompressed bytes accepted after the rows (then PG_PNG_TOO_LONG)
constexpr long long MAX_TEXT_CHUNK = 1 << 20;   // PngImagePlugin.MAX_TEXT_CHUNK (ImageFile.SAFEBLOCK)
constexpr long long MAX_TEXT_MEMORY = 64 * MAX_TEXT_CHUNK;
constexpr uint32_t ADLER_MOD = 65521;

// Table entry: bits 0-4 bits consumed (the code length, minus the root bits in a subtable; the subtable's index bits
// in a K_SUB root entry), bits 5-7 kind, bits 8-12 extra bits, bits 16-31 value.
enum : uint32_t { K_INVALID = 0, K_LIT = 1, K_LEN = 2, K_EOB = 3, K_SUB = 4, K_DIST = 5, K_SYM = 6 };
enum { TBL_LIT = 0, TBL_DIST = 1, TBL_CLEN = 2 };

__host__ __device__ __forceinline__ uint32_t entry(uint32_t kind, uint32_t nbits, uint32_t extra, uint32_t value) {
  return nbits | (kind << 5) | (extra << 8) | (value << 16);
}
__host__ __device__ __forceinline__ uint32_t e_bits(uint32_t e) { return e & 31; }
__host__ __device__ __forceinline__ uint32_t e_kind(uint32_t e) { return (e >> 5) & 7; }
__host__ __device__ __forceinline__ uint32_t e_extra(uint32_t e) { return (e >> 8) & 31; }
__host__ __device__ __forceinline__ uint32_t e_value(uint32_t e) { return e >> 16; }

// RFC 1951 §3.2.5 in closed form: length codes 257..285 and distance codes 0..29 (286, 287, 30 and 31 stay invalid)
__host__ __device__ __forceinline__ uint32_t symbol_entry(int kind, int sym, int nbits) {
  if (kind == TBL_CLEN) return entry(K_SYM, nbits, 0, sym);
  if (kind == TBL_DIST) {
    if (sym >= 30) return 0;
    if (sym < 4) return entry(K_DIST, nbits, 0, sym + 1);
    const int extra = (sym >> 1) - 1;
    return entry(K_DIST, nbits, extra, ((2 + (sym & 1)) << extra) + 1);
  }
  if (sym < 256) return entry(K_LIT, nbits, 0, sym);
  if (sym == 256) return entry(K_EOB, nbits, 0, 0);
  if (sym >= 286) return 0;
  const int c = sym - 257;
  if (c < 8) return entry(K_LEN, nbits, 0, c + 3);
  if (c == 28) return entry(K_LEN, nbits, 0, 258);
  const int extra = (c >> 2) - 1;
  return entry(K_LEN, nbits, extra, ((4 + (c & 3)) << extra) + 3);
}

struct InflateSmem {                  // one warp's tables and the code lengths of its current block
  uint32_t lit[LIT_ENTRIES];
  uint32_t dist[DIST_ENTRIES];
  uint32_t clen[CLEN_ENTRIES];
  uint16_t code[288 + 32];            // bit-reversed canonical code of each symbol (table build scratch)
  uint8_t lens[288 + 32];             // code lengths: literal/length at 0, distance at 288 (the fixed code's layout)
  int count[16], next[16];            // lane 0's canonical-code counters (kept out of local memory)
  int ok;
};

__host__ __device__ __forceinline__ void warp_sync() {
#ifdef __CUDA_ARCH__
  __syncwarp();
#endif
}

__host__ __device__ __forceinline__ int warp_sum(int v) {
#ifdef __CUDA_ARCH__
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
#endif
  return v;
}

__host__ __device__ __forceinline__ int warp_exclusive_scan(int v, int lane) {
#ifdef __CUDA_ARCH__
  int x = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int y = __shfl_up_sync(0xffffffffu, x, o);
    if (lane >= o) x += y;
  }
  return x - v;
#else
  (void)lane;
  (void)v;
  return 0;
#endif
}

__host__ __device__ __forceinline__ uint32_t reverse_bits(uint32_t c, int len) {
#ifdef __CUDA_ARCH__
  return __brev(c) >> (32 - len);
#else
  uint32_t r = 0;
  for (int i = 0; i < len; ++i) r |= ((c >> i) & 1u) << (len - 1 - i);
  return r;
#endif
}

// Builds table t (root bits `root`, `cap` entries) for symbols [0, n) with code lengths `lens`, all lanes of the warp
// together (host: lane 0 of 1).  Returns false (every lane) for an over-subscribed or incomplete set, except an empty or
// single one-bit distance code, which zlib accepts; its unused codes stay invalid.
__host__ __device__ bool build_table(InflateSmem& sm, const uint8_t* lens, int n, int kind, int root, int cap, uint32_t* t,
                                     int lane, int nlanes) {
  const int rsize = 1 << root;
  for (int i = lane; i < rsize; i += nlanes) t[i] = 0;
  warp_sync();
  if (lane == 0) {
    int* count = sm.count;
    int* next = sm.next;
    for (int l = 0; l < 16; ++l) count[l] = 0;
    for (int s = 0; s < n; ++s) ++count[lens[s]];
    count[0] = 0;
    int left = 1, total = 0, maxlen = 0;
    for (int l = 1; l < 16; ++l) {
      left = (left << 1) - count[l];
      total += count[l];
      if (count[l]) maxlen = l;
      if (left < 0) break;
    }
    bool ok = left >= 0 && (left == 0 || (kind == TBL_DIST && (total == 0 || (total == 1 && maxlen == 1))));
    if (ok) {
      next[1] = 0;
      for (int l = 1; l < 15; ++l) next[l + 1] = (next[l] + count[l]) << 1;
      for (int s = 0; s < n; ++s) {
        const int l = lens[s];
        if (!l) continue;
        const uint32_t rev = reverse_bits((uint32_t)next[l]++, l);
        sm.code[s] = (uint16_t)rev;
        if (l > root) {                                           // the longest code under each root prefix
          uint32_t& r = t[rev & (rsize - 1)];
          r = r > (uint32_t)l ? r : (uint32_t)l;
        }
      }
    }
    sm.ok = ok;
  }
  warp_sync();
  if (!sm.ok) return false;
  // subtables in root-index order: each lane sizes a contiguous range of root entries, then a warp scan places them
  const int per = (rsize + nlanes - 1) / nlanes;
  const int i0 = lane * per, i1 = i0 + per < rsize ? i0 + per : rsize;
  int mine = 0;
  for (int i = i0; i < i1; ++i)
    if (t[i]) mine += 1 << (t[i] - root);
  int off = rsize + warp_exclusive_scan(mine, lane);
  const int total = warp_sum(mine);
  if (rsize + total > cap) {
    warp_sync();
    return false;
  }
  for (int i = i0; i < i1; ++i)
    if (t[i]) {
      const int sb = (int)t[i] - root;
      t[i] = entry(K_SUB, sb, 0, off);
      off += 1 << sb;
    }
  warp_sync();
  for (int s = lane; s < n; s += nlanes) {
    const int l = lens[s];
    if (!l) continue;
    const uint32_t rev = sm.code[s];
    if (l <= root) {
      const uint32_t e = symbol_entry(kind, s, l);
      for (uint32_t i = rev; i < (uint32_t)rsize; i += 1u << l) t[i] = e;
    } else {
      const uint32_t sub = t[rev & (rsize - 1)];
      const uint32_t base = e_value(sub), size = 1u << e_bits(sub);
      const uint32_t e = symbol_entry(kind, s, l - root);
      for (uint32_t i = rev >> root; i < size; i += 1u << (l - root)) t[base + i] = e;
    }
  }
  warp_sync();
  return true;
}

// LSB-first bit reader over one stream; bytes past its end read as zero, and consuming them is an error.
struct Bits {
  const uint8_t* in;
  long long n, pos;
  uint64_t buf;
  int cnt;
  __host__ __device__ __forceinline__ void refill() {
    if (pos + 8 <= n) {                       // eight independent byte loads, then keep the bytes that fit
      uint64_t w = 0;
#pragma unroll
      for (int k = 0; k < 8; ++k) w |= (uint64_t)in[pos + k] << (8 * k);
      buf |= w << cnt;
      const int bytes = (64 - cnt) >> 3;
      pos += bytes;
      cnt += 8 * bytes;
      return;
    }
    while (cnt <= 56) {
      buf |= (uint64_t)(pos < n ? in[pos] : 0) << cnt;
      ++pos;
      cnt += 8;
    }
  }
  __host__ __device__ __forceinline__ uint32_t take(int k) {       // k <= cnt
    const uint32_t v = (uint32_t)(buf & ((1ull << k) - 1));
    buf >>= k;
    cnt -= k;
    return v;
  }
  __host__ __device__ __forceinline__ bool overrun() const { return pos * 8 - cnt > n * 8; }
  __host__ __device__ __forceinline__ long long byte_pos() const { return pos - (cnt >> 3); }   // when cnt % 8 == 0
};

__host__ __device__ __forceinline__ uint32_t lookup(Bits& br, const uint32_t* t, int root) {
  uint32_t e = t[br.buf & ((1u << root) - 1)];
  if (e_kind(e) == K_SUB) {
    br.take(root);
    e = t[e_value(e) + (br.buf & ((1u << e_bits(e)) - 1))];
  }
  br.take(e_bits(e));
  return e;
}

// Fills sm.lens with the fixed code (RFC 1951 §3.2.6) and builds both tables.
__host__ __device__ bool fixed_tables(InflateSmem& sm, int lane, int nlanes) {
  for (int s = lane; s < 288 + 32; s += nlanes) sm.lens[s] = s < 144 ? 8 : s < 256 ? 9 : s < 280 ? 7 : s < 288 ? 8 : 5;
  warp_sync();
  return build_table(sm, sm.lens, 288, TBL_LIT, LIT_ROOT, LIT_ENTRIES, sm.lit, lane, nlanes) &&
         build_table(sm, sm.lens + 288, 32, TBL_DIST, DIST_ROOT, DIST_ENTRIES, sm.dist, lane, nlanes);
}

// Reads a dynamic block header (RFC 1951 §3.2.7) and builds its tables; zlib's checks, PG_PNG_* status.
__host__ __device__ int dynamic_tables(InflateSmem& sm, Bits& br, int lane, int nlanes) {
  br.refill();
  const int hlit = (int)br.take(5) + 257, hdist = (int)br.take(5) + 1, hclen = (int)br.take(4) + 4;
  if (hlit > 286 || hdist > 30) return PG_PNG_BAD_DEFLATE;
  constexpr uint8_t order[19] = {16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15};
  br.refill();
  warp_sync();                                               // the previous block's lens and tables are no longer read
#pragma unroll
  for (int i = 0; i < 19; ++i) {
    const uint32_t v = i < hclen ? br.take(3) : 0;
    if (lane == 0) sm.lens[order[i]] = (uint8_t)v;
  }
  if (br.overrun()) return PG_PNG_TRUNCATED;
  warp_sync();
  if (!build_table(sm, sm.lens, 19, TBL_CLEN, CLEN_ROOT, CLEN_ENTRIES, sm.clen, lane, nlanes)) return PG_PNG_BAD_DEFLATE;
  // every lane decodes the same lengths; lane 0 stores them
  int i = 0, prev = -1;
  while (i < hlit + hdist) {
    br.refill();
    const uint32_t e = lookup(br, sm.clen, CLEN_ROOT);
    if (e_kind(e) != K_SYM) return PG_PNG_BAD_DEFLATE;
    const int sym = (int)e_value(e);
    int rep, val;
    if (sym < 16) {
      rep = 1;
      val = sym;
    } else if (sym == 16) {
      if (prev < 0) return PG_PNG_BAD_DEFLATE;
      rep = 3 + (int)br.take(2);
      val = prev;
    } else {
      rep = sym == 17 ? 3 + (int)br.take(3) : 11 + (int)br.take(7);
      val = 0;
    }
    if (i + rep > hlit + hdist) return PG_PNG_BAD_DEFLATE;
    if (lane == 0)
      for (int k = 0; k < rep; ++k) sm.lens[i + k] = (uint8_t)val;
    i += rep;
    prev = val;
  }
  if (br.overrun()) return PG_PNG_TRUNCATED;
  warp_sync();
  if (sm.lens[256] == 0) return PG_PNG_BAD_DEFLATE;           // no end-of-block code
  if (!build_table(sm, sm.lens, hlit, TBL_LIT, LIT_ROOT, LIT_ENTRIES, sm.lit, lane, nlanes)) return PG_PNG_BAD_DEFLATE;
  // the distance lengths follow the literal/length ones; copy them down so that the fixed layout (lens + 288) is shared
  uint8_t* dl = sm.lens + 288;
  warp_sync();
  if (lane == 0)
    for (int k = hdist - 1; k >= 0; --k) dl[k] = sm.lens[hlit + k];
  warp_sync();
  if (!build_table(sm, dl, hdist, TBL_DIST, DIST_ROOT, DIST_ENTRIES, sm.dist, lane, nlanes)) return PG_PNG_BAD_DEFLATE;
  return PG_PNG_OK;
}

// Adler-32 of out[0, len), all lanes: a = 1 + sum d_i, b = len + sum (len - i) d_i (mod 65521).
__host__ __device__ uint32_t adler32(const uint8_t* out, long long len, int lane, int nlanes) {
  unsigned long long s1 = 0, s2 = 0;
  long long w = (len - lane) % ADLER_MOD;                     // (len - i) mod 65521 for i = lane, lane + nlanes, ...
  for (long long i = lane; i < len; i += nlanes) {
    const uint32_t d = out[i];
    s1 += d;
    s2 += (unsigned long long)w * d;
    w = w >= nlanes ? w - nlanes : w + ADLER_MOD - nlanes;
  }
  const int a = warp_sum((int)(s1 % ADLER_MOD)), b = warp_sum((int)(s2 % ADLER_MOD));
  const uint32_t A = (uint32_t)((1 + (unsigned long long)a) % ADLER_MOD);
  const uint32_t B = (uint32_t)(((unsigned long long)(len % ADLER_MOD) + (unsigned long long)b) % ADLER_MOD);
  return (B << 16) | A;
}

// Inflates the zlib stream in[0, n) into out (at most cap bytes), every lane of the warp (host: one lane).  Status
// PG_PNG_OK only for a stream zlib decodes without error, of at least `need` bytes, with nothing after its Adler-32;
// *produced receives the decompressed length.
__host__ __device__ int inflate_zlib(const uint8_t* __restrict__ in, long long n, uint8_t* __restrict__ out, long long cap,
                                     long long need, InflateSmem& sm, int lane, int nlanes, long long* produced) {
  *produced = 0;
  if (n < 2) return PG_PNG_TRUNCATED;
  const int cmf = in[0], flg = in[1];
  if ((cmf & 15) != 8 || (cmf >> 4) > 7 || ((cmf << 8) | flg) % 31 != 0 || (flg & 0x20)) return PG_PNG_BAD_ZLIB;
  const long long window = 1LL << ((cmf >> 4) + 8);
  Bits br{in, n, 2, 0, 0};
  long long o = 0;
  int final_block = 0;
  do {
    br.refill();
    final_block = (int)br.take(1);
    const int type = (int)br.take(2);
    if (type == 0) {                                          // stored
      br.take(br.cnt & 7);
      const long long p = br.byte_pos();
      if (p + 4 > n) return PG_PNG_TRUNCATED;
      const uint32_t len = in[p] | (in[p + 1] << 8), nlen = in[p + 2] | (in[p + 3] << 8);
      if ((len ^ 0xffffu) != nlen) return PG_PNG_BAD_DEFLATE;
      if (p + 4 + len > n) return PG_PNG_TRUNCATED;
      if (o + len > cap) return PG_PNG_TOO_LONG;
      for (long long j = lane; j < len; j += nlanes) out[o + j] = in[p + 4 + j];
      o += len;
      br.pos = p + 4 + len;
      br.buf = 0;
      br.cnt = 0;
      continue;
    }
    if (type == 3) return PG_PNG_BAD_DEFLATE;
    if (type == 1) {
      warp_sync();
      if (!fixed_tables(sm, lane, nlanes)) return PG_PNG_BAD_DEFLATE;
    } else {
      const int st = dynamic_tables(sm, br, lane, nlanes);
      if (st) return st;
    }
    for (;;) {
      if (br.cnt < 48) br.refill();
      if (br.overrun()) return PG_PNG_TRUNCATED;
      const uint32_t e = lookup(br, sm.lit, LIT_ROOT);
      const uint32_t k = e_kind(e);
      if (k == K_LIT) {
        if (o >= cap) return PG_PNG_TOO_LONG;
        if (lane == 0) out[o] = (uint8_t)e_value(e);
        ++o;
        continue;
      }
      if (k == K_EOB) break;
      if (k != K_LEN) return PG_PNG_BAD_DEFLATE;
      const long long len = e_value(e) + br.take(e_extra(e));
      const uint32_t d = lookup(br, sm.dist, DIST_ROOT);
      if (e_kind(d) != K_DIST) return PG_PNG_BAD_DEFLATE;
      const long long dist = e_value(d) + br.take(e_extra(d));
      if (br.overrun()) return PG_PNG_TRUNCATED;
      if (dist > o || dist > window) return PG_PNG_BAD_DEFLATE;
      if (o + len > cap) return PG_PNG_TOO_LONG;
      warp_sync();                                            // literals stored by lane 0 are visible to every lane
      uint8_t* dst = out + o;
      const uint8_t* src = dst - dist;
      if (dist >= len) {
        for (long long j = lane; j < len; j += nlanes) dst[j] = src[j];
      } else {                                                // overlapping: lane i copies src[i mod dist], ...
        const int step = nlanes % (int)dist;
        int r = lane % (int)dist;
        for (long long j = lane; j < len; j += nlanes) {
          dst[j] = src[r];
          r += step;
          if (r >= dist) r -= (int)dist;
        }
      }
      o += len;
    }
  } while (!final_block);
  if (br.overrun()) return PG_PNG_TRUNCATED;
  br.take(br.cnt & 7);
  const long long p = br.byte_pos();
  if (p + 4 > n) return PG_PNG_TRUNCATED;
  if (p + 4 != n) return PG_PNG_BAD_ZLIB;                     // bytes after the stream
  const uint32_t want = ((uint32_t)in[p] << 24) | ((uint32_t)in[p + 1] << 16) | ((uint32_t)in[p + 2] << 8) | in[p + 3];
  warp_sync();
  if (adler32(out, o, lane, nlanes) != want) return PG_PNG_BAD_ZLIB;
  *produced = o;
  if (o < need) return PG_PNG_TRUNCATED;
  return PG_PNG_OK;
}

// ------------------------------------------------------------------------------------------------------------------
// Batch layout shared by the kernels and the host test entry
// ------------------------------------------------------------------------------------------------------------------

struct PngImg {
  int orig;                          // index in the caller's batch (status array)
  int width, height, depth, ctype, bpp, entries;
  int nchunks;
  long long row_bytes;               // without the filter byte
  long long z_off, z_len;            // the gathered zlib stream in the workspace
  long long raw_off, need, cap;      // inflated rows (need = height * (1 + row_bytes)) and room for more
  long long chunk0;                  // first IDAT payload in the chunk table
  uint8_t* dst;
  long long dst_stride;
  uint8_t pal[256 * 3];
};

struct Chunk {                       // one IDAT payload: packed input [src, src + len) -> stream bytes [dst, dst + len)
  long long src, len, dst;
};

__host__ __device__ inline void gather_stream(const PngImg& im, const Chunk* chunks, const uint8_t* bytes, uint8_t* z,
                                              int lane, int nlanes) {
  for (int c = 0; c < im.nchunks; ++c) {
    const Chunk ch = chunks[im.chunk0 + c];
    for (long long j = lane; j < ch.len; j += nlanes) z[im.z_off + ch.dst + j] = bytes[ch.src + j];
  }
}

constexpr int INFLATE_WARPS = 4;

__global__ void __launch_bounds__(32 * INFLATE_WARPS)
png_inflate_kernel(const uint8_t* __restrict__ bytes, const PngImg* __restrict__ imgs, const Chunk* __restrict__ chunks,
                   const int* __restrict__ order, int nimg, int* __restrict__ next, uint8_t* __restrict__ z,
                   uint8_t* __restrict__ raw, int* __restrict__ status) {
  __shared__ InflateSmem smem[INFLATE_WARPS];
  InflateSmem& sm = smem[threadIdx.x >> 5];
  const int lane = threadIdx.x & 31;
  for (;;) {
    int k = 0;
    if (lane == 0) k = atomicAdd(next, 1);
    k = __shfl_sync(0xffffffffu, k, 0);
    if (k >= nimg) return;
    const PngImg& im = imgs[order[k]];
    gather_stream(im, chunks, bytes, z, lane, 32);
    __syncwarp();
    long long produced;
    const int st = inflate_zlib(z + im.z_off, im.z_len, raw + im.raw_off, im.cap, im.need, sm, lane, 32, &produced);
    if (lane == 0 && st) status[im.orig] = st;
    __syncwarp();
  }
}

// Reconstructs bytes [x0, x1) of one row (RFC 2083 §6): row and prev point at the bytes after the filter byte.
__host__ __device__ inline void unfilter_span(uint8_t* __restrict__ row, const uint8_t* __restrict__ prev, int ft, int bpp,
                                              long long x0, long long x1) {
  switch (ft) {
    case 1:
      for (long long x = x0 < bpp ? bpp : x0; x < x1; ++x) row[x] = (uint8_t)(row[x] + row[x - bpp]);
      break;
    case 2:
      if (prev)
        for (long long x = x0; x < x1; ++x) row[x] = (uint8_t)(row[x] + prev[x]);
      break;
    case 3:
      for (long long x = x0; x < x1; ++x) {
        const int a = x >= bpp ? row[x - bpp] : 0, b = prev ? prev[x] : 0;
        row[x] = (uint8_t)(row[x] + ((a + b) >> 1));
      }
      break;
    case 4:
      for (long long x = x0; x < x1; ++x) {
        const int a = x >= bpp ? row[x - bpp] : 0, b = prev ? prev[x] : 0, c = prev && x >= bpp ? prev[x - bpp] : 0;
        const int p = a + b - c, pa = abs(p - a), pb = abs(p - b), pc = abs(p - c);
        row[x] = (uint8_t)(row[x] + (pa <= pb && pa <= pc ? a : pb <= pc ? b : c));
      }
      break;
    default:
      break;
  }
}

constexpr int UNFILTER_THREADS = 128, UNFILTER_TILE = 32;

// One CTA per image.  Rows go in groups of UNFILTER_THREADS, one per thread; at step k thread t reconstructs column tile
// k - t of its row, whose upper neighbour (thread t - 1, or the previous group's last row) was finished at step k - 1
// and whose left neighbour is its own earlier tile.
__global__ void __launch_bounds__(UNFILTER_THREADS)
png_unfilter_kernel(const PngImg* __restrict__ imgs, uint8_t* __restrict__ raw, int* __restrict__ status) {
  const PngImg& im = imgs[blockIdx.x];
  __shared__ int bad;
  if (threadIdx.x == 0) bad = status[im.orig];
  __syncthreads();
  if (bad) return;
  const long long rb = im.row_bytes, stride = rb + 1;
  const long long tiles = (rb + UNFILTER_TILE - 1) / UNFILTER_TILE;
  uint8_t* base = raw + im.raw_off;
  for (long long g0 = 0; g0 < im.height; g0 += UNFILTER_THREADS) {
    const long long r = g0 + threadIdx.x;
    const int rows = (int)min((long long)UNFILTER_THREADS, (long long)im.height - g0);
    const bool active = threadIdx.x < rows;
    uint8_t* row = base + r * stride + 1;
    const uint8_t* prev = r > 0 ? row - stride : nullptr;
    const int ft = active ? row[-1] : 0;
    if (ft > 4) bad = 1;
    __syncthreads();
    if (bad) {
      if (threadIdx.x == 0) status[im.orig] = PG_PNG_BAD_FILTER;
      return;
    }
    for (long long step = 0; step < tiles + rows - 1; ++step) {
      const long long k = step - threadIdx.x;
      if (active && k >= 0 && k < tiles)
        unfilter_span(row, prev, ft, im.bpp, k * UNFILTER_TILE, min(rb, (k + 1) * UNFILTER_TILE));
      __syncthreads();
    }
  }
}

// Output pixel (x, y): Pillow's unpackers for the PNG raw modes followed by convert('RGB').
__host__ __device__ inline void rgb_pixel(const PngImg& im, const uint8_t* __restrict__ raw, int x, int y) {
  const uint8_t* row = raw + im.raw_off + (long long)y * (im.row_bytes + 1) + 1;
  uint8_t* o = im.dst + (long long)y * im.dst_stride + 3 * (long long)x;
  const int d = im.depth;
  if (im.ctype == 0 || im.ctype == 3) {
    int v;
    if (d < 8) {
      const long long bit = (long long)x * d;
      v = (row[bit >> 3] >> (8 - d - (int)(bit & 7))) & ((1 << d) - 1);
    } else if (d == 8) {
      v = row[x];
    } else {
      v = (row[2 * x] << 8) | row[2 * x + 1];
    }
    if (im.ctype == 3) {                                      // an index past the palette is black
      const bool in = v < im.entries;
      o[0] = in ? im.pal[3 * v] : 0;
      o[1] = in ? im.pal[3 * v + 1] : 0;
      o[2] = in ? im.pal[3 * v + 2] : 0;
      return;
    }
    // 1 bit: 0 / 255; 2 and 4 bits scale by 85 and 17; I;16 -> RGB clips to 255
    const uint8_t g = (uint8_t)(d < 8 ? v * (255 / ((1 << d) - 1)) : v > 255 ? 255 : v);
    o[0] = o[1] = o[2] = g;
    return;
  }
  const int bps = d >> 3;                                     // bytes per sample; 16-bit samples keep the high byte
  const int spp = im.ctype == 2 ? 3 : im.ctype == 4 ? 2 : 4;
  const uint8_t* p = row + (long long)x * spp * bps;
  if (im.ctype == 4) {
    o[0] = o[1] = o[2] = p[0];
  } else {
    o[0] = p[0];
    o[1] = p[bps];
    o[2] = p[2 * bps];
  }
}

__global__ void __launch_bounds__(256)
png_rgb_kernel(const PngImg* __restrict__ imgs, const long long* __restrict__ pix0, int n, long long npix,
               const uint8_t* __restrict__ raw, const int* __restrict__ status) {
  const long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= npix) return;
  int lo = 0, hi = n - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (pix0[mid] <= g) lo = mid; else hi = mid - 1;
  }
  const PngImg& im = imgs[lo];
  if (status[im.orig]) return;
  const long long local = g - pix0[lo];
  const int y = (int)(local / im.width);
  rgb_pixel(im, raw, (int)(local - (long long)y * im.width), y);
}

// ------------------------------------------------------------------------------------------------------------------
// Host: chunk walk
// ------------------------------------------------------------------------------------------------------------------

inline uint32_t be32(const uint8_t* p) { return ((uint32_t)p[0] << 24) | ((uint32_t)p[1] << 16) | ((uint32_t)p[2] << 8) | p[3]; }

uint32_t crc32(const uint8_t* p, long long n, uint32_t c = 0) {
  static uint32_t table[256];
  static bool init = [] {
    for (uint32_t i = 0; i < 256; ++i) {
      uint32_t v = i;
      for (int k = 0; k < 8; ++k) v = v & 1 ? 0xedb88320u ^ (v >> 1) : v >> 1;
      table[i] = v;
    }
    return true;
  }();
  (void)init;
  c = ~c;
  for (long long i = 0; i < n; ++i) c = table[(c ^ p[i]) & 255] ^ (c >> 8);
  return ~c;
}

inline bool is_cid(const uint8_t* c) {        // PngImagePlugin.is_cid: rb"\w\w\w\w"
  for (int i = 0; i < 4; ++i) {
    const uint8_t b = c[i];
    if (!((b >= 'a' && b <= 'z') || (b >= 'A' && b <= 'Z') || (b >= '0' && b <= '9') || b == '_')) return false;
  }
  return true;
}

inline bool cid_is(const uint8_t* c, const char* s) { return memcmp(c, s, 4) == 0; }

struct Why {
  char* buf;
  size_t cap;
  int fail(int st, const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, cap, fmt, ap);
    va_end(ap);
    return st;
  }
};

// Decompressed length of the zlib stream s[0, n) when it is complete, valid and shorter than MAX_TEXT_CHUNK; -1 else.
long long text_stream_length(const uint8_t* s, long long n) {
  static thread_local std::vector<uint8_t> out;
  static thread_local InflateSmem sm;
  out.resize(MAX_TEXT_CHUNK);
  long long produced = 0;
  const int st = inflate_zlib(s, n, out.data(), MAX_TEXT_CHUNK - 1, 0, sm, 0, 1, &produced);
  return st == PG_PNG_OK ? produced : -1;
}

// The chunks Pillow's PngStream reads, with the conditions under which its handler raises (or, for a compressed text
// chunk, under which its size is not known here): those files go to the host.  `text` accumulates check_text_memory.
int check_ancillary(const uint8_t* cid, const uint8_t* s, long long len, const pg_png_info* info, long long* text,
                    Why* why) {
  const char* c = reinterpret_cast<const char*>(cid);
  if (cid_is(cid, "acTL") || cid_is(cid, "fcTL") || cid_is(cid, "fdAT"))
    return why->fail(PG_PNG_UNSUPPORTED, "APNG (%.4s chunk)", c);
  if (cid_is(cid, "gAMA") && len < 4) return why->fail(PG_PNG_UNSUPPORTED, "short gAMA chunk");
  if (cid_is(cid, "cHRM") && len % 4) return why->fail(PG_PNG_UNSUPPORTED, "cHRM length not a multiple of 4");
  if (cid_is(cid, "sRGB") && len < 1) return why->fail(PG_PNG_UNSUPPORTED, "truncated sRGB chunk");
  if (cid_is(cid, "pHYs") && len < 9) return why->fail(PG_PNG_UNSUPPORTED, "truncated pHYs chunk");
  if (cid_is(cid, "tRNS")) {
    const int ct = info->color_type;
    if ((ct == 0 && len < 2) || (ct == 2 && len < 6)) return why->fail(PG_PNG_UNSUPPORTED, "short tRNS chunk");
    if (ct == 3 && info->palette_entries == 0) return why->fail(PG_PNG_UNSUPPORTED, "tRNS in a palette image without PLTE");
  }
  const uint8_t* nul = static_cast<const uint8_t*>(memchr(s, 0, (size_t)len));
  if (cid_is(cid, "tEXt")) {
    if (nul && nul > s) *text += len - (nul - s) - 1;
  } else if (cid_is(cid, "zTXt")) {
    const long long k = nul ? nul - s : len;
    if (k < len - 1) {
      if (s[k + 1] != 0) return why->fail(PG_PNG_UNSUPPORTED, "zTXt compression method %d", s[k + 1]);
      const long long got = text_stream_length(s + k + 2, len - k - 2);
      if (got < 0) return why->fail(PG_PNG_UNSUPPORTED, "zTXt stream not checked (corrupt, or above MAX_TEXT_CHUNK)");
      if (k > 0) *text += got;
    } else if (k > 0) {
      return why->fail(PG_PNG_UNSUPPORTED, "empty zTXt stream");
    }
  } else if (cid_is(cid, "iTXt")) {
    if (nul && len - (nul - s) - 1 >= 2) {
      const uint8_t* r = nul + 1;
      const int cf = r[0], cm = r[1];
      const uint8_t* end = s + len;
      const uint8_t* z1 = static_cast<const uint8_t*>(memchr(r + 2, 0, (size_t)(end - (r + 2))));
      const uint8_t* z2 = z1 ? static_cast<const uint8_t*>(memchr(z1 + 1, 0, (size_t)(end - (z1 + 1)))) : nullptr;
      if (z2) {
        long long vlen = end - (z2 + 1);                      // bytes of the value: at least its characters
        if (cf != 0 && cm == 0) {
          vlen = text_stream_length(z2 + 1, vlen);
          if (vlen < 0) return why->fail(PG_PNG_UNSUPPORTED, "iTXt stream not checked (corrupt, or above MAX_TEXT_CHUNK)");
        }
        if (cf == 0 || cm == 0) *text += vlen;
      }
    }
  } else if (cid_is(cid, "iCCP")) {
    if (!nul || nul + 1 >= s + len || nul[1] != 0) return why->fail(PG_PNG_UNSUPPORTED, "iCCP chunk not checked");
    if (text_stream_length(nul + 2, s + len - (nul + 2)) < 0)
      return why->fail(PG_PNG_UNSUPPORTED, "iCCP profile not checked (corrupt, or above MAX_TEXT_CHUNK)");
  }
  if (*text > MAX_TEXT_MEMORY) return why->fail(PG_PNG_UNSUPPORTED, "text chunks above MAX_TEXT_MEMORY");
  return PG_PNG_OK;
}

int parse(const uint8_t* d, long long n, pg_png_info* info, Why* why) {
  memset(info, 0, sizeof(*info));
  static const uint8_t sig[8] = {0x89, 'P', 'N', 'G', '\r', '\n', 0x1a, '\n'};
  if (!d || n < 8 || memcmp(d, sig, 8) != 0) return why->fail(PG_PNG_BAD_HEADER, "not a PNG file");
  long long pos = 8, text = 0;
  bool ihdr = false, plte = false;
  for (;;) {                                                  // chunks before the first IDAT: Pillow checks every CRC
    if (pos + 8 > n) return why->fail(PG_PNG_BAD_HEADER, "file ends before IDAT");
    const long long len = be32(d + pos);
    const uint8_t* cid = d + pos + 4;
    const uint8_t* s = d + pos + 8;
    if (!is_cid(cid)) return why->fail(PG_PNG_BAD_HEADER, "broken chunk type at %lld", pos);
    if (cid_is(cid, "IDAT")) break;
    if (pos + 12 + len > n) return why->fail(PG_PNG_BAD_HEADER, "truncated %.4s chunk", (const char*)cid);
    if (crc32(s, len, crc32(cid, 4)) != be32(s + len))
      return why->fail(PG_PNG_BAD_HEADER, "bad CRC in %.4s chunk", (const char*)cid);
    if (!ihdr) {
      if (!cid_is(cid, "IHDR") || len != 13) return why->fail(PG_PNG_BAD_HEADER, "no IHDR chunk first");
      ihdr = true;
      const uint32_t w = be32(s), h = be32(s + 4);
      const int depth = s[8], ct = s[9];
      if (w == 0 || h == 0 || w > 0x7fffffffu || h > 0x7fffffffu)
        return why->fail(PG_PNG_BAD_HEADER, "image size %u x %u", w, h);
      const bool valid = (ct == 0 && (depth == 1 || depth == 2 || depth == 4 || depth == 8 || depth == 16)) ||
                         (ct == 3 && (depth == 1 || depth == 2 || depth == 4 || depth == 8)) ||
                         ((ct == 2 || ct == 4 || ct == 6) && (depth == 8 || depth == 16));
      if (!valid) return why->fail(PG_PNG_BAD_HEADER, "bit depth %d with colour type %d", depth, ct);
      if (s[11] != 0) return why->fail(PG_PNG_BAD_HEADER, "unknown filter method %d", s[11]);
      if (s[10] != 0) return why->fail(PG_PNG_UNSUPPORTED, "compression method %d", s[10]);
      if (s[12] != 0) return why->fail(PG_PNG_UNSUPPORTED, "interlaced (Adam7)");
      info->width = (int32_t)w;
      info->height = (int32_t)h;
      info->bit_depth = depth;
      info->color_type = ct;
      info->channels = ct == 2 ? 3 : ct == 4 ? 2 : ct == 6 ? 4 : 1;
      info->row_bytes = ((long long)w * info->channels * depth + 7) / 8;
      if ((double)h * (double)(info->row_bytes + 1) > (double)(1LL << 40))
        return why->fail(PG_PNG_UNSUPPORTED, "image too large");
    } else if (cid_is(cid, "IHDR")) {
      return why->fail(PG_PNG_UNSUPPORTED, "second IHDR chunk");
    } else if (cid_is(cid, "IEND")) {
      return why->fail(PG_PNG_BAD_HEADER, "no IDAT chunk");
    } else if (cid_is(cid, "PLTE")) {
      if (info->color_type == 3) {
        if (plte || len % 3 || len == 0 || len > 768) return why->fail(PG_PNG_UNSUPPORTED, "PLTE of %lld bytes", len);
        plte = true;
        info->palette_entries = (int32_t)(len / 3);
        memcpy(info->palette, s, (size_t)len);
      }
    } else {
      const int st = check_ancillary(cid, s, len, info, &text, why);
      if (st) return st;
    }
    pos += 12 + len;
  }
  if (!ihdr) return why->fail(PG_PNG_BAD_HEADER, "no IHDR chunk first");
  info->idat_offset = pos;
  for (; pos + 8 <= n && cid_is(d + pos + 4, "IDAT"); pos += 12 + be32(d + pos)) {   // the run of consecutive IDATs
    const long long len = be32(d + pos);
    if (pos + 12 + len > n) return why->fail(PG_PNG_UNSUPPORTED, "truncated IDAT chunk");
    info->zlib_bytes += len;
    ++info->idat_chunks;
  }
  // What Pillow's load_end reads after the image data, up to IEND (no CRC checks there; a short or broken chunk header
  // ends the walk)
  while (pos + 8 <= n) {
    const long long len = be32(d + pos);
    const uint8_t* cid = d + pos + 4;
    if (!is_cid(cid) || cid_is(cid, "IEND")) break;
    if (cid_is(cid, "IDAT")) return why->fail(PG_PNG_UNSUPPORTED, "IDAT chunks not consecutive");
    if (pos + 8 + len > n) return why->fail(PG_PNG_UNSUPPORTED, "truncated %.4s chunk after IDAT", (const char*)cid);
    if (cid_is(cid, "IHDR")) return why->fail(PG_PNG_UNSUPPORTED, "IHDR chunk after IDAT");
    if (!cid_is(cid, "PLTE")) {
      const int st = check_ancillary(cid, d + pos + 8, len, info, &text, why);
      if (st) return st;
    }
    pos += 12 + len;
  }
  info->bpp = std::max(1, info->channels * info->bit_depth / 8);
  info->status = PG_PNG_OK;
  return PG_PNG_OK;
}

// ------------------------------------------------------------------------------------------------------------------
// Host: batch plan
// ------------------------------------------------------------------------------------------------------------------

struct Plan {
  std::vector<PngImg> imgs;
  std::vector<Chunk> chunks;
  std::vector<int> order;                            // images by decreasing compressed size
  std::vector<long long> pix0;
  long long npix = 0, zbytes = 0, rawbytes = 0;
  size_t off_bytes = 0, off_meta = 0, off_z = 0, off_raw = 0, total = 0;
  size_t meta_bytes = 0, m_imgs = 0, m_chunks = 0, m_order = 0, m_pix0 = 0, m_next = 0;
};

inline size_t align_up(size_t x, size_t a) { return (x + a - 1) / a * a; }

// packed / offsets may be null (workspace sizing: the chunk count comes from the infos); dst may be null.
int make_plan(const uint8_t* packed, const int64_t* offsets, const pg_png_info* infos, int n, int64_t packed_bytes,
              const pg_image* dst, Plan* P) {
  if (!infos || n <= 0 || packed_bytes < 0) {
    set_last_error("pg_png: null infos, n <= 0 or packed_bytes < 0");
    return 1;
  }
  long long nchunks = 0;
  for (int i = 0; i < n; ++i) {
    const pg_png_info& inf = infos[i];
    if (inf.status != PG_PNG_OK) continue;
    PngImg im;
    memset(&im, 0, sizeof(im));
    im.orig = i;
    im.width = inf.width;
    im.height = inf.height;
    im.depth = inf.bit_depth;
    im.ctype = inf.color_type;
    im.bpp = inf.bpp;
    im.entries = inf.palette_entries;
    im.row_bytes = inf.row_bytes;
    im.nchunks = inf.idat_chunks;
    im.chunk0 = nchunks;
    im.z_off = P->zbytes;
    im.z_len = inf.zlib_bytes;
    im.need = (long long)inf.height * (inf.row_bytes + 1);
    im.cap = im.need + PNG_SLACK;
    im.raw_off = P->rawbytes;
    memcpy(im.pal, inf.palette, sizeof(im.pal));
    if (inf.width <= 0 || inf.height <= 0 || inf.bpp < 1 || inf.idat_chunks < 0 || inf.zlib_bytes < 0 ||
        inf.row_bytes != ((long long)inf.width * std::max(inf.channels, 1) * inf.bit_depth + 7) / 8) {
      set_last_error("pg_png: info %d is inconsistent (not from pg_png_parse?)", i);
      return 1;
    }
    if (dst) {
      if (!dst[i].data || dst[i].height != inf.height || dst[i].width != inf.width ||
          dst[i].row_stride < 3LL * inf.width) {
        set_last_error("pg_png_decode: destination %d must be %d x %d x 3 with row_stride >= %lld", i, inf.height,
                       inf.width, 3LL * inf.width);
        return 1;
      }
      im.dst = const_cast<uint8_t*>(dst[i].data);
      im.dst_stride = dst[i].row_stride;
    }
    if (packed) {                                      // the IDAT run, re-walked within the file's bytes
      const long long f0 = offsets[i], f1 = offsets[i + 1];
      long long pos = f0 + inf.idat_offset, at = 0;
      for (int c = 0; c < inf.idat_chunks; ++c) {
        if (pos + 8 > f1) {
          set_last_error("pg_png_decode: file %d does not match its info", i);
          return 1;
        }
        const long long len = be32(packed + pos);
        if (pos + 8 + len > f1 || memcmp(packed + pos + 4, "IDAT", 4) != 0) {
          set_last_error("pg_png_decode: file %d does not match its info", i);
          return 1;
        }
        P->chunks.push_back({pos + 8, len, at});
        at += len;
        pos += 12 + len;
      }
      if (at != inf.zlib_bytes) {
        set_last_error("pg_png_decode: file %d does not match its info", i);
        return 1;
      }
    }
    nchunks += inf.idat_chunks;
    P->zbytes += align_up((size_t)inf.zlib_bytes, 16);
    P->rawbytes += align_up((size_t)im.cap, 16);
    P->pix0.push_back(P->npix);
    P->npix += (long long)inf.width * inf.height;
    P->imgs.push_back(im);
  }
  const int nimg = (int)P->imgs.size();
  P->order.resize(nimg);
  std::iota(P->order.begin(), P->order.end(), 0);
  std::stable_sort(P->order.begin(), P->order.end(),
                   [P](int a, int b) { return P->imgs[a].z_len > P->imgs[b].z_len; });
  P->m_imgs = 0;
  P->m_chunks = align_up(P->m_imgs + nimg * sizeof(PngImg), 16);
  P->m_order = align_up(P->m_chunks + nchunks * sizeof(Chunk), 16);
  P->m_pix0 = align_up(P->m_order + nimg * sizeof(int), 16);
  P->m_next = align_up(P->m_pix0 + nimg * sizeof(long long), 16);
  P->meta_bytes = align_up(P->m_next + sizeof(int), 256);
  P->off_bytes = 0;
  P->off_meta = align_up((size_t)packed_bytes, 256);
  P->off_z = P->off_meta + P->meta_bytes;
  P->off_raw = align_up(P->off_z + P->zbytes, 256);
  P->total = align_up(P->off_raw + P->rawbytes, 256);
  return 0;
}

}  // namespace

int png_parse(const uint8_t* data, int64_t bytes, pg_png_info* info) {
  if (!info) {
    set_last_error("pg_png_parse: null info");
    return -1;
  }
  char msg[200];
  msg[0] = 0;
  Why why{msg, sizeof(msg)};
  const int st = parse(data, bytes, info, &why);
  info->status = st;
  if (st) set_last_error("%s", msg);
  return st;
}

size_t png_workspace_bytes(const pg_png_info* infos, int n, int64_t packed_bytes) {
  Plan P;
  if (make_plan(nullptr, nullptr, infos, n, packed_bytes, nullptr, &P)) return 0;
  return P.total;
}

int png_decode(const uint8_t* packed, const int64_t* offsets, const pg_png_info* infos, int n, const pg_image* dst,
               void* workspace, size_t workspace_bytes, int32_t* status_out, cudaStream_t stream) {
  if (!packed || !offsets || !infos || !dst || !status_out || n <= 0) {
    set_last_error("pg_png_decode: null argument");
    return 1;
  }
  Plan P;
  if (make_plan(packed, offsets, infos, n, offsets[n], dst, &P)) return 1;
  if (!workspace || workspace_bytes < P.total || (reinterpret_cast<uintptr_t>(workspace) & 255)) {
    set_last_error("pg_png_decode: workspace too small (%zu < %zu) or not 256-byte aligned", workspace_bytes, P.total);
    return 1;
  }
  uint8_t* ws = reinterpret_cast<uint8_t*>(workspace);
  const int nimg = (int)P.imgs.size();
  std::vector<uint8_t> meta(P.meta_bytes, 0);
  memcpy(meta.data() + P.m_imgs, P.imgs.data(), nimg * sizeof(PngImg));
  memcpy(meta.data() + P.m_chunks, P.chunks.data(), P.chunks.size() * sizeof(Chunk));
  memcpy(meta.data() + P.m_order, P.order.data(), nimg * sizeof(int));
  memcpy(meta.data() + P.m_pix0, P.pix0.data(), nimg * sizeof(long long));
  std::vector<int32_t> host_status(n);                  // the parse status of skipped images, 0 for decoded ones
  for (int i = 0; i < n; ++i) host_status[i] = infos[i].status;
  cudaError_t e = cudaMemcpyAsync(ws + P.off_bytes, packed, (size_t)offsets[n], cudaMemcpyHostToDevice, stream);
  if (e == cudaSuccess) e = cudaMemcpyAsync(ws + P.off_meta, meta.data(), P.meta_bytes, cudaMemcpyHostToDevice, stream);
  if (e == cudaSuccess)
    e = cudaMemcpyAsync(status_out, host_status.data(), (size_t)n * sizeof(int32_t), cudaMemcpyHostToDevice, stream);
  if (e != cudaSuccess) {
    set_last_error("pg_png_decode: upload: %s", cudaGetErrorString(e));
    return 1;
  }
  if (nimg == 0) return 0;
  const uint8_t* meta_d = ws + P.off_meta;
  const PngImg* d_imgs = reinterpret_cast<const PngImg*>(meta_d + P.m_imgs);
  const Chunk* d_chunks = reinterpret_cast<const Chunk*>(meta_d + P.m_chunks);
  const int* d_order = reinterpret_cast<const int*>(meta_d + P.m_order);
  const long long* d_pix0 = reinterpret_cast<const long long*>(meta_d + P.m_pix0);
  int* d_next = reinterpret_cast<int*>(ws + P.off_meta + P.m_next);
  uint8_t* d_z = ws + P.off_z;
  uint8_t* d_raw = ws + P.off_raw;
  int sms = 132;
  {
    int dev = 0;
    if (cudaGetDevice(&dev) == cudaSuccess) cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  }
  {
    ProfScope prof("png_inflate", stream);
    const int blocks = std::min((nimg + INFLATE_WARPS - 1) / INFLATE_WARPS, 4 * sms);
    png_inflate_kernel<<<blocks, 32 * INFLATE_WARPS, 0, stream>>>(ws + P.off_bytes, d_imgs, d_chunks, d_order, nimg, d_next,
                                                                 d_z, d_raw, status_out);
  }
  {
    ProfScope prof("png_unfilter", stream);
    png_unfilter_kernel<<<nimg, UNFILTER_THREADS, 0, stream>>>(d_imgs, d_raw, status_out);
  }
  {
    ProfScope prof("png_rgb", stream);
    png_rgb_kernel<<<(unsigned)((P.npix + 255) / 256), 256, 0, stream>>>(d_imgs, d_pix0, nimg, P.npix, d_raw, status_out);
  }
  e = cudaGetLastError();
  if (e != cudaSuccess) {
    set_last_error("pg_png_decode launch: %s", cudaGetErrorString(e));
    return 1;
  }
  return 0;
}

int64_t png_decode_host(const uint8_t* packed, const int64_t* offsets, const pg_png_info* infos, int n, uint8_t* rgb_out,
                        int32_t* status_out) {
  if (!packed || !offsets || !infos || !status_out || n <= 0) {
    set_last_error("pg_png_decode_host: null argument");
    return -1;
  }
  Plan P;
  if (make_plan(packed, offsets, infos, n, offsets[n], nullptr, &P)) return -1;
  for (int i = 0; i < n; ++i) status_out[i] = infos[i].status;
  std::vector<uint8_t> z((size_t)P.zbytes + 16), raw((size_t)P.rawbytes + 16);
  static thread_local InflateSmem sm;
  long long out_off = 0;
  for (PngImg im : P.imgs) {
    gather_stream(im, P.chunks.data(), packed, z.data(), 0, 1);
    long long produced;
    int st = inflate_zlib(z.data() + im.z_off, im.z_len, raw.data() + im.raw_off, im.cap, im.need, sm, 0, 1, &produced);
    uint8_t* base = raw.data() + im.raw_off;
    const long long stride = im.row_bytes + 1;
    for (long long r = 0; !st && r < im.height; ++r)
      if (base[r * stride] > 4) st = PG_PNG_BAD_FILTER;
    for (long long r = 0; !st && r < im.height; ++r)
      unfilter_span(base + r * stride + 1, r ? base + (r - 1) * stride + 1 : nullptr, base[r * stride], im.bpp, 0,
                    im.row_bytes);
    status_out[im.orig] = st;
    const long long bytes = 3LL * im.width * im.height;
    if (!st && rgb_out) {
      im.dst = rgb_out + out_off;
      im.dst_stride = 3LL * im.width;
      for (int y = 0; y < im.height; ++y)
        for (int x = 0; x < im.width; ++x) rgb_pixel(im, raw.data(), x, y);
    }
    out_off += bytes;
  }
  return out_off;
}

}  // namespace pg

extern "C" int pg_png_parse(const uint8_t* data_host, int64_t bytes, pg_png_info* info_out) {
  return pg::png_parse(data_host, bytes, info_out);
}

extern "C" size_t pg_png_workspace_bytes(const pg_png_info* infos_host, int32_t n, int64_t packed_bytes) {
  return pg::png_workspace_bytes(infos_host, n, packed_bytes);
}

extern "C" int pg_png_decode(const uint8_t* packed_host, const int64_t* offsets_host, const pg_png_info* infos_host,
                             int32_t n, const pg_image* dst_host, void* workspace, size_t workspace_bytes,
                             int32_t* status_out, void* stream) {
  return pg::png_decode(packed_host, offsets_host, infos_host, n, dst_host, workspace, workspace_bytes, status_out,
                        reinterpret_cast<cudaStream_t>(stream));
}

extern "C" int64_t pg_png_decode_host(const uint8_t* packed_host, const int64_t* offsets_host,
                                      const pg_png_info* infos_host, int32_t n, uint8_t* rgb_out, int32_t* status_out) {
  return pg::png_decode_host(packed_host, offsets_host, infos_host, n, rgb_out, status_out);
}
