// Baseline JPEG decoding on the GPU, byte-identical to Pillow's `Image.open(f).convert('RGB')` over libjpeg-turbo with
// its defaults (ISLOW IDCT, fancy upsampling).  Four stages:
//   host   marker walk (pg_jpeg_parse): frame, tables, restart interval, entropy-coded byte range, restart segments;
//   kernel 1  Huffman decode of each entropy-coded segment (a restart interval, or the whole scan without DRI): byte
//             de-stuffing, DC prediction reset per segment, quantised coefficients -> int16 blocks.  A short segment
//             takes one thread (entropy_kernel); a long one, such as a photo without restart markers, one CTA that
//             decodes it in self-synchronising chunks (chunked_kernel); both kernels may run in one call;
//   kernel 2  dequantise + jpeg_idct_islow (CONST_BITS 13, PASS1_BITS 2, 64-bit products like libjpeg's JLONG) + the
//             post-IDCT range-limit table with its `& RANGE_MASK` wrap -> component planes padded to whole MCUs;
//   kernel 3  fancy upsampling (jdsample.c h2v1 / h2v2, plain replication when the chroma width is <= 2) fused with
//             jdcolor.c's fixed-point YCbCr->RGB (SCALEBITS 16) -> uint8 RGB rows in the caller's pg_image destinations.
// Multi-scan files (progressive SOF2, or sequential in several scans; pg_jpeg_parse_multiscan) differ only in how the
// coefficients are filled: their blocks are zeroed, then multiscan_kernel decodes one thread per segment of every scan
// (DC / AC first and refinement scans with jdphuff.c's arithmetic), one launch per dependency level: a scan runs after
// every earlier scan that shares a component and a coefficient with it.  Kernels 2 and 3 are the same for both.
// Per-image status: a corrupt image stops its own segments and is not colour-converted; the other images are unaffected.
// Every read is bounded by the image's own segment, every write by its own planes and destination.
#include <cuda_runtime.h>
#include <stdarg.h>
#include <stdio.h>
#include <string.h>

#include <algorithm>
#include <atomic>
#include <climits>
#include <map>
#include <string>
#include <vector>

#include "../../include/pigeon_b200.h"
#include "prof.h"
#include "tma_host.h"

namespace pg {
namespace {

constexpr int LOOK_BITS = 9;

struct HuffTbl {                     // libjpeg d_derived_tbl: 9-bit lookahead plus the canonical maxcode / valoffset
  uint16_t look[1 << LOOK_BITS];     // (code length << 8) | symbol, 0 when the code is longer than LOOK_BITS
  int32_t maxcode[18];               // largest code of each length, -1 when none; [17] is a sentinel
  int32_t valoff[17];                // symbol index of the first code of each length, minus that code
  uint8_t vals[256];
};

struct Comp {
  int h, v;                          // sampling factors within the MCU (1 x 1 for a single-component scan)
  int bw, bh;                        // block grid, padded to whole MCUs
  int dw, dh;                        // libjpeg downsampled_width / downsampled_height
  int dc, ac;                        // indices into the batch's Huffman table array
  long long coef_off;                // first block of this component in the coefficient buffer
  long long plane_off;               // first byte of this component's plane (bw*8 x bh*8)
  int16_t q[64];                     // quantisation table in natural order, as libjpeg's ISLOW_MULT_TYPE (short)
};

struct ImgDesc {
  int orig;                          // index in the caller's batch (status array)
  int width, height, ncomp, hmax, vmax, mcux, mcuy, restart_interval;
  Comp c[3];
  uint8_t* dst;
  long long dst_stride;
};

struct Seg {
  long long start, end;              // entropy-coded bytes [start, end) in the packed input
  int img, mcu0, nmcu;
};

struct PlaneWork {                   // one component plane of one image: IDCT work items [block0, block0 + bw*bh)
  long long block0;
  int img, comp;
};

// entropy-data status codes written by the decode kernel (pg_jpeg_info.status uses the same numbering)
constexpr int ST_BAD_CODE = PG_JPEG_BAD_CODE, ST_OVERRUN = PG_JPEG_OVERRUN, ST_MARKER = PG_JPEG_UNEXPECTED_MARKER;

inline size_t align_up(size_t x, size_t a) { return (x + a - 1) / a * a; }

// jpeg_natural_order: zig-zag index -> natural (row-major) index
static const uint8_t h_natural[64] = {0,  1,  8,  16, 9,  2,  3,  10, 17, 24, 32, 25, 18, 11, 4,  5,
                                      12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6,  7,  14, 21, 28,
                                      35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51,
                                      58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};
__constant__ uint8_t c_natural[64] = {0,  1,  8,  16, 9,  2,  3,  10, 17, 24, 32, 25, 18, 11, 4,  5,
                                      12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6,  7,  14, 21, 28,
                                      35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51,
                                      58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};

// ------------------------------------------------------------------------------------------------------------------
// Host: marker walk
// ------------------------------------------------------------------------------------------------------------------

struct Why {
  char* buf;
  size_t len;
  int set(int status, const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, len, fmt, ap);
    va_end(ap);
    return status;
  }
};

inline int be16(const uint8_t* p) { return (p[0] << 8) | p[1]; }

// jdhuff.c jpeg_make_d_derived_tbl: canonical codes; a code that does not fit its length is a bad table.
bool make_huff(const uint8_t* bits, const uint8_t* vals, bool is_dc, HuffTbl* t) {
  int count = 0;
  for (int l = 0; l < 16; ++l) count += bits[l];
  if (count > 256) return false;
  if (is_dc)
    for (int i = 0; i < count; ++i)
      if (vals[i] > 15) return false;
  int huffcode[256], huffsize[256];
  int p = 0;
  for (int l = 1; l <= 16; ++l)
    for (int i = 0; i < bits[l - 1]; ++i) huffsize[p++] = l;
  int code = 0, si = 1;
  p = 0;
  while (p < count) {
    while (p < count && huffsize[p] == si) { huffcode[p++] = code; ++code; }
    if (code >= (1 << si)) return false;
    code <<= 1;
    ++si;
  }
  if (!t) return true;
  memset(t, 0, sizeof(*t));
  p = 0;
  for (int l = 1; l <= 16; ++l) {
    if (bits[l - 1]) {
      t->valoff[l] = p - huffcode[p];
      p += bits[l - 1];
      t->maxcode[l] = huffcode[p - 1];
    } else {
      t->maxcode[l] = -1;
    }
  }
  t->maxcode[17] = 0x7fffffff;
  memcpy(t->vals, vals, count);
  p = 0;
  for (int l = 1; l <= LOOK_BITS; ++l)
    for (int i = 0; i < bits[l - 1]; ++i, ++p) {
      const int base = huffcode[p] << (LOOK_BITS - l);
      for (int e = 0; e < (1 << (LOOK_BITS - l)); ++e) t->look[base + e] = (uint16_t)((l << 8) | vals[p]);
    }
  return true;
}

// Walks the entropy-coded data from `pos` to the marker that ends the scan.  Every restart marker ends a segment;
// `segs` (optional) receives each segment's [start, end).  Returns PG_JPEG_OK and the end-of-scan marker position.
int walk_scan(const uint8_t* d, int64_t n, int64_t pos, std::vector<std::pair<int64_t, int64_t>>* segs, int* nseg,
              int64_t* marker_pos, Why* why) {
  int count = 0;
  int64_t seg_start = pos;
  for (;;) {
    const void* f = pos < n ? memchr(d + pos, 0xFF, (size_t)(n - pos)) : nullptr;
    if (!f) return why->set(PG_JPEG_NO_EOI, "entropy-coded data runs to the end of the file (no EOI)");
    const int64_t q = (const uint8_t*)f - d;
    int64_t r = q + 1;
    while (r < n && d[r] == 0xFF) ++r;                 // fill bytes
    if (r >= n) return why->set(PG_JPEG_NO_EOI, "entropy-coded data runs to the end of the file (no EOI)");
    const int m = d[r];
    if (m == 0x00) { pos = r + 1; continue; }          // stuffed 0xFF
    if (m >= 0xD0 && m <= 0xD7) {
      if ((m - 0xD0) != (count & 7))
        return why->set(PG_JPEG_BAD_RST, "restart marker RST%d where RST%d was expected", m - 0xD0, count & 7);
      if (segs) segs->push_back({seg_start, q});
      ++count;
      seg_start = pos = r + 1;
      continue;
    }
    if (segs) segs->push_back({seg_start, q});
    *nseg = count + 1;
    *marker_pos = q;
    return PG_JPEG_OK;
  }
}

// One scan of a multi-scan file, as the multi-scan walk finds it: what pg_jpeg_scans reports, plus the Huffman tables
// the scan selected (copied at its SOS: a later DHT may redefine them) and, when asked for, its segments.
struct ScanRec {
  pg_jpeg_scan pub;
  uint8_t dc_bits[3][16], ac_bits[3][16];
  uint8_t dc_vals[3][256], ac_vals[3][256];
  std::vector<std::pair<int64_t, int64_t>> segs;
};

struct MultiScan {
  bool want_segs = false;
  bool multi = false;                // progressive, more than one scan, or one scan that is not all components in order
  std::vector<ScanRec> scans;
  uint16_t qt[3][64];                // quantisation table of each component, latched at its first scan (zig-zag)
  bool latched[3] = {false, false, false};
  int coef_bits[3][64];              // jdphuff.c coef_bits: bit position each coefficient has reached, -1 before any
  int tables = 0;                    // Huffman table selections over all scans
  int64_t first_scan = 0, eoi = 0;
};

int parse_scan(const uint8_t* d, int64_t n, const uint8_t* s, int len, int64_t pos, pg_jpeg_info* info, MultiScan* ms,
               bool saw_jfif, bool saw_adobe, int adobe_transform, int64_t* next, Why* why);
int finish_multiscan(pg_jpeg_info* info, MultiScan* ms, Why* why);

// The marker walk of pg_jpeg_parse; with `ms` that of pg_jpeg_parse_multiscan, which also takes SOF2 and any number
// of scans, and lets DHT / DQT / DRI / APPn / COM appear between scans.
int parse(const uint8_t* d, int64_t n, pg_jpeg_info* info, std::vector<std::pair<int64_t, int64_t>>* segs, Why* why,
          MultiScan* ms = nullptr) {
  memset(info, 0, sizeof(*info));
  if (!d || n < 4 || d[0] != 0xFF || d[1] != 0xD8) return info->status = why->set(PG_JPEG_BAD_HEADER, "no SOI marker");
  int64_t pos = 2;
  bool saw_jfif = false, saw_adobe = false, saw_sof = false;
  int adobe_transform = -1;
  for (;;) {
    const bool after_scan = ms && !ms->scans.empty();
    if (pos >= n && after_scan) return info->status = why->set(PG_JPEG_NO_EOI, "no EOI after the last scan");
    if (pos >= n) return info->status = why->set(PG_JPEG_BAD_HEADER, "truncated before the scan");
    if (d[pos] != 0xFF)
      return info->status = why->set(PG_JPEG_BAD_HEADER, "expected a marker at byte %lld", (long long)pos);
    const int64_t marker_pos = pos;
    while (pos < n && d[pos] == 0xFF) ++pos;            // fill bytes before a marker
    if (pos >= n && after_scan) return info->status = why->set(PG_JPEG_NO_EOI, "no EOI after the last scan");
    if (pos >= n) return info->status = why->set(PG_JPEG_BAD_HEADER, "truncated before the scan");
    const int m = d[pos++];
    if (m == 0x01) continue;                            // TEM: standalone, ignored as libjpeg does
    if (after_scan) {
      if (m == 0xD9) {
        ms->eoi = marker_pos;
        return info->status = finish_multiscan(info, ms, why);
      }
      if ((m >= 0xD0 && m <= 0xD7) || m == 0x00 || m == 0xD8)
        return info->status = why->set(PG_JPEG_UNEXPECTED_MARKER, "marker 0x%02X between scans", m);
      if (pos + 2 > n || be16(d + pos) < 2 || pos + be16(d + pos) > n)
        return info->status = why->set(PG_JPEG_NO_EOI, "truncated between scans");
    }
    if (m == 0xD8 || m == 0xD9 || (m >= 0xD0 && m <= 0xD7) || m == 0x00)
      return info->status = why->set(PG_JPEG_BAD_HEADER, "marker 0x%02X before the first scan", m);
    if (pos + 2 > n) return info->status = why->set(PG_JPEG_BAD_HEADER, "truncated marker 0x%02X", m);
    const int L = be16(d + pos);
    if (L < 2 || pos + L > n) return info->status = why->set(PG_JPEG_BAD_HEADER, "truncated marker segment 0x%02X", m);
    const uint8_t* s = d + pos + 2;
    const int len = L - 2;
    pos += L;
    if (m >= 0xC0 && m <= 0xCF && m != 0xC4 && m != 0xC8 && m != 0xCC) {
      if (saw_sof) return info->status = why->set(PG_JPEG_BAD_HEADER, "second frame header");
      saw_sof = true;
      info->sof = m;
      if (len < 6) return info->status = why->set(PG_JPEG_BAD_HEADER, "short frame header");
      info->precision = s[0];
      info->height = be16(s + 1);
      info->width = be16(s + 3);
      info->components = s[5];
      if (ms && m == 0xC2) ms->multi = true;
      if (m != 0xC0 && m != 0xC1 && !(ms && m == 0xC2)) {
        const char* kind = m == 0xC2 || m == 0xC6 || m == 0xCA || m == 0xCE ? "progressive"
                           : m == 0xC3 || m == 0xC7 || m == 0xCB || m == 0xCF ? "lossless"
                                                                               : "hierarchical or arithmetic";
        return info->status = why->set(PG_JPEG_UNSUPPORTED, "SOF%d (%s) is not decoded", m - 0xC0, kind);
      }
      if (len != 6 + 3 * info->components || info->components < 1)
        return info->status = why->set(PG_JPEG_BAD_HEADER, "frame header length %d for %d components", len, info->components);
      if (info->precision != 8)
        return info->status = why->set(PG_JPEG_UNSUPPORTED, "%d-bit samples are not decoded", info->precision);
      if (info->height == 0) return info->status = why->set(PG_JPEG_UNSUPPORTED, "height defined by DNL is not decoded");
      if (info->width == 0) return info->status = why->set(PG_JPEG_BAD_HEADER, "zero width");
      if (info->components != 1 && info->components != 3)
        return info->status = why->set(PG_JPEG_UNSUPPORTED, "%d components are not decoded", info->components);
      for (int c = 0; c < info->components; ++c) {
        info->component_id[c] = s[6 + 3 * c];
        info->h_samp[c] = s[7 + 3 * c] >> 4;
        info->v_samp[c] = s[7 + 3 * c] & 15;
        info->quant_table[c] = s[8 + 3 * c];
        if (info->h_samp[c] < 1 || info->h_samp[c] > 4 || info->v_samp[c] < 1 || info->v_samp[c] > 4 ||
            info->quant_table[c] > 3)
          return info->status = why->set(PG_JPEG_BAD_HEADER, "bad sampling factor or table of component %d", c);
      }
      if (info->components == 3) {
        const int h = info->h_samp[0], v = info->v_samp[0];
        const bool luma_ok = (h == 1 && v == 1) || (h == 2 && v == 1) || (h == 2 && v == 2);
        for (int c = 1; c < 3; ++c)
          if (!luma_ok || info->h_samp[c] != 1 || info->v_samp[c] != 1)
            return info->status = why->set(PG_JPEG_UNSUPPORTED, "sampling %dx%d,%dx%d,%dx%d is not decoded", h, v,
                                           info->h_samp[1], info->v_samp[1], info->h_samp[2], info->v_samp[2]);
      }
      continue;
    }
    switch (m) {
      case 0xC4: {                                      // DHT
        int o = 0;
        while (o < len) {
          const int tc = s[o] >> 4, th = s[o] & 15;
          if (tc > 1 || th > 3 || o + 17 > len) return info->status = why->set(PG_JPEG_BAD_HEADER, "bad DHT segment");
          int count = 0;
          for (int i = 0; i < 16; ++i) count += s[o + 1 + i];
          if (count > 256 || o + 17 + count > len) return info->status = why->set(PG_JPEG_BAD_HEADER, "bad DHT segment");
          uint8_t* bits = tc ? info->ac_bits[th] : info->dc_bits[th];
          uint8_t* vals = tc ? info->ac_vals[th] : info->dc_vals[th];
          memcpy(bits, s + o + 1, 16);
          memset(vals, 0, 256);
          memcpy(vals, s + o + 17, count);
          info->table_mask |= 1 << ((tc ? 8 : 4) + th);
          o += 17 + count;
        }
        break;
      }
      case 0xDB: {                                      // DQT, 8- or 16-bit entries
        int o = 0;
        while (o < len) {
          const int pq = s[o] >> 4, tq = s[o] & 15;
          if (pq > 1 || tq > 3 || o + 1 + 64 * (pq + 1) > len)
            return info->status = why->set(PG_JPEG_BAD_HEADER, "bad DQT segment");
          for (int k = 0; k < 64; ++k) info->qt[tq][k] = (uint16_t)(pq ? be16(s + o + 1 + 2 * k) : s[o + 1 + k]);
          info->table_mask |= 1 << tq;
          o += 1 + 64 * (pq + 1);
        }
        break;
      }
      case 0xDD:                                        // DRI
        if (len != 2) return info->status = why->set(PG_JPEG_BAD_HEADER, "bad DRI segment");
        info->restart_interval = be16(s);
        break;
      case 0xE0:                                        // jdmarker.c examine_app0
        if (len >= 14 && memcmp(s, "JFIF\0", 5) == 0) saw_jfif = true;
        break;
      case 0xEE:                                        // jdmarker.c examine_app14
        if (len >= 12 && memcmp(s, "Adobe", 5) == 0) { saw_adobe = true; adobe_transform = s[11]; }
        break;
      case 0xC8: case 0xCC:
        return info->status = why->set(PG_JPEG_UNSUPPORTED, "arithmetic coding is not decoded");
      case 0xDC:
        return info->status = why->set(PG_JPEG_UNSUPPORTED, "height defined by DNL is not decoded");
      case 0xDA: {                                      // SOS
        if (!saw_sof) return info->status = why->set(PG_JPEG_BAD_HEADER, "scan before the frame header");
        if (ms) {
          const int st = parse_scan(d, n, s, len, pos, info, ms, saw_jfif, saw_adobe, adobe_transform, &pos, why);
          if (st) return info->status = st;
          break;
        }
        const int ns = len >= 1 ? s[0] : 0;
        if (len != 4 + 2 * ns || ns < 1) return info->status = why->set(PG_JPEG_BAD_HEADER, "bad SOS segment");
        if (ns != info->components)
          return info->status = why->set(PG_JPEG_UNSUPPORTED, "a scan of %d of %d components (more than one scan)", ns,
                                         info->components);
        for (int c = 0; c < ns; ++c) {
          if (s[1 + 2 * c] != info->component_id[c])
            return info->status = why->set(PG_JPEG_BAD_HEADER, "scan components differ from the frame's");
          info->dc_table[c] = s[2 + 2 * c] >> 4;
          info->ac_table[c] = s[2 + 2 * c] & 15;
          if (info->dc_table[c] > 3 || info->ac_table[c] > 3)
            return info->status = why->set(PG_JPEG_BAD_HEADER, "bad Huffman table index");
          if (!(info->table_mask & (1 << info->quant_table[c])) || !(info->table_mask & (16 << info->dc_table[c])) ||
              !(info->table_mask & (256 << info->ac_table[c])))
            return info->status = why->set(PG_JPEG_BAD_HEADER, "component %d uses an undefined table", c);
          if (!make_huff(info->dc_bits[info->dc_table[c]], info->dc_vals[info->dc_table[c]], true, nullptr) ||
              !make_huff(info->ac_bits[info->ac_table[c]], info->ac_vals[info->ac_table[c]], false, nullptr))
            return info->status = why->set(PG_JPEG_BAD_HEADER, "invalid Huffman table");
        }
        const uint8_t* t = s + 1 + 2 * ns;
        if (t[0] != 0 || t[1] != 63 || t[2] != 0)
          return info->status = why->set(PG_JPEG_BAD_HEADER, "spectral selection %d..%d / approximation %d in a sequential scan",
                                         t[0], t[1], t[2]);
        // jdapimin.c default_decompress_parms: which 3-component files libjpeg treats as RGB
        if (info->components == 3 && !saw_jfif) {
          const bool rgb = saw_adobe ? adobe_transform == 0
                                     : (info->component_id[0] == 'R' && info->component_id[1] == 'G' &&
                                        info->component_id[2] == 'B');
          if (rgb) return info->status = why->set(PG_JPEG_UNSUPPORTED, "RGB colour transform is not decoded");
        }
        info->scan_offset = pos;
        int nseg = 0;
        int64_t mp = 0;
        int st = walk_scan(d, n, pos, segs, &nseg, &mp, why);
        if (st) return info->status = st;
        info->scan_bytes = mp - pos;
        info->num_segments = nseg;
        const int hmax = info->components == 3 ? info->h_samp[0] : 1, vmax = info->components == 3 ? info->v_samp[0] : 1;
        const long long mcus = (long long)((info->width + 8 * hmax - 1) / (8 * hmax)) * ((info->height + 8 * vmax - 1) / (8 * vmax));
        const long long want = info->restart_interval ? (mcus + info->restart_interval - 1) / info->restart_interval : 1;
        if (nseg != want)
          return info->status = why->set(PG_JPEG_BAD_RST, "%d entropy-coded segments where %lld were expected", nseg, want);
        // after the scan: only EOI may end the file; another SOS is a second scan
        int64_t p = mp;
        for (;;) {
          while (p < n && d[p] == 0xFF) ++p;
          if (p >= n) return info->status = why->set(PG_JPEG_NO_EOI, "no EOI after the scan");
          const int mm = d[p++];
          if (mm == 0xD9) return info->status = PG_JPEG_OK;
          if (mm == 0xDA) return info->status = why->set(PG_JPEG_UNSUPPORTED, "more than one scan");
          if ((mm >= 0xD0 && mm <= 0xD7) || mm == 0x01 || mm == 0x00)
            return info->status = why->set(PG_JPEG_UNEXPECTED_MARKER, "marker 0x%02X after the scan", mm);
          if (p + 2 > n || be16(d + p) < 2 || p + be16(d + p) > n)
            return info->status = why->set(PG_JPEG_NO_EOI, "truncated after the scan");
          p += be16(d + p);
          if (p < n && d[p] != 0xFF) return info->status = why->set(PG_JPEG_BAD_HEADER, "garbage after the scan");
        }
      }
      default:
        if ((m >= 0xE0 && m <= 0xEF) || m == 0xFE) break;   // APPn / COM: skipped
        return info->status = why->set(PG_JPEG_BAD_HEADER, "unknown marker 0x%02X", m);
    }
  }
}

// Blocks per row and rows of the scan's MCU grid: the frame's MCUs when interleaved, else the single component's own
// blocks, ceil(downsampled size / 8) per side (jdinput.c per_scan_setup).
void scan_grid(const pg_jpeg_info* info, int ncomp_scan, int c, int* cols, int* rows) {
  const int hmax = info->components == 3 ? info->h_samp[0] : 1, vmax = info->components == 3 ? info->v_samp[0] : 1;
  if (ncomp_scan > 1) {
    *cols = (info->width + 8 * hmax - 1) / (8 * hmax);
    *rows = (info->height + 8 * vmax - 1) / (8 * vmax);
    return;
  }
  const int h = info->components == 3 ? info->h_samp[c] : 1, v = info->components == 3 ? info->v_samp[c] : 1;
  *cols = (int)(((long long)info->width * h + 8LL * hmax - 1) / (8LL * hmax));
  *rows = (int)(((long long)info->height * v + 8LL * vmax - 1) / (8LL * vmax));
}

// One SOS of the multi-scan walk (s: its segment, pos: the first entropy-coded byte).  Validates the scan as libjpeg
// 3.1 does at the start of its pass (jdphuff.c start_pass_phuff_decoder, jdhuff.c start_pass_huff_decoder, jdinput.c
// latch_quant_tables), walks its entropy-coded data and sets *next to the marker that ends it.
int parse_scan(const uint8_t* d, int64_t n, const uint8_t* s, int len, int64_t pos, pg_jpeg_info* info, MultiScan* ms,
               bool saw_jfif, bool saw_adobe, int adobe_transform, int64_t* next, Why* why) {
  const bool progressive = info->sof == 0xC2;
  const int ns = len >= 1 ? s[0] : 0;
  if (len != 4 + 2 * ns || ns < 1 || ns > info->components) return why->set(PG_JPEG_BAD_HEADER, "bad SOS segment");
  if ((int)ms->scans.size() >= PG_JPEG_MAX_SCANS)
    return why->set(PG_JPEG_UNSUPPORTED, "more than %d scans", PG_JPEG_MAX_SCANS);
  ms->scans.emplace_back();
  ScanRec& sc = ms->scans.back();
  memset(&sc.pub, 0, sizeof(sc.pub));
  pg_jpeg_scan& p = sc.pub;
  p.components = ns;
  const uint8_t* t = s + 1 + 2 * ns;
  p.ss = t[0];
  p.se = t[1];
  p.ah = t[2] >> 4;
  p.al = t[2] & 15;
  if (ns != info->components || ms->scans.size() > 1) ms->multi = true;
  for (int j = 0; j < ns; ++j) {
    int c = 0;
    while (c < info->components && info->component_id[c] != s[1 + 2 * j]) ++c;
    if (c == info->components) return why->set(PG_JPEG_BAD_HEADER, "scan component id %d is not in the frame", s[1 + 2 * j]);
    for (int i = 0; i < j; ++i)
      if (p.component[i] == c) return why->set(PG_JPEG_BAD_HEADER, "component id %d twice in one scan", s[1 + 2 * j]);
    if (c != j) ms->multi = true;
    p.component[j] = c;
    info->dc_table[c] = s[2 + 2 * j] >> 4;
    info->ac_table[c] = s[2 + 2 * j] & 15;
    if (info->dc_table[c] > 3 || info->ac_table[c] > 3) return why->set(PG_JPEG_BAD_HEADER, "bad Huffman table index");
  }
  const bool dc_band = p.ss == 0;
  if (progressive) {                                    // JERR_BAD_PROGRESSION
    const bool bad = (dc_band ? p.se != 0 : (p.ss > p.se || p.se > 63 || ns != 1)) ||
                     (p.ah != 0 && p.al != p.ah - 1) || p.al > 13;
    if (bad) return why->set(PG_JPEG_BAD_HEADER, "bad progression: Ss=%d Se=%d Ah=%d Al=%d", p.ss, p.se, p.ah, p.al);
  } else if (p.ss != 0 || p.se != 63 || t[2] != 0) {
    return why->set(PG_JPEG_BAD_HEADER, "spectral selection %d..%d / approximation %d in a sequential scan", t[0], t[1],
                    t[2]);
  }
  if (ms->scans.size() == 1) {
    ms->first_scan = pos;
    if (info->components == 3 && !saw_jfif) {           // as in the single-scan walk
      const bool rgb = saw_adobe ? adobe_transform == 0
                                 : (info->component_id[0] == 'R' && info->component_id[1] == 'G' &&
                                    info->component_id[2] == 'B');
      if (rgb) return why->set(PG_JPEG_UNSUPPORTED, "RGB colour transform is not decoded");
    }
  }
  const bool need_dc = !progressive || (dc_band && p.ah == 0), need_ac = !progressive || !dc_band;
  for (int j = 0; j < ns; ++j) {
    const int c = p.component[j];
    if (!ms->latched[c]) {
      if (!(info->table_mask & (1 << info->quant_table[c])))
        return why->set(PG_JPEG_BAD_HEADER, "component %d uses an undefined table", c);
      memcpy(ms->qt[c], info->qt[info->quant_table[c]], sizeof(ms->qt[c]));
      ms->latched[c] = true;
    }
    const int td = info->dc_table[c], ta = info->ac_table[c];
    if ((need_dc && !(info->table_mask & (16 << td))) || (need_ac && !(info->table_mask & (256 << ta))))
      return why->set(PG_JPEG_BAD_HEADER, "component %d uses an undefined table", c);
    if ((need_dc && !make_huff(info->dc_bits[td], info->dc_vals[td], true, nullptr)) ||
        (need_ac && !make_huff(info->ac_bits[ta], info->ac_vals[ta], false, nullptr)))
      return why->set(PG_JPEG_BAD_HEADER, "invalid Huffman table");
    memcpy(sc.dc_bits[j], info->dc_bits[td], 16);
    memcpy(sc.dc_vals[j], info->dc_vals[td], 256);
    memcpy(sc.ac_bits[j], info->ac_bits[ta], 16);
    memcpy(sc.ac_vals[j], info->ac_vals[ta], 256);
    ms->tables += need_dc + need_ac;
    // progression state (jdphuff.c): what libjpeg only warns about is left to the host decoder
    if (progressive && !dc_band && ms->coef_bits[c][0] < 0)
      return why->set(PG_JPEG_UNSUPPORTED, "bogus progression: AC scan of component %d before its DC scan", c);
    for (int k = p.ss; k <= p.se; ++k) {
      const int cur = ms->coef_bits[c][k];
      if (progressive && p.ah != (cur < 0 ? 0 : cur))
        return why->set(PG_JPEG_UNSUPPORTED, "bogus progression: scan with Ah=%d for coefficient %d of component %d at bit %d",
                        p.ah, k, c, cur);
      if (progressive && p.ah == 0 && cur >= 0)
        return why->set(PG_JPEG_UNSUPPORTED, "coefficient %d of component %d is sent twice", k, c);
      ms->coef_bits[c][k] = p.al;
    }
  }
  // dependency level: after every earlier scan that shares a component and a coefficient position
  p.level = 1;
  for (size_t i = 0; i + 1 < ms->scans.size(); ++i) {
    const pg_jpeg_scan& q = ms->scans[i].pub;
    if (q.ss > p.se || p.ss > q.se) continue;
    bool shared = false;
    for (int a = 0; a < q.components; ++a)
      for (int b = 0; b < ns; ++b) shared |= q.component[a] == p.component[b];
    if (shared) p.level = std::max(p.level, q.level + 1);
  }
  p.restart_interval = info->restart_interval;
  int nseg = 0;
  int64_t mp = 0;
  const int st = walk_scan(d, n, pos, ms->want_segs ? &sc.segs : nullptr, &nseg, &mp, why);
  if (st) return st;
  int cols = 0, rows = 0;
  scan_grid(info, ns, p.component[0], &cols, &rows);
  const long long mcus = (long long)cols * rows;
  const long long want = p.restart_interval ? (mcus + p.restart_interval - 1) / p.restart_interval : 1;
  if (nseg != want)
    return why->set(PG_JPEG_BAD_RST, "scan %d: %d entropy-coded segments where %lld were expected",
                    (int)ms->scans.size(), nseg, want);
  p.num_segments = nseg;
  *next = mp;
  return PG_JPEG_OK;
}

// At the EOI of a multi-scan file: every coefficient of every component sent and refined to bit 0 (else libjpeg would
// smooth the blocks of a progressive file, or leave a component blank), then the info fields of a multi-scan file.
int finish_multiscan(pg_jpeg_info* info, MultiScan* ms, Why* why) {
  for (int c = 0; c < info->components; ++c)
    for (int k = 0; k < 64; ++k)
      if (ms->coef_bits[c][k] != 0) {
        if (info->sof != 0xC2) return why->set(PG_JPEG_UNSUPPORTED, "component %d has no scan", c);
        return why->set(PG_JPEG_UNSUPPORTED, "incomplete progression: coefficient %d of component %d %s", k, c,
                        ms->coef_bits[c][k] < 0 ? "is never sent" : "is not refined to bit 0");
      }
  long long segs = 0;
  for (const ScanRec& sc : ms->scans) segs += sc.pub.num_segments;
  if (segs > 0x7fffffff) return why->set(PG_JPEG_UNSUPPORTED, "too many entropy-coded segments");
  info->num_segments = (int32_t)segs;
  info->restart_interval = ms->scans[0].pub.restart_interval;
  info->scan_offset = ms->first_scan;
  info->scan_bytes = ms->eoi - ms->first_scan;
  info->table_mask = (info->table_mask & 0xFFF) | PG_JPEG_MULTISCAN | (ms->tables << 16);
  return PG_JPEG_OK;
}

// pg_jpeg_parse_multiscan: the single-scan walk's result for every file that is not multi-scan (so that a file
// pg_jpeg_parse accepts gets the identical info), else the multi-scan walk's.
int parse_multiscan(const uint8_t* d, int64_t n, pg_jpeg_info* info, MultiScan* ms, Why* why) {
  const int st = parse(d, n, info, nullptr, why);
  if (st == PG_JPEG_OK) return st;
  std::vector<char> msg2(why->len);
  Why why2{msg2.data(), msg2.size()};
  msg2[0] = 0;
  pg_jpeg_info mi;
  for (int c = 0; c < 3; ++c)
    for (int k = 0; k < 64; ++k) ms->coef_bits[c][k] = -1;
  const int st2 = parse(d, n, &mi, nullptr, &why2, ms);
  if (!ms->multi) return st;
  *info = mi;
  snprintf(why->buf, why->len, "%s", msg2.data());
  return st2;
}

// ------------------------------------------------------------------------------------------------------------------
// Device: entropy decode
// ------------------------------------------------------------------------------------------------------------------

struct BitReader {
  const uint8_t* p;
  const uint8_t* end;
  uint64_t acc;                      // MSB-aligned
  int nbits;
  int zeros;                         // zero bytes fed past the segment end
  int err;

  __host__ __device__ __forceinline__ void fill() {
    while (nbits <= 56) {
      uint32_t c = 0;
      if (p < end) {
        c = *p++;
        if (c == 0xFF) {             // jdhuff.c: skip fill bytes; FF 00 is a data 0xFF, anything else a marker
          while (p < end && *p == 0xFF) ++p;
          if (p < end && *p == 0x00) {
            ++p;
          } else {
            err = ST_MARKER;
            p = end;
            c = 0;
          }
        }
      } else {
        ++zeros;
      }
      acc |= (uint64_t)c << (56 - nbits);
      nbits += 8;
    }
  }
  __host__ __device__ __forceinline__ int get(int s) {           // s in 1..16, after fill()
    const int r = (int)(acc >> (64 - s));
    acc <<= s;
    nbits -= s;
    return r;
  }
  __host__ __device__ __forceinline__ bool overrun() const { return zeros * 8 > nbits; }
};

template <class Reader>
__host__ __device__ __forceinline__ int huff_decode(Reader& br, const HuffTbl& t) {
  const int e = t.look[br.acc >> (64 - LOOK_BITS)];
  if (e >> 8) {
    br.acc <<= (e >> 8);
    br.nbits -= (e >> 8);
    return e & 0xFF;
  }
  int l = LOOK_BITS + 1;
  int code = (int)(br.acc >> (64 - l));
  while (code > t.maxcode[l]) {
    if (++l > 16) { br.err = ST_BAD_CODE; return 0; }
    code = (int)(br.acc >> (64 - l));
  }
  br.acc <<= l;
  br.nbits -= l;
  return t.vals[(t.valoff[l] + code) & 0xFF];
}

__host__ __device__ __forceinline__ int huff_extend(int x, int s) { return x < (1 << (s - 1)) ? x + (int)(~0u << s) + 1 : x; }

// Decodes the MCUs of one entropy-coded segment into int16 blocks (natural order); `blk` is 64 int16 of scratch.
// Returns 0 or the segment's PG_JPEG_* error.
__host__ __device__ inline int decode_segment(const uint8_t* __restrict__ bytes, const ImgDesc& im,
                                              const HuffTbl* __restrict__ tbls, const Seg& sg, int16_t* blk,
                                              int16_t* __restrict__ coef) {
#ifdef __CUDA_ARCH__
  const uint8_t* natural = c_natural;
#else
  const uint8_t* natural = h_natural;
#endif
  BitReader br{bytes + sg.start, bytes + sg.end, 0, 0, 0, 0};
  int pred[3] = {0, 0, 0};
  const int ncomp = im.ncomp;
  for (int mi = 0; mi < sg.nmcu && !br.err; ++mi) {
    const int mcu = sg.mcu0 + mi;
    const int my = mcu / im.mcux, mx = mcu - my * im.mcux;
    for (int c = 0; c < ncomp && !br.err; ++c) {
      const Comp& cp = im.c[c];
      const HuffTbl& dct = tbls[cp.dc];
      const HuffTbl& act = tbls[cp.ac];
      for (int bv = 0; bv < cp.v && !br.err; ++bv)
        for (int bh = 0; bh < cp.h && !br.err; ++bh) {
          for (int i = 0; i < 64; i += 8) *reinterpret_cast<uint4*>(blk + i) = make_uint4(0, 0, 0, 0);
          br.fill();
          int s = huff_decode(br, dct);                 // DC difference, predicted per component within the segment
          if (s) s = huff_extend(br.get(s), s);
          pred[c] += s;
          blk[0] = (int16_t)pred[c];
          for (int k = 1; k < 64;) {
            if (br.nbits < 32) br.fill();
            const int rs = huff_decode(br, act);
            const int r = rs >> 4;
            s = rs & 15;
            if (s) {
              k += r;
              if (k > 63) { br.err = ST_BAD_CODE; break; }
              blk[natural[k]] = (int16_t)huff_extend(br.get(s), s);
              ++k;
            } else {
              if (r != 15) break;
              k += 16;
            }
          }
          if (br.err) break;
          const long long b = cp.coef_off + (long long)(my * cp.v + bv) * cp.bw + (mx * cp.h + bh);
          uint4* o = reinterpret_cast<uint4*>(coef + b * 64);
          for (int i = 0; i < 8; ++i) o[i] = reinterpret_cast<const uint4*>(blk)[i];
        }
    }
    if (!br.err && br.overrun()) br.err = ST_OVERRUN;
  }
  return br.err;
}

constexpr int ENTROPY_THREADS = 32;

// One thread per entropy-coded segment; `lanes` segments per warp (fewer than 32 when the batch has few segments, so
// that they spread over the SMs instead of sharing one warp).
__global__ void __launch_bounds__(ENTROPY_THREADS)
entropy_kernel(const uint8_t* __restrict__ bytes, const ImgDesc* __restrict__ imgs, const HuffTbl* __restrict__ tbls,
               const Seg* __restrict__ segs, int nseg, int lanes, int16_t* __restrict__ coef, int* __restrict__ status) {
  __shared__ __align__(16) int16_t blk_smem[ENTROPY_THREADS][64];
  const int lane = threadIdx.x;
  if (lane >= lanes) return;
  const int si = blockIdx.x * lanes + lane;
  if (si >= nseg) return;
  const Seg sg = segs[si];
  const ImgDesc& im = imgs[sg.img];
  const int err = decode_segment(bytes, im, tbls, sg, blk_smem[lane], coef);
  if (err) atomicCAS(status + im.orig, 0, err);
}

// ------------------------------------------------------------------------------------------------------------------
// Device: chunked entropy decode of long single-scan segments (self-synchronising Huffman decoding)
// ------------------------------------------------------------------------------------------------------------------
//
// After Weissenberger and Schmidt, "Massively parallel Huffman decoding on GPUs" (ICPP 2018).  One CTA per segment:
//   1. de-stuff the segment (FF 00 -> FF, fill bytes dropped) into plain bytes, so that a chunk can start at any bit;
//   2. cut those bytes into chunks.  A chunk owns the blocks whose DC code starts inside it; its state at a block start
//      is (bit offset, block slot within the MCU), and its exit state is the state at the first block start at or after
//      its end.  Round 0 decodes every chunk from a guess (its first bit, slot 0; chunk 0 from the true state); each
//      later round re-decodes the chunks whose start (the previous chunk's exit) changed, until none did.  Huffman codes
//      resynchronise within a few codes, so that takes few rounds; it never takes more than one round per chunk;
//   3. block-wide exclusive scans of the blocks each chunk starts and of its DC differences per component give every
//      chunk its absolute first block and DC predictors; every chunk decodes once more and writes its blocks.
// Only that last pass reports errors: the first event in stream order that decode_segment meets, a bad code at its
// block or an overrun at the end of its MCU.  A speculative decode that meets a bad code reports nothing (chunk_sync).
// All synchronisation is __syncthreads within the CTA.

constexpr int CHUNK_THREADS = 256;
constexpr int MIN_CHUNK_BYTES = 512;    // automatic chunk size: max(MIN_CHUNK_BYTES, de-stuffed bytes / CHUNK_THREADS)
constexpr int MAX_CHUNKS = 1024;        // chunk states live in shared memory; a forced size is raised to fit them
constexpr long long NO_EVENT = LLONG_MAX;

// Segments of at least this many compressed bytes take the chunked kernel under the automatic schedule.
constexpr long long LONG_SEGMENT_BYTES = 32768;

// Process-wide entropy-kernel choice (pg_jpeg_set_schedule): 0 = automatic, 1 = one thread per segment, 2 = chunked
// for every single-scan segment; a nonzero chunk size forces the chunks' size in bytes.
std::atomic<int> g_jpeg_schedule{0};
std::atomic<int> g_jpeg_chunk_bytes{0};

// jdhuff.c's de-stuffing as BitReader::fill applies it: after an FF, further FF fill bytes and one 00 are dropped.  A
// segment holds no marker (walk_scan ends it at the first FF of one), so every FF is followed by FF or 00.
__host__ __device__ __forceinline__ bool stuffing_byte(const uint8_t* d, long long i) {
  return i > 0 && d[i - 1] == 0xFF && (d[i] == 0xFF || d[i] == 0x00);
}

__host__ __device__ inline long long destuff_count(const uint8_t* d, long long i0, long long i1) {
  long long n = 0;
  for (long long i = i0; i < i1; ++i) n += !stuffing_byte(d, i);
  return n;
}

__host__ __device__ inline void destuff_copy(const uint8_t* d, long long i0, long long i1, uint8_t* out) {
  for (long long i = i0; i < i1; ++i)
    if (!stuffing_byte(d, i)) *out++ = d[i];
}

// Chunk size in bytes and chunk count of a segment of `len` de-stuffed bytes; `forced` > 0 is the forced size.
__host__ __device__ inline void chunk_geometry(long long len, int forced, long long* cb, int* nch) {
  long long c = forced > 0 ? forced : std::max<long long>(MIN_CHUNK_BYTES, (len + CHUNK_THREADS - 1) / CHUNK_THREADS);
  if ((len + c - 1) / c > MAX_CHUNKS) c = (len + MAX_CHUNKS - 1) / MAX_CHUNKS;
  *cb = c;
  *nch = (int)std::max<long long>(1, (len + c - 1) / c);
}

// BitReader over de-stuffed bytes, started at any bit; zero bytes past the end, as BitReader feeds them.
struct PlainBits {
  const uint8_t* p;
  const uint8_t* end;
  uint64_t acc;
  int nbits;
  int err;
  long long past;                    // zero bytes fed past the end

  __host__ __device__ __forceinline__ void start(const uint8_t* data, long long len, long long bit) {
    const long long byte = bit >> 3;
    p = data + std::min(byte, len);
    end = data + len;
    past = byte > len ? byte - len : 0;
    acc = 0;
    nbits = 0;
    err = 0;
    fill();
    acc <<= (bit & 7);
    nbits -= (int)(bit & 7);
  }
  __host__ __device__ __forceinline__ void fill() {
    while (nbits <= 56) {
      uint32_t c = 0;
      if (p < end) c = *p++; else ++past;
      acc |= (uint64_t)c << (56 - nbits);
      nbits += 8;
    }
  }
  __host__ __device__ __forceinline__ int get(int s) {
    const int r = (int)(acc >> (64 - s));
    acc <<= s;
    nbits -= s;
    return r;
  }
  __host__ __device__ __forceinline__ long long bit(const uint8_t* data) const { return ((p - data) + past) * 8 - nbits; }
};

// One segment as its chunks see it: the de-stuffed bytes, the MCU's block slots and where each slot's blocks go.
struct ChunkSeg {
  const uint8_t* data;
  long long len;                     // de-stuffed bytes
  const HuffTbl* tb;                 // DC and AC table of component c at tb[2c], tb[2c + 1]
  int bpm, total, mcu0, mcux;        // blocks per MCU, blocks of the segment, its first MCU, MCUs per row
  int comp[6];                       // component of each slot
  long long off[6];                  // first block of the slot's component + its offset within the MCU
  int rowstep[6], colstep[6];        // blocks per MCU row (v * bw) and per MCU column (h) of the slot's component
};

__host__ __device__ inline void chunk_seg_init(ChunkSeg& cs, const ImgDesc& im, const Seg& sg, const uint8_t* data,
                                               long long len, const HuffTbl* tb) {
  cs.data = data;
  cs.len = len;
  cs.tb = tb;
  cs.mcu0 = sg.mcu0;
  cs.mcux = im.mcux;
  int s = 0;
  for (int c = 0; c < im.ncomp; ++c)
    for (int bv = 0; bv < im.c[c].v; ++bv)
      for (int bh = 0; bh < im.c[c].h; ++bh, ++s) {
        cs.comp[s] = c;
        cs.off[s] = im.c[c].coef_off + (long long)bv * im.c[c].bw + bh;
        cs.rowstep[s] = im.c[c].v * im.c[c].bw;
        cs.colstep[s] = im.c[c].h;
      }
  cs.bpm = s;
  cs.total = sg.nmcu * s;
}

// One block, as decode_segment decodes it; with STORE its AC coefficients go to `blk` (zeroed first).  Returns true on a
// bad code, where decode_segment stops without storing the block.
template <bool STORE>
__host__ __device__ __forceinline__ bool chunk_block(PlainBits& br, const HuffTbl& dct, const HuffTbl& act, int16_t* blk,
                                                     int* diff) {
#ifdef __CUDA_ARCH__
  const uint8_t* natural = c_natural;
#else
  const uint8_t* natural = h_natural;
#endif
  br.fill();
  int s = huff_decode(br, dct);
  if (br.err) return true;
  if (s) s = huff_extend(br.get(s), s);
  *diff = s;
  if (STORE)
    for (int i = 0; i < 64; i += 8) *reinterpret_cast<uint4*>(blk + i) = make_uint4(0, 0, 0, 0);
  for (int k = 1; k < 64;) {
    if (br.nbits < 32) br.fill();
    const int rs = huff_decode(br, act);
    if (br.err) return true;
    const int r = rs >> 4;
    s = rs & 15;
    if (s) {
      k += r;
      if (k > 63) return true;
      const int v = br.get(s);
      if (STORE) blk[natural[k]] = (int16_t)huff_extend(v, s);
      ++k;
    } else {
      if (r != 15) break;
      k += 16;
    }
  }
  return false;
}

struct ChunkRun {
  long long exit;                    // (bit << 3) | slot
  int count;                         // blocks started
  unsigned dc0, dc1, dc2;            // DC differences per component, modulo 2^32 like decode_segment's int predictor
};

// Synchronisation pass: decodes the blocks that start in [state's bit, end_bit) without writing them.  A bad code means
// the decode started out of step: it resumes one bit further on, at the same slot, which keeps it resynchronising.  A
// decode from the true state meets one only where decode_segment stops with the image's error; nothing after that
// point is written or reported, so what the pass counts there does not matter.
__host__ __device__ inline ChunkRun chunk_sync(const ChunkSeg& cs, long long state, long long end_bit) {
  ChunkRun r{0, 0, 0u, 0u, 0u};
  long long bit = state >> 3;
  int slot = (int)(state & 7);
  PlainBits br;
  br.start(cs.data, cs.len, bit);
  while (bit < end_bit) {
    const int c = cs.comp[slot];
    int diff = 0;
    if (chunk_block<false>(br, cs.tb[2 * c], cs.tb[2 * c + 1], nullptr, &diff)) {
      bit = br.bit(cs.data) + 1;
      br.start(cs.data, cs.len, bit);
      continue;
    }
    if (c == 0) r.dc0 += diff; else if (c == 1) r.dc1 += diff; else r.dc2 += diff;
    ++r.count;
    slot = slot + 1 == cs.bpm ? 0 : slot + 1;
    bit = br.bit(cs.data);
  }
  r.exit = (bit << 3) | slot;
  return r;
}

// Final pass of one synchronised chunk: block `block` of the segment onwards, with DC predictors p0..p2, written to
// `coef` through `blk` (64 int16 of scratch).  Returns the chunk's first event, 2 * block for a bad code and
// 2 * (last block of the MCU) + 1 for an MCU that ends past the data, or NO_EVENT.
__host__ __device__ inline long long chunk_final(const ChunkSeg& cs, long long state, long long end_bit, long long block,
                                                 unsigned p0, unsigned p1, unsigned p2, int16_t* blk,
                                                 int16_t* __restrict__ coef) {
  long long bit = state >> 3;
  int slot = (int)(state & 7);
  PlainBits br;
  br.start(cs.data, cs.len, bit);
  const long long data_bits = cs.len * 8;
  while (block < cs.total && bit < end_bit) {
    const int c = cs.comp[slot];
    int diff = 0;
    if (chunk_block<true>(br, cs.tb[2 * c], cs.tb[2 * c + 1], blk, &diff)) return 2 * block;
    unsigned pred;
    if (c == 0) pred = p0 += diff; else if (c == 1) pred = p1 += diff; else pred = p2 += diff;
    blk[0] = (int16_t)pred;
    const int mcu = cs.mcu0 + (int)(block / cs.bpm);
    const int my = mcu / cs.mcux, mx = mcu - my * cs.mcux;
    const long long b = cs.off[slot] + (long long)my * cs.rowstep[slot] + (long long)mx * cs.colstep[slot];
    uint4* o = reinterpret_cast<uint4*>(coef + b * 64);
    for (int i = 0; i < 8; ++i) o[i] = reinterpret_cast<const uint4*>(blk)[i];
    bit = br.bit(cs.data);
    if (slot == cs.bpm - 1 && bit > data_bits) return 2 * block + 1;
    ++block;
    slot = slot + 1 == cs.bpm ? 0 : slot + 1;
  }
  return NO_EVENT;
}

struct ChunkSums {
  long long n;
  unsigned a, b, c;
};

__device__ __forceinline__ ChunkSums operator+(const ChunkSums& x, const ChunkSums& y) {
  return ChunkSums{x.n + y.n, x.a + y.a, x.b + y.b, x.c + y.c};
}

// Exclusive scan over the CTA's threads in thread order; *total gets the sum.  `ws` holds one value per warp.
__device__ __forceinline__ ChunkSums block_exclusive_scan(ChunkSums v, ChunkSums* ws, ChunkSums* total) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarp = blockDim.x >> 5;
  ChunkSums inc = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    ChunkSums y{__shfl_up_sync(0xffffffffu, inc.n, o), __shfl_up_sync(0xffffffffu, inc.a, o),
                __shfl_up_sync(0xffffffffu, inc.b, o), __shfl_up_sync(0xffffffffu, inc.c, o)};
    if (lane >= o) inc = inc + y;
  }
  if (lane == 31) ws[warp] = inc;
  __syncthreads();
  ChunkSums before{0, 0u, 0u, 0u}, all{0, 0u, 0u, 0u};
  for (int w = 0; w < nwarp; ++w) {
    if (w < warp) before = before + ws[w];
    all = all + ws[w];
  }
  __syncthreads();
  *total = all;
  ChunkSums ex{inc.n - v.n, inc.a - v.a, inc.b - v.b, inc.c - v.c};
  return before + ex;
}

// One CTA per long segment.  Dynamic shared memory: the chunk states, `cap` chunks (>= every segment's chunk count).
__global__ void __launch_bounds__(CHUNK_THREADS, 2)
chunked_kernel(const uint8_t* __restrict__ bytes, const ImgDesc* __restrict__ imgs, const HuffTbl* __restrict__ tbls,
               const Seg* __restrict__ segs, int cap, int forced, uint8_t* destuffed, int16_t* __restrict__ coef,
               int* __restrict__ status) {
  __shared__ __align__(16) HuffTbl tb[6];
  __shared__ __align__(16) int16_t blk_smem[CHUNK_THREADS][64];
  __shared__ ChunkSeg cs;
  __shared__ ChunkSums scan_ws[CHUNK_THREADS / 32];
  __shared__ unsigned long long first_event;
  extern __shared__ __align__(16) unsigned char chunk_smem[];
  long long* st = reinterpret_cast<long long*>(chunk_smem);        // start state of each chunk
  long long* ex = st + cap;                                        // its exit state
  int* cnt = reinterpret_cast<int*>(ex + cap);                      // blocks it starts
  unsigned* d0 = reinterpret_cast<unsigned*>(cnt + cap);            // its DC differences per component
  unsigned* d1 = d0 + cap;
  unsigned* d2 = d1 + cap;

  const int tid = threadIdx.x, T = blockDim.x;
  const Seg sg = segs[blockIdx.x];
  const ImgDesc& im = imgs[sg.img];
  constexpr int TBL_WORDS = sizeof(HuffTbl) / 4;
  for (int w = tid; w < 2 * im.ncomp * TBL_WORDS; w += T) {
    const int t = w / TBL_WORDS, j = w - t * TBL_WORDS;
    const HuffTbl& src = tbls[(t & 1) ? im.c[t >> 1].ac : im.c[t >> 1].dc];
    reinterpret_cast<uint32_t*>(&tb[t])[j] = reinterpret_cast<const uint32_t*>(&src)[j];
  }

  // 1. de-stuff: each thread a contiguous byte range, placed by a scan of the data-byte counts
  const long long n = sg.end - sg.start;
  const uint8_t* src = bytes + sg.start;
  uint8_t* dst = destuffed + sg.start;
  const long long per = (n + T - 1) / T;
  const long long i0 = std::min(n, tid * per), i1 = std::min(n, i0 + per);
  ChunkSums tot;
  const ChunkSums at = block_exclusive_scan(ChunkSums{destuff_count(src, i0, i1), 0u, 0u, 0u}, scan_ws, &tot);
  destuff_copy(src, i0, i1, dst + at.n);
  if (tid == 0) {
    chunk_seg_init(cs, im, sg, dst, tot.n, tb);
    first_event = (unsigned long long)NO_EVENT;
  }
  __syncthreads();                   // de-stuffed bytes (global) and cs visible to the CTA

  // 2. synchronisation rounds; thread tid owns chunks [c0, c1)
  long long cb;
  int nch;
  chunk_geometry(cs.len, forced, &cb, &nch);
  const int per_thread = (nch + T - 1) / T;
  const int c0 = std::min(nch, tid * per_thread), c1 = std::min(nch, c0 + per_thread);
  unsigned dirty = 0;
  for (int t = c0; t < c1; ++t) {
    st[t] = (t * cb * 8) << 3;
    ChunkRun r{0, 0, 0u, 0u, 0u};
    if (t < nch - 1) r = chunk_sync(cs, st[t], (t + 1) * cb * 8);
    ex[t] = r.exit; cnt[t] = r.count; d0[t] = r.dc0; d1[t] = r.dc1; d2[t] = r.dc2;
  }
  for (;;) {
    __syncthreads();
    for (int t = std::max(c0, 1); t < c1; ++t)
      if (ex[t - 1] != st[t]) {
        st[t] = ex[t - 1];
        dirty |= 1u << (t - c0);
      }
    if (!__syncthreads_or(dirty != 0)) break;
    for (int t = c0; t < c1; ++t)
      if (dirty & (1u << (t - c0))) {
        if (t < nch - 1) {
          const ChunkRun r = chunk_sync(cs, st[t], (t + 1) * cb * 8);
          ex[t] = r.exit; cnt[t] = r.count; d0[t] = r.dc0; d1[t] = r.dc1; d2[t] = r.dc2;
        }
      }
    dirty = 0;
  }

  // 3. absolute first block and DC predictors of every chunk, then the final pass
  ChunkSums mine{0, 0u, 0u, 0u};
  for (int t = c0; t < c1; ++t) mine = mine + ChunkSums{cnt[t], d0[t], d1[t], d2[t]};
  ChunkSums pre = block_exclusive_scan(mine, scan_ws, &tot);
  long long event = NO_EVENT;
  for (int t = c0; t < c1; ++t) {
    const long long end_bit = t == nch - 1 ? LLONG_MAX : (t + 1) * cb * 8;
    event = std::min(event, chunk_final(cs, st[t], end_bit, pre.n, pre.a, pre.b, pre.c, blk_smem[tid], coef));
    pre = pre + ChunkSums{cnt[t], d0[t], d1[t], d2[t]};
  }
  if (event != NO_EVENT) atomicMin(&first_event, (unsigned long long)event);
  __syncthreads();
  if (tid == 0 && first_event != (unsigned long long)NO_EVENT)
    atomicCAS(status + im.orig, 0, (first_event & 1) ? ST_OVERRUN : ST_BAD_CODE);
}

// The chunked decode of one segment on the host, in the kernel's order of rounds and passes.  Returns the segment's
// error (0 when none) and sets *rounds to the synchronisation rounds it took.
int chunked_segment_host(const uint8_t* bytes, const ImgDesc& im, const HuffTbl* tbls, const Seg& sg, int forced,
                         int16_t* coef, int* rounds) {
  const long long n = sg.end - sg.start;
  std::vector<uint8_t> buf((size_t)n);
  destuff_copy(bytes + sg.start, 0, n, buf.data());
  HuffTbl tb[6];
  for (int c = 0; c < im.ncomp; ++c) {
    tb[2 * c] = tbls[im.c[c].dc];
    tb[2 * c + 1] = tbls[im.c[c].ac];
  }
  ChunkSeg cs;
  chunk_seg_init(cs, im, sg, buf.data(), destuff_count(bytes + sg.start, 0, n), tb);
  long long cb;
  int nch;
  chunk_geometry(cs.len, forced, &cb, &nch);
  std::vector<long long> st(nch);
  std::vector<ChunkRun> run(nch, ChunkRun{0, 0, 0u, 0u, 0u});
  for (int t = 0; t < nch; ++t) {
    st[t] = (t * cb * 8) << 3;
    if (t < nch - 1) run[t] = chunk_sync(cs, st[t], (t + 1) * cb * 8);
  }
  *rounds = 1;
  for (;;) {
    std::vector<int> dirty;
    for (int t = 1; t < nch; ++t)
      if (run[t - 1].exit != st[t]) {
        st[t] = run[t - 1].exit;
        dirty.push_back(t);
      }
    if (dirty.empty()) break;
    ++*rounds;
    for (int t : dirty)
      if (t < nch - 1) run[t] = chunk_sync(cs, st[t], (t + 1) * cb * 8);
  }
  long long block = 0, event = NO_EVENT;
  unsigned p0 = 0, p1 = 0, p2 = 0;
  alignas(16) int16_t blk[64];
  for (int t = 0; t < nch; ++t) {
    const long long end_bit = t == nch - 1 ? LLONG_MAX : (t + 1) * cb * 8;
    event = std::min(event, chunk_final(cs, st[t], end_bit, block, p0, p1, p2, blk, coef));
    block += run[t].count;
    p0 += run[t].dc0; p1 += run[t].dc1; p2 += run[t].dc2;
  }
  return event == NO_EVENT ? 0 : (event & 1) ? ST_OVERRUN : ST_BAD_CODE;
}

// ------------------------------------------------------------------------------------------------------------------
// Device: entropy decode of multi-scan files
// ------------------------------------------------------------------------------------------------------------------

enum ScanKind { SCAN_SEQUENTIAL, SCAN_DC_FIRST, SCAN_DC_REFINE, SCAN_AC_FIRST, SCAN_AC_REFINE };

struct ScanDesc {                    // one scan of one multi-scan image
  int img, kind, ncomp;
  int comp[3], dc[3], ac[3];         // frame component indices in scan order; indices into the batch's Huffman tables
  int ss, se, al;
  int cols;                          // MCUs per row: the frame's when interleaved, else the component's blocks
};

struct MSeg {                        // one entropy-coded segment of a scan
  long long start, end;
  int scan, mcu0, nmcu;
};

__host__ __device__ __forceinline__ void refine_bit(BitReader& br, int16_t* c, int p1) {
  if (br.nbits < 16) br.fill();
  const int v = *c;
  if (br.get(1) && !(v & p1)) *c = (int16_t)(v >= 0 ? v + p1 : v - p1);
}

// Decodes the blocks of one segment of a multi-scan file into the image's zero-initialised coefficients, with
// libjpeg-turbo's jdhuff.c (sequential) and jdphuff.c (progressive) arithmetic.  Every coefficient is read and written
// on its own: scans of the same dependency level update different coefficients of the same blocks concurrently.
// Returns 0 or the segment's PG_JPEG_* error.
__host__ __device__ inline int decode_scan_segment(const uint8_t* __restrict__ bytes, const ImgDesc& im,
                                                   const HuffTbl* __restrict__ tbls, const ScanDesc& sc, const MSeg& sg,
                                                   int16_t* __restrict__ coef) {
#ifdef __CUDA_ARCH__
  const uint8_t* natural = c_natural;
#else
  const uint8_t* natural = h_natural;
#endif
  BitReader br{bytes + sg.start, bytes + sg.end, 0, 0, 0, 0};
  int pred0 = 0, pred1 = 0, pred2 = 0;
  int eobrun = 0;
  const int p1 = 1 << sc.al;
  for (int mi = 0; mi < sg.nmcu && !br.err; ++mi) {
    const int mcu = sg.mcu0 + mi;
    const int my = mcu / sc.cols, mx = mcu - my * sc.cols;
    for (int j = 0; j < sc.ncomp && !br.err; ++j) {
      const Comp& cp = im.c[sc.comp[j]];
      const int nv = sc.ncomp > 1 ? cp.v : 1, nh = sc.ncomp > 1 ? cp.h : 1;
      for (int bv = 0; bv < nv && !br.err; ++bv)
        for (int bh = 0; bh < nh && !br.err; ++bh) {
          const long long b = cp.coef_off + (long long)(my * nv + bv) * cp.bw + (mx * nh + bh);
          int16_t* blk = coef + b * 64;
          if (sc.kind == SCAN_DC_REFINE) {
            if (br.nbits < 16) br.fill();
            if (br.get(1)) blk[0] = (int16_t)(blk[0] | p1);
            continue;
          }
          if (sc.kind == SCAN_SEQUENTIAL || sc.kind == SCAN_DC_FIRST) {
            if (br.nbits < 32) br.fill();
            int s = huff_decode(br, tbls[sc.dc[j]]);
            if (br.err) break;
            if (s) s = huff_extend(br.get(s), s);
            // predictor of scan component j, kept in registers (an indexed array would live in local memory)
            const int pv = (j == 0 ? pred0 : j == 1 ? pred1 : pred2) + s;
            if (j == 0) pred0 = pv; else if (j == 1) pred1 = pv; else pred2 = pv;
            blk[0] = (int16_t)((unsigned)pv << sc.al);
            if (sc.kind == SCAN_DC_FIRST) continue;
          }
          const HuffTbl& act = tbls[sc.ac[j]];
          if (sc.kind != SCAN_AC_REFINE) {           // sequential AC, or the first scan of a band
            if (eobrun > 0) { --eobrun; continue; }
            for (int k = sc.kind == SCAN_SEQUENTIAL ? 1 : sc.ss; k <= sc.se; ++k) {
              if (br.nbits < 32) br.fill();
              const int rs = huff_decode(br, act);
              if (br.err) break;
              const int r = rs >> 4, s = rs & 15;
              if (s) {
                k += r;
                if (k > sc.se) { br.err = ST_BAD_CODE; break; }
                blk[natural[k]] = (int16_t)((unsigned)huff_extend(br.get(s), s) << sc.al);
              } else if (r == 15) {
                k += 15;
              } else {
                if (sc.kind == SCAN_SEQUENTIAL) break;
                eobrun = (1 << r) - 1;
                if (r) eobrun += br.get(r);
                break;
              }
            }
            continue;
          }
          int k = sc.ss;                              // decode_mcu_AC_refine
          if (eobrun == 0) {
            for (; k <= sc.se; ++k) {
              if (br.nbits < 32) br.fill();
              const int rs = huff_decode(br, act);
              if (br.err) break;
              int r = rs >> 4, s = rs & 15;
              if (s) {
                s = br.get(1) ? p1 : -p1;              // a newly nonzero coefficient is +-1 at this bit
              } else if (r != 15) {
                eobrun = 1 << r;
                if (r) eobrun += br.get(r);
                break;
              }
              // skip r zero coefficients, appending a correction bit to every nonzero one on the way
              for (; k <= sc.se; ++k) {
                int16_t* c = blk + natural[k];
                if (*c) refine_bit(br, c, p1);
                else if (--r < 0) break;
              }
              if (s) {
                if (k > sc.se) { br.err = ST_BAD_CODE; break; }
                blk[natural[k]] = (int16_t)s;
              }
            }
          }
          if (eobrun > 0 && !br.err) {                // the rest of the band: correction bits only
            for (; k <= sc.se; ++k) {
              int16_t* c = blk + natural[k];
              if (*c) refine_bit(br, c, p1);
            }
            --eobrun;
          }
        }
    }
    if (!br.err && br.overrun()) br.err = ST_OVERRUN;
  }
  return br.err;
}

// One thread per segment of the launch's dependency level, packed into warps as in entropy_kernel.  A segment of an
// image that an earlier level (or another segment) has already failed is skipped.
__global__ void __launch_bounds__(ENTROPY_THREADS, 1)
multiscan_kernel(const uint8_t* __restrict__ bytes, const ImgDesc* __restrict__ imgs, const HuffTbl* __restrict__ tbls,
                 const ScanDesc* __restrict__ scans, const MSeg* __restrict__ segs, int nseg, int lanes,
                 int16_t* __restrict__ coef, int* __restrict__ status) {
  const int lane = threadIdx.x;
  if (lane >= lanes) return;
  const int si = blockIdx.x * lanes + lane;
  if (si >= nseg) return;
  const MSeg sg = segs[si];
  const ScanDesc& sc = scans[sg.scan];
  const ImgDesc& im = imgs[sc.img];
  if (*(volatile const int*)(status + im.orig)) return;
  const int err = decode_scan_segment(bytes, im, tbls, sc, sg, coef);
  if (err) atomicCAS(status + im.orig, 0, err);
}

// ------------------------------------------------------------------------------------------------------------------
// Device: dequantise + jpeg_idct_islow
// ------------------------------------------------------------------------------------------------------------------

constexpr int CONST_BITS = 13, PASS1_BITS = 2;
constexpr long long FIX_0_298631336 = 2446, FIX_0_390180644 = 3196, FIX_0_541196100 = 4433, FIX_0_765366865 = 6270,
                    FIX_0_899976223 = 7373, FIX_1_175875602 = 9633, FIX_1_501321110 = 12299, FIX_1_847759065 = 15137,
                    FIX_1_961570560 = 16069, FIX_2_053119869 = 16819, FIX_2_562915447 = 20995, FIX_3_072711026 = 25172;

__host__ __device__ __forceinline__ long long descale(long long x, int n) { return (x + (1LL << (n - 1))) >> n; }

// jdmaster.c prepare_range_limit_table, post-IDCT part, indexed by (x & RANGE_MASK)
__host__ __device__ __forceinline__ uint8_t idct_range_limit(long long v) {
  const int x = (int)(v & 1023);
  return (uint8_t)(x < 128 ? x + 128 : x < 512 ? 255 : x < 896 ? 0 : x - 896);
}

// One 1-D pass of jidctint.c on 8 values in0..in7 (in0 already scaled by the caller); returns the 8 outputs before
// descaling.
__host__ __device__ __forceinline__ void idct_1d(long long z0, long long z1in, long long z2in, long long z3in, long long z4in,
                                        long long z5in, long long z6in, long long z7in, long long out[8]) {
  // even part
  long long z2 = z2in, z3 = z6in;
  long long z1 = (z2 + z3) * FIX_0_541196100;
  long long tmp2 = z1 + z3 * (-FIX_1_847759065);
  long long tmp3 = z1 + z2 * FIX_0_765366865;
  long long tmp0 = (z0 + z4in) * (1LL << CONST_BITS);
  long long tmp1 = (z0 - z4in) * (1LL << CONST_BITS);
  const long long tmp10 = tmp0 + tmp3, tmp13 = tmp0 - tmp3, tmp11 = tmp1 + tmp2, tmp12 = tmp1 - tmp2;
  // odd part
  tmp0 = z7in; tmp1 = z5in; tmp2 = z3in; tmp3 = z1in;
  z1 = tmp0 + tmp3; z2 = tmp1 + tmp2; z3 = tmp0 + tmp2;
  long long z4 = tmp1 + tmp3;
  const long long z5 = (z3 + z4) * FIX_1_175875602;
  tmp0 = tmp0 * FIX_0_298631336;
  tmp1 = tmp1 * FIX_2_053119869;
  tmp2 = tmp2 * FIX_3_072711026;
  tmp3 = tmp3 * FIX_1_501321110;
  z1 = z1 * (-FIX_0_899976223);
  z2 = z2 * (-FIX_2_562915447);
  z3 = z3 * (-FIX_1_961570560);
  z4 = z4 * (-FIX_0_390180644);
  z3 += z5; z4 += z5;
  tmp0 += z1 + z3; tmp1 += z2 + z4; tmp2 += z2 + z3; tmp3 += z1 + z4;
  out[0] = tmp10 + tmp3; out[7] = tmp10 - tmp3;
  out[1] = tmp11 + tmp2; out[6] = tmp11 - tmp2;
  out[2] = tmp12 + tmp1; out[5] = tmp12 - tmp1;
  out[3] = tmp13 + tmp0; out[4] = tmp13 - tmp0;
}

__device__ __forceinline__ int find_plane(const PlaneWork* __restrict__ pw, int np, long long b) {
  int lo = 0, hi = np - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (pw[mid].block0 <= b) lo = mid; else hi = mid - 1;
  }
  return lo;
}

// Dequantise + IDCT of block `local` of component plane `cp` into its 8x8 pixels.
__host__ __device__ inline void idct_block(const Comp& cp, long long local, const int16_t* __restrict__ coef,
                                           uint8_t* __restrict__ planes) {
  const int by = (int)(local / cp.bw), bx = (int)(local - (long long)by * cp.bw);
  int16_t in[64];
  const uint4* src = reinterpret_cast<const uint4*>(coef + (cp.coef_off + local) * 64);
#pragma unroll
  for (int i = 0; i < 8; ++i) *reinterpret_cast<uint4*>(in + 8 * i) = src[i];
  int ws[64];
#pragma unroll
  for (int col = 0; col < 8; ++col) {              // pass 1: columns; DEQUANTIZE is a short x short product
    long long o[8];
    idct_1d((int)in[col] * (int)cp.q[col], (int)in[8 + col] * (int)cp.q[8 + col], (int)in[16 + col] * (int)cp.q[16 + col],
            (int)in[24 + col] * (int)cp.q[24 + col], (int)in[32 + col] * (int)cp.q[32 + col],
            (int)in[40 + col] * (int)cp.q[40 + col], (int)in[48 + col] * (int)cp.q[48 + col],
            (int)in[56 + col] * (int)cp.q[56 + col], o);
#pragma unroll
    for (int r = 0; r < 8; ++r) ws[8 * r + col] = (int)descale(o[r], CONST_BITS - PASS1_BITS);
  }
  uint8_t* dst = planes + cp.plane_off + (long long)(by * 8) * (cp.bw * 8) + bx * 8;
#pragma unroll
  for (int row = 0; row < 8; ++row) {              // pass 2: rows
    long long o[8];
    const int* wr = ws + 8 * row;
    idct_1d(wr[0], wr[1], wr[2], wr[3], wr[4], wr[5], wr[6], wr[7], o);
    uint32_t lo = 0, hi = 0;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      lo |= (uint32_t)idct_range_limit(descale(o[i], CONST_BITS + PASS1_BITS + 3)) << (8 * i);
      hi |= (uint32_t)idct_range_limit(descale(o[4 + i], CONST_BITS + PASS1_BITS + 3)) << (8 * i);
    }
    *reinterpret_cast<uint2*>(dst + (long long)row * cp.bw * 8) = make_uint2(lo, hi);
  }
}

// One thread per 8x8 block.
__global__ void __launch_bounds__(128)
idct_kernel(const ImgDesc* __restrict__ imgs, const PlaneWork* __restrict__ pw, int np, long long nblocks,
            const int16_t* __restrict__ coef, uint8_t* __restrict__ planes, const int* __restrict__ status) {
  const long long b = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= nblocks) return;
  const PlaneWork w = pw[find_plane(pw, np, b)];
  const ImgDesc& im = imgs[w.img];
  if (status[im.orig]) return;
  idct_block(im.c[w.comp], b - w.block0, coef, planes);
}

// ------------------------------------------------------------------------------------------------------------------
// Device: upsample + colour convert
// ------------------------------------------------------------------------------------------------------------------

// jdsample.c, one output sample of a chroma component at output column x of output row y
__host__ __device__ __forceinline__ int chroma_sample(const uint8_t* __restrict__ pl, int stride, int dw, int dh, int hmax,
                                             int vmax, int x, int y) {
  if (hmax == 1) return pl[(long long)y * stride + x];
  const int j = x >> 1;
  if (vmax == 1) {                                  // h2v1
    const uint8_t* r = pl + (long long)y * stride;
    if (dw <= 2) return r[j];
    if (!(x & 1)) return j == 0 ? r[0] : (r[j] * 3 + r[j - 1] + 1) >> 2;
    return j == dw - 1 ? r[j] : (r[j] * 3 + r[j + 1] + 2) >> 2;
  }
  const int yy = y >> 1;                            // h2v2
  if (dw <= 2) return pl[(long long)yy * stride + j];
  const int y2 = (y & 1) ? (yy + 1 < dh ? yy + 1 : dh - 1) : (yy > 0 ? yy - 1 : 0);   // context rows replicate the component's edge rows
  const uint8_t* r0 = pl + (long long)yy * stride;
  const uint8_t* r1 = pl + (long long)y2 * stride;
  const int cs = r0[j] * 3 + r1[j];
  if (!(x & 1)) return j == 0 ? (cs * 4 + 8) >> 4 : (cs * 3 + (r0[j - 1] * 3 + r1[j - 1]) + 8) >> 4;
  return j == dw - 1 ? (cs * 4 + 7) >> 4 : (cs * 3 + (r0[j + 1] * 3 + r1[j + 1]) + 7) >> 4;
}

__host__ __device__ __forceinline__ uint8_t clamp255(int v) { return (uint8_t)(v < 0 ? 0 : v > 255 ? 255 : v); }

// Output pixel (x, y) of image `im`: luma, upsampled chroma, jdcolor.c ycc_rgb_convert; grayscale is replicated.
__host__ __device__ inline void color_pixel(const ImgDesc& im, int x, int y, const uint8_t* __restrict__ planes) {
  uint8_t* o = im.dst + (long long)y * im.dst_stride + 3 * x;
  const int Y = planes[im.c[0].plane_off + (long long)y * (im.c[0].bw * 8) + x];
  if (im.ncomp == 1) { o[0] = o[1] = o[2] = (uint8_t)Y; return; }
  const Comp& cb = im.c[1];
  const Comp& cr = im.c[2];
  const int Cb = chroma_sample(planes + cb.plane_off, cb.bw * 8, cb.dw, cb.dh, im.hmax, im.vmax, x, y);
  const int Cr = chroma_sample(planes + cr.plane_off, cr.bw * 8, cr.dw, cr.dh, im.hmax, im.vmax, x, y);
  // jdcolor.c build_ycc_rgb_table with SCALEBITS 16, evaluated per sample with the same integer formulas
  constexpr int SCALEBITS = 16;
  constexpr long long ONE_HALF = 1LL << (SCALEBITS - 1);
  constexpr long long F_1_40200 = (long long)(1.40200 * (1L << SCALEBITS) + 0.5),
                      F_1_77200 = (long long)(1.77200 * (1L << SCALEBITS) + 0.5),
                      F_0_71414 = (long long)(0.71414 * (1L << SCALEBITS) + 0.5),
                      F_0_34414 = (long long)(0.34414 * (1L << SCALEBITS) + 0.5);
  const long long xb = Cb - 128, xr = Cr - 128;
  const int cr_r = (int)((F_1_40200 * xr + ONE_HALF) >> SCALEBITS);
  const int cb_b = (int)((F_1_77200 * xb + ONE_HALF) >> SCALEBITS);
  const long long cr_g = -F_0_71414 * xr;
  const long long cb_g = -F_0_34414 * xb + ONE_HALF;
  o[0] = clamp255(Y + cr_r);
  o[1] = clamp255(Y + (int)((cb_g + cr_g) >> SCALEBITS));
  o[2] = clamp255(Y + cb_b);
}

// One thread per output pixel; pix0[i] = first pixel of image i in the flattened batch.
__global__ void __launch_bounds__(256)
color_kernel(const ImgDesc* __restrict__ imgs, const long long* __restrict__ pix0, int n, long long npix,
             const uint8_t* __restrict__ planes, const int* __restrict__ status) {
  const long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= npix) return;
  int lo = 0, hi = n - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (pix0[mid] <= g) lo = mid; else hi = mid - 1;
  }
  const ImgDesc& im = imgs[lo];
  if (status[im.orig]) return;
  const long long local = g - pix0[lo];
  const int y = (int)(local / im.width);
  color_pixel(im, (int)(local - (long long)y * im.width), y, planes);
}

// ------------------------------------------------------------------------------------------------------------------
// Host: batch plan
// ------------------------------------------------------------------------------------------------------------------

struct Plan {
  std::vector<ImgDesc> imgs;
  std::vector<HuffTbl> tbls;
  std::vector<Seg> segs;
  std::vector<PlaneWork> planes;
  std::vector<long long> pix0;
  std::vector<ScanDesc> scans;                        // multi-scan images
  std::vector<MSeg> msegs;                            // their segments, ordered by dependency level
  std::vector<int> level0;                            // msegs of level L: [level0[L - 1], level0[L])
  long long nblocks = 0, plane_bytes = 0, npix = 0;
  long long multi_coef0 = -1, multi_coef1 = -1;       // blocks [multi_coef0, multi_coef1) hold every multi-scan image
  size_t off_imgs = 0, off_tbls = 0, off_segs = 0, off_planes = 0, off_pix0 = 0, off_scans = 0, off_msegs = 0,
         meta_bytes = 0;
  size_t off_bytes = 0, off_meta = 0, off_coef = 0, off_plane = 0, off_destuff = 0, total = 0;
};

// Index of the Huffman table (bits, vals) in the batch's de-duplicated table array; -1 for an invalid table.
int huff_index(std::map<std::string, int>& index, std::vector<HuffTbl>& tbls, const uint8_t* bits, const uint8_t* vals,
               int cls) {
  std::string key(1, (char)cls);
  key.append((const char*)bits, 16);
  key.append((const char*)vals, 256);
  auto it = index.find(key);
  if (it != index.end()) return it->second;
  const int idx = (int)tbls.size();
  tbls.emplace_back();
  if (!make_huff(bits, vals, cls == 0, &tbls.back())) return -1;
  index.emplace(key, idx);
  return idx;
}

// The scans of multi-scan image k (file bytes [base, base + len) of the packed input), found again by the multi-scan
// walk that validated them: their descriptors, segments (by level), latched quantisation tables and Huffman tables.
int plan_multiscan(const uint8_t* packed, int64_t base, int64_t len, const pg_jpeg_info& in, int i, int k, ImgDesc& d,
                   std::map<std::string, int>& tbl_index, std::vector<std::vector<MSeg>>& by_level, Plan* P) {
  MultiScan ms;
  ms.want_segs = true;
  pg_jpeg_info w;
  char msg[200];
  Why why{msg, sizeof(msg)};
  if (parse_multiscan(packed + base, len, &w, &ms, &why) != PG_JPEG_OK || !(w.table_mask & PG_JPEG_MULTISCAN) ||
      w.width != in.width || w.height != in.height || w.components != in.components ||
      w.num_segments != in.num_segments || memcmp(w.h_samp, in.h_samp, sizeof(w.h_samp)) ||
      memcmp(w.v_samp, in.v_samp, sizeof(w.v_samp))) {
    set_last_error("jpeg: image %d does not match its pg_jpeg_info", i);
    return 1;
  }
  for (int c = 0; c < d.ncomp; ++c)
    for (int q = 0; q < 64; ++q) d.c[c].q[h_natural[q]] = (int16_t)ms.qt[c][q];
  const bool progressive = w.sof == 0xC2;
  for (const ScanRec& r : ms.scans) {
    const pg_jpeg_scan& p = r.pub;
    ScanDesc sd;
    memset(&sd, 0, sizeof(sd));
    sd.img = k;
    sd.kind = !progressive ? SCAN_SEQUENTIAL
              : p.ss == 0  ? (p.ah ? SCAN_DC_REFINE : SCAN_DC_FIRST)
                           : (p.ah ? SCAN_AC_REFINE : SCAN_AC_FIRST);
    sd.ncomp = p.components;
    sd.ss = p.ss; sd.se = p.se; sd.al = p.al;
    int rows = 0;
    scan_grid(&w, p.components, p.component[0], &sd.cols, &rows);
    for (int j = 0; j < p.components; ++j) {
      sd.comp[j] = p.component[j];
      const bool need_dc = sd.kind == SCAN_SEQUENTIAL || sd.kind == SCAN_DC_FIRST;
      const bool need_ac = sd.kind == SCAN_SEQUENTIAL || sd.kind == SCAN_AC_FIRST || sd.kind == SCAN_AC_REFINE;
      sd.dc[j] = need_dc ? huff_index(tbl_index, P->tbls, r.dc_bits[j], r.dc_vals[j], 0) : 0;
      sd.ac[j] = need_ac ? huff_index(tbl_index, P->tbls, r.ac_bits[j], r.ac_vals[j], 1) : 0;
      if (sd.dc[j] < 0 || sd.ac[j] < 0) {
        set_last_error("jpeg: image %d has an invalid Huffman table", i);
        return 1;
      }
    }
    const int total = sd.cols * rows;
    const int ri = p.restart_interval ? p.restart_interval : total;
    if ((int)by_level.size() < p.level) by_level.resize(p.level);
    for (int s = 0; s < p.num_segments; ++s) {
      MSeg sg;
      sg.start = base + r.segs[s].first;
      sg.end = base + r.segs[s].second;
      sg.scan = (int)P->scans.size();
      sg.mcu0 = s * ri;
      sg.nmcu = std::min(ri, total - sg.mcu0);
      by_level[p.level - 1].push_back(sg);
    }
    P->scans.push_back(sd);
  }
  return 0;
}

// Sizes every region from the parse results; with `packed` it also fills the tables the kernels read.
int make_plan(const uint8_t* packed, const int64_t* offsets, const pg_jpeg_info* infos, int n, int64_t packed_bytes,
              const pg_image* dst, Plan* P) {
  if (n <= 0 || !infos || packed_bytes < 0) { set_last_error("jpeg: bad argument"); return 1; }
  std::map<std::string, int> tbl_index;
  long long segs = 0, msegs = 0, mtables = 0;
  for (int i = 0; i < n; ++i) {
    const pg_jpeg_info& in = infos[i];
    if (in.status != PG_JPEG_OK) continue;
    if (in.width <= 0 || in.height <= 0 || (in.components != 1 && in.components != 3) || in.num_segments < 1) {
      set_last_error("jpeg: image %d has an inconsistent pg_jpeg_info", i);
      return 1;
    }
    const bool multi = (in.table_mask & PG_JPEG_MULTISCAN) != 0;
    ImgDesc d;
    memset(&d, 0, sizeof(d));
    d.orig = i;
    d.width = in.width; d.height = in.height; d.ncomp = in.components;
    d.hmax = in.components == 3 ? in.h_samp[0] : 1;
    d.vmax = in.components == 3 ? in.v_samp[0] : 1;
    d.mcux = (in.width + 8 * d.hmax - 1) / (8 * d.hmax);
    d.mcuy = (in.height + 8 * d.vmax - 1) / (8 * d.vmax);
    d.restart_interval = in.restart_interval;
    for (int c = 0; c < d.ncomp; ++c) {
      Comp& cp = d.c[c];
      cp.h = d.ncomp == 3 ? in.h_samp[c] : 1;
      cp.v = d.ncomp == 3 ? in.v_samp[c] : 1;
      cp.bw = d.mcux * cp.h; cp.bh = d.mcuy * cp.v;
      cp.dw = (int)(((long long)in.width * cp.h + d.hmax - 1) / d.hmax);
      cp.dh = (int)(((long long)in.height * cp.v + d.vmax - 1) / d.vmax);
      cp.coef_off = P->nblocks;
      cp.plane_off = P->plane_bytes;
      if (multi && c == 0 && P->multi_coef0 < 0) P->multi_coef0 = P->nblocks;
      P->planes.push_back({P->nblocks, (int)P->imgs.size(), c});
      P->nblocks += (long long)cp.bw * cp.bh;
      P->plane_bytes += (long long)align_up((size_t)cp.bw * cp.bh * 64, 16);
      if (multi) {                                    // tables per scan: plan_multiscan
        P->multi_coef1 = P->nblocks;
        continue;
      }
      for (int k = 0; k < 64; ++k) cp.q[h_natural[k]] = (int16_t)in.qt[in.quant_table[c]][k];
      for (int cls = 0; cls < 2; ++cls) {
        const int th = cls ? in.ac_table[c] : in.dc_table[c];
        const int idx = huff_index(tbl_index, P->tbls, cls ? in.ac_bits[th] : in.dc_bits[th],
                                   cls ? in.ac_vals[th] : in.dc_vals[th], cls);
        if (idx < 0) {
          set_last_error("jpeg: image %d has an invalid Huffman table", i);
          return 1;
        }
        (cls ? cp.ac : cp.dc) = idx;
      }
    }
    if (dst) {
      if (!dst[i].data || dst[i].height != in.height || dst[i].width != in.width || dst[i].row_stride < 3LL * in.width) {
        set_last_error("jpeg: destination %d does not match the %dx%d image", i, in.width, in.height);
        return 1;
      }
      d.dst = const_cast<uint8_t*>(dst[i].data);
      d.dst_stride = dst[i].row_stride;
    }
    P->pix0.push_back(P->npix);
    P->npix += (long long)in.width * in.height;
    if (multi) {
      msegs += in.num_segments;
      mtables += (unsigned)in.table_mask >> 16;
    } else {
      segs += in.num_segments;
    }
    P->imgs.push_back(d);
  }
  // Without the files, the multi-scan regions are sized by bounds from the infos: a scan has at least one segment,
  // and the batch has no more Huffman tables than selections.
  std::vector<std::vector<MSeg>> by_level;
  if (packed) {
    int k = 0;
    for (int i = 0; i < n; ++i) {
      const pg_jpeg_info& in = infos[i];
      if (in.status != PG_JPEG_OK) continue;
      if (in.table_mask & PG_JPEG_MULTISCAN) {
        const int64_t base = offsets[i], len = offsets[i + 1] - offsets[i];
        if (base < 0 || len < 0 || offsets[i + 1] > packed_bytes) {
          set_last_error("jpeg: image %d lies outside the packed input", i);
          return 1;
        }
        if (plan_multiscan(packed, base, len, in, i, k, P->imgs[k], tbl_index, by_level, P)) return 1;
      }
      ++k;
    }
    P->level0.push_back(0);
    for (auto& v : by_level) {
      P->msegs.insert(P->msegs.end(), v.begin(), v.end());
      P->level0.push_back((int)P->msegs.size());
    }
    if ((long long)P->msegs.size() != msegs) {
      set_last_error("jpeg: the multi-scan images do not match their pg_jpeg_info");
      return 1;
    }
  }
  const size_t nimg = P->imgs.size();
  const size_t ntbls = packed ? P->tbls.size() : P->tbls.size() + (size_t)mtables;
  const size_t nscans = packed ? P->scans.size() : (size_t)msegs;
  size_t off = 0;
  P->off_imgs = off; off += align_up(nimg * sizeof(ImgDesc), 256);
  P->off_tbls = off; off += align_up(ntbls * sizeof(HuffTbl), 256);
  P->off_segs = off; off += align_up((size_t)segs * sizeof(Seg), 256);
  P->off_planes = off; off += align_up(P->planes.size() * sizeof(PlaneWork), 256);
  P->off_pix0 = off; off += align_up(nimg * sizeof(long long), 256);
  P->off_scans = off; off += align_up(nscans * sizeof(ScanDesc), 256);
  P->off_msegs = off; off += align_up((size_t)msegs * sizeof(MSeg), 256);
  P->meta_bytes = off;
  size_t total = 0;
  P->off_bytes = total; total += align_up((size_t)packed_bytes, 256);
  P->off_meta = total; total += P->meta_bytes;
  P->off_coef = total; total += align_up((size_t)P->nblocks * 128, 256);
  P->off_plane = total; total += align_up((size_t)P->plane_bytes, 256);
  P->off_destuff = total; total += align_up((size_t)packed_bytes, 256);   // de-stuffed long segments, in place
  P->total = total;
  if (!packed) return 0;
  // restart segments, found again by the same walk that validated them in pg_jpeg_parse
  int k = 0;
  for (int i = 0; i < n; ++i) {
    const pg_jpeg_info& in = infos[i];
    if (in.status != PG_JPEG_OK) continue;
    if (in.table_mask & PG_JPEG_MULTISCAN) { ++k; continue; }
    const ImgDesc& d = P->imgs[k];
    const int64_t base = offsets[i], len = offsets[i + 1] - offsets[i];
    if (base < 0 || len < 0 || offsets[i + 1] > packed_bytes || in.scan_offset < 0 || in.scan_bytes < 0 ||
        in.scan_offset + in.scan_bytes > len) {
      set_last_error("jpeg: image %d lies outside the packed input", i);
      return 1;
    }
    std::vector<std::pair<int64_t, int64_t>> ranges;
    char msg[160];
    Why why{msg, sizeof(msg)};
    int nseg = 0;
    int64_t mp = 0;
    if (walk_scan(packed + base, len, in.scan_offset, &ranges, &nseg, &mp, &why) || nseg != in.num_segments) {
      set_last_error("jpeg: image %d does not match its pg_jpeg_info", i);
      return 1;
    }
    const int total_mcus = d.mcux * d.mcuy;
    const int ri = d.restart_interval ? d.restart_interval : total_mcus;
    for (int s = 0; s < nseg; ++s) {
      Seg sg;
      sg.start = base + ranges[s].first;
      sg.end = base + ranges[s].second;
      sg.img = k;
      sg.mcu0 = s * ri;
      sg.nmcu = std::min(ri, total_mcus - sg.mcu0);
      P->segs.push_back(sg);
    }
    ++k;
  }
  return 0;
}

}  // namespace

int jpeg_parse(const uint8_t* data, int64_t bytes, pg_jpeg_info* info) {
  if (!info) { set_last_error("pg_jpeg_parse: null info"); return -1; }
  char msg[200];
  Why why{msg, sizeof(msg)};
  msg[0] = 0;
  const int st = parse(data, bytes, info, nullptr, &why);
  if (st) set_last_error("%s", msg);
  return st;
}

int jpeg_parse_multiscan(const uint8_t* data, int64_t bytes, pg_jpeg_info* info) {
  if (!info) { set_last_error("pg_jpeg_parse_multiscan: null info"); return -1; }
  char msg[200];
  Why why{msg, sizeof(msg)};
  msg[0] = 0;
  MultiScan ms;
  const int st = parse_multiscan(data, bytes, info, &ms, &why);
  if (st) set_last_error("%s", msg);
  return st;
}

int jpeg_scans(const uint8_t* data, int64_t bytes, pg_jpeg_scan* out, int cap) {
  char msg[200];
  Why why{msg, sizeof(msg)};
  msg[0] = 0;
  MultiScan ms;
  pg_jpeg_info info;
  if (parse_multiscan(data, bytes, &info, &ms, &why) != PG_JPEG_OK) {
    set_last_error("%s", msg);
    return -1;
  }
  std::vector<pg_jpeg_scan> scans;
  if (info.table_mask & PG_JPEG_MULTISCAN) {
    for (const ScanRec& r : ms.scans) scans.push_back(r.pub);
  } else {                                            // a single-scan file, as pg_jpeg_parse describes it
    pg_jpeg_scan p;
    memset(&p, 0, sizeof(p));
    p.components = info.components;
    for (int c = 0; c < info.components; ++c) p.component[c] = c;
    p.se = 63;
    p.restart_interval = info.restart_interval;
    p.num_segments = info.num_segments;
    p.level = 1;
    scans.push_back(p);
  }
  for (int i = 0; i < (int)scans.size() && i < cap && out; ++i) out[i] = scans[i];
  return (int)scans.size();
}

int jpeg_set_schedule(int mode, int chunk_bytes) {
  if (mode < 0 || mode > 2 || chunk_bytes < 0) {
    set_last_error("pg_jpeg_set_schedule: mode %d not in {0, 1, 2} or chunk_bytes %d < 0", mode, chunk_bytes);
    return 1;
  }
  g_jpeg_schedule.store(mode, std::memory_order_relaxed);
  g_jpeg_chunk_bytes.store(chunk_bytes, std::memory_order_relaxed);
  return 0;
}

int64_t jpeg_entropy_host(const uint8_t* packed, const int64_t* offsets, const pg_jpeg_info* infos, int n, int chunk_bytes,
                          int16_t* coef_out, int32_t* status_out, int32_t* rounds_out) {
  if (!packed || !offsets || !infos || !status_out || n <= 0) {
    set_last_error("pg_jpeg_entropy_host: null argument");
    return -1;
  }
  for (int i = 0; i < n; ++i)
    if (infos[i].status == PG_JPEG_OK && (infos[i].table_mask & PG_JPEG_MULTISCAN)) {
      set_last_error("pg_jpeg_entropy_host: image %d is a multi-scan file", i);
      return -1;
    }
  Plan P;
  if (make_plan(packed, offsets, infos, n, offsets[n], nullptr, &P)) return -1;
  std::vector<int16_t> own;
  int16_t* coef = coef_out;
  if (!coef) {
    own.resize((size_t)P.nblocks * 64);
    coef = own.data();
  }
  memset(coef, 0, (size_t)P.nblocks * 128);
  for (int i = 0; i < n; ++i) {
    status_out[i] = infos[i].status;
    if (rounds_out) rounds_out[i] = 0;
  }
  alignas(16) int16_t blk[64];
  for (const Seg& sg : P.segs) {
    const ImgDesc& im = P.imgs[sg.img];
    int err = 0, rounds = 0;
    if (chunk_bytes == 0) err = decode_segment(packed, im, P.tbls.data(), sg, blk, coef);
    else err = chunked_segment_host(packed, im, P.tbls.data(), sg, std::max(chunk_bytes, 0), coef, &rounds);
    if (err && !status_out[im.orig]) status_out[im.orig] = err;
    if (rounds_out) rounds_out[im.orig] = std::max(rounds_out[im.orig], rounds);
  }
  return P.nblocks;
}

size_t jpeg_workspace_bytes(const pg_jpeg_info* infos, int n, int64_t packed_bytes) {
  Plan P;
  if (make_plan(nullptr, nullptr, infos, n, packed_bytes, nullptr, &P)) return 0;
  return P.total;
}

int jpeg_decode(const uint8_t* packed, const int64_t* offsets, const pg_jpeg_info* infos, int n, const pg_image* dst,
                void* workspace, size_t workspace_bytes, int32_t* status_out, cudaStream_t stream) {
  if (!packed || !offsets || !infos || !dst || !status_out || n <= 0) {
    set_last_error("pg_jpeg_decode: null argument");
    return 1;
  }
  Plan P;
  if (make_plan(packed, offsets, infos, n, offsets[n], dst, &P)) return 1;
  // short segments (restart intervals, small files) first, one thread each; then the long ones, one CTA each
  const int schedule = g_jpeg_schedule.load(std::memory_order_relaxed);
  const int forced = g_jpeg_chunk_bytes.load(std::memory_order_relaxed);
  const int nshort = (int)(std::stable_partition(P.segs.begin(), P.segs.end(), [schedule](const Seg& s) {
                             return schedule == 1 || (schedule == 0 && s.end - s.start < LONG_SEGMENT_BYTES);
                           }) - P.segs.begin());
  const int nlong = (int)P.segs.size() - nshort;
  if (!workspace || workspace_bytes < P.total || (reinterpret_cast<uintptr_t>(workspace) & 255)) {
    set_last_error("pg_jpeg_decode: workspace too small (%zu < %zu) or not 256-byte aligned", workspace_bytes, P.total);
    return 1;
  }
  uint8_t* ws = reinterpret_cast<uint8_t*>(workspace);
  const size_t nimg = P.imgs.size();
  std::vector<uint8_t> meta(P.meta_bytes, 0);
  memcpy(meta.data() + P.off_imgs, P.imgs.data(), nimg * sizeof(ImgDesc));
  memcpy(meta.data() + P.off_tbls, P.tbls.data(), P.tbls.size() * sizeof(HuffTbl));
  memcpy(meta.data() + P.off_segs, P.segs.data(), P.segs.size() * sizeof(Seg));
  memcpy(meta.data() + P.off_planes, P.planes.data(), P.planes.size() * sizeof(PlaneWork));
  memcpy(meta.data() + P.off_pix0, P.pix0.data(), nimg * sizeof(long long));
  memcpy(meta.data() + P.off_scans, P.scans.data(), P.scans.size() * sizeof(ScanDesc));
  memcpy(meta.data() + P.off_msegs, P.msegs.data(), P.msegs.size() * sizeof(MSeg));
  std::vector<int32_t> host_status(n);   // the parse status of skipped images, 0 for the ones the kernels decode
  for (int i = 0; i < n; ++i) host_status[i] = infos[i].status;
  cudaError_t e = cudaMemcpyAsync(ws + P.off_bytes, packed, (size_t)offsets[n], cudaMemcpyHostToDevice, stream);
  if (e == cudaSuccess)
    e = cudaMemcpyAsync(ws + P.off_meta, meta.data(), P.meta_bytes, cudaMemcpyHostToDevice, stream);
  if (e == cudaSuccess)
    e = cudaMemcpyAsync(status_out, host_status.data(), (size_t)n * sizeof(int32_t), cudaMemcpyHostToDevice, stream);
  if (e != cudaSuccess) { set_last_error("pg_jpeg_decode: upload: %s", cudaGetErrorString(e)); return 1; }
  if (nimg == 0) return 0;
  const uint8_t* meta_d = ws + P.off_meta;
  const ImgDesc* d_imgs = reinterpret_cast<const ImgDesc*>(meta_d + P.off_imgs);
  const HuffTbl* d_tbls = reinterpret_cast<const HuffTbl*>(meta_d + P.off_tbls);
  const Seg* d_segs = reinterpret_cast<const Seg*>(meta_d + P.off_segs);
  const PlaneWork* d_pw = reinterpret_cast<const PlaneWork*>(meta_d + P.off_planes);
  const long long* d_pix0 = reinterpret_cast<const long long*>(meta_d + P.off_pix0);
  int16_t* d_coef = reinterpret_cast<int16_t*>(ws + P.off_coef);
  uint8_t* d_planes = ws + P.off_plane;
  int sms = 132;
  {
    int dev = 0;
    if (cudaGetDevice(&dev) == cudaSuccess) cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  }
  // one segment per warp until every SM holds 16 warps, then pack lanes
  auto lanes_for = [sms](long long segs) {
    return (int)std::min<long long>(ENTROPY_THREADS, std::max<long long>(1, (segs + 16LL * sms - 1) / (16LL * sms)));
  };
  if (!P.msegs.empty()) {
    // before any entropy launch: the range of multi-scan blocks may hold baseline images between them
    ProfScope prof("jpeg_zero_coef", stream);
    e = cudaMemsetAsync(d_coef + P.multi_coef0 * 64, 0, (size_t)(P.multi_coef1 - P.multi_coef0) * 128, stream);
    if (e != cudaSuccess) { set_last_error("pg_jpeg_decode: memset: %s", cudaGetErrorString(e)); return 1; }
  }
  if (nshort > 0) {
    const int lanes = lanes_for(nshort);
    ProfScope prof("jpeg_entropy", stream);
    entropy_kernel<<<(nshort + lanes - 1) / lanes, ENTROPY_THREADS, 0, stream>>>(ws + P.off_bytes, d_imgs, d_tbls, d_segs,
                                                                                  nshort, lanes, d_coef, status_out);
  }
  if (nlong > 0) {
    const int cap = forced > 0 ? MAX_CHUNKS : CHUNK_THREADS;     // chunk_geometry's bound on a segment's chunks
    const size_t smem = (size_t)cap * (2 * sizeof(long long) + sizeof(int) + 3 * sizeof(unsigned));
    e = cudaFuncSetAttribute(chunked_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) { set_last_error("pg_jpeg_decode: %s", cudaGetErrorString(e)); return 1; }
    ProfScope prof("jpeg_entropy_chunked", stream);
    chunked_kernel<<<nlong, CHUNK_THREADS, smem, stream>>>(ws + P.off_bytes, d_imgs, d_tbls, d_segs + nshort, cap, forced,
                                                           ws + P.off_destuff, d_coef, status_out);
  }
  if (!P.msegs.empty()) {
    // Multi-scan images (coefficients zeroed above): one launch per dependency level.  The scans of one level share
    // no coefficient; a later level reads what earlier ones wrote, ordered by the stream alone.
    static const char* level_names[] = {"jpeg_entropy_multiscan.1", "jpeg_entropy_multiscan.2", "jpeg_entropy_multiscan.3",
                                        "jpeg_entropy_multiscan.4", "jpeg_entropy_multiscan.5+"};
    const ScanDesc* d_scans = reinterpret_cast<const ScanDesc*>(meta_d + P.off_scans);
    const MSeg* d_msegs = reinterpret_cast<const MSeg*>(meta_d + P.off_msegs);
    for (size_t L = 0; L + 1 < P.level0.size(); ++L) {
      const int s0 = P.level0[L], ns = P.level0[L + 1] - s0;
      if (ns == 0) continue;
      const int lanes = lanes_for(ns);
      ProfScope prof(level_names[std::min<size_t>(L, 4)], stream);
      multiscan_kernel<<<(ns + lanes - 1) / lanes, ENTROPY_THREADS, 0, stream>>>(
          ws + P.off_bytes, d_imgs, d_tbls, d_scans, d_msegs + s0, ns, lanes, d_coef, status_out);
    }
  }
  {
    ProfScope prof("jpeg_idct", stream);
    idct_kernel<<<(unsigned)((P.nblocks + 127) / 128), 128, 0, stream>>>(d_imgs, d_pw, (int)P.planes.size(), P.nblocks,
                                                                         d_coef, d_planes, status_out);
  }
  {
    ProfScope prof("jpeg_color", stream);
    color_kernel<<<(unsigned)((P.npix + 255) / 256), 256, 0, stream>>>(d_imgs, d_pix0, (int)nimg, P.npix, d_planes, status_out);
  }
  e = cudaGetLastError();
  if (e != cudaSuccess) { set_last_error("pg_jpeg_decode launch: %s", cudaGetErrorString(e)); return 1; }
  return 0;
}

}  // namespace pg

extern "C" int pg_jpeg_parse(const uint8_t* data_host, int64_t bytes, pg_jpeg_info* info_out) {
  return pg::jpeg_parse(data_host, bytes, info_out);
}

extern "C" int pg_jpeg_parse_multiscan(const uint8_t* data_host, int64_t bytes, pg_jpeg_info* info_out) {
  return pg::jpeg_parse_multiscan(data_host, bytes, info_out);
}

extern "C" int pg_jpeg_scans(const uint8_t* data_host, int64_t bytes, pg_jpeg_scan* out, int32_t cap) {
  return pg::jpeg_scans(data_host, bytes, out, cap);
}

extern "C" int pg_jpeg_set_schedule(int32_t mode, int32_t chunk_bytes) { return pg::jpeg_set_schedule(mode, chunk_bytes); }

extern "C" int64_t pg_jpeg_entropy_host(const uint8_t* packed_host, const int64_t* offsets_host,
                                        const pg_jpeg_info* infos_host, int32_t n, int32_t chunk_bytes, int16_t* coef_out,
                                        int32_t* status_out, int32_t* rounds_out) {
  return pg::jpeg_entropy_host(packed_host, offsets_host, infos_host, n, chunk_bytes, coef_out, status_out, rounds_out);
}

extern "C" size_t pg_jpeg_workspace_bytes(const pg_jpeg_info* infos_host, int32_t n, int64_t packed_bytes) {
  return pg::jpeg_workspace_bytes(infos_host, n, packed_bytes);
}

extern "C" int pg_jpeg_decode(const uint8_t* packed_host, const int64_t* offsets_host, const pg_jpeg_info* infos_host,
                              int32_t n, const pg_image* dst_host, void* workspace, size_t workspace_bytes,
                              int32_t* status_out, void* stream) {
  return pg::jpeg_decode(packed_host, offsets_host, infos_host, n, dst_host, workspace, workspace_bytes, status_out,
                         reinterpret_cast<cudaStream_t>(stream));
}
