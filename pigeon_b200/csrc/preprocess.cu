// CLIPProcessor image pre-processing on the GPU ("next" row N2): uint8 RGB images of arbitrary size ->
// resize shortest edge to `size` (Pillow BICUBIC) -> center crop -> /255 -> (x - mean) / std -> [n, 3, size, size].
// Bit-exact with Pillow's libImaging/Resample.c: coefficients are evaluated in double with the same operation order
// (no FMA contraction: explicit *_rn intrinsics), normalised, rounded to 22-bit fixed point; the horizontal pass runs
// first and leaves a rounded, clipped uint8 intermediate; then the vertical pass.  Only the rows / columns that
// survive the center crop are computed.  Byte/integer work, HBM-bound: one block per image row, rows staged in
// shared memory, coalesced stores.
//
// pg_preprocess_clip_window first cuts each image to a source rectangle that may extend past it (torchvision's
// CenterCrop, which pads, or a Pillow crop box): the rectangle stands in for the image in every step above, and a
// sample outside the image reads the image's fill colour.  The bounds test sits where a row is staged into shared
// memory, so no padded copy of an image is ever made.  Images are walked grid-stride along grid.y, so a batch may hold
// more than 65535 of them.
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <math.h>

#include <vector>

#include "../../include/pigeon_b200.h"
#include "preprocess.h"
#include "prof.h"
#include "tma_host.h"

namespace pg {
namespace {

constexpr int PRECISION_BITS = 32 - 8 - 2;
constexpr int MAX_KSIZE = 513;          // down-scaling factors up to 128
constexpr int MAX_WIDTH_BYTES = 96 * 1024;
constexpr int MAX_GRID_IMAGES = 65535;  // grid.y limit: the kernels loop over images beyond it

struct Plan {                           // per image, computed on the host (integer + a few double operations)
  const uint8_t* data;
  long long row_stride;
  int height, width;                    // of the source rectangle (the whole image without a window)
  int new_h, new_w;                     // size after the shortest-edge resize
  int top, left;                        // center-crop origin in the resized image
  int first_row, num_rows;              // input rows the vertical pass reads
  int ksize_h, ksize_v;
  long long inter_off;                  // byte offset of this image's intermediate in the workspace
};

struct Crop {                           // per image of a windowed call: where the source rectangle lies
  int src_h, src_w;                     // the image itself
  int x0, y0;                           // source rectangle origin in the image; may be negative
  uint32_t fill;                        // RGB of samples outside the image, R in the low byte
};

struct Layout {
  size_t plans, crops, coef, bounds, inter, total;
  int ks;                               // coefficient row stride (max ksize in the batch)
  int max_rows, max_row_bytes;
};

inline size_t align_up(size_t x, size_t a) { return (x + a - 1) / a * a; }

// Resample.c precompute_coeffs, bounds of one output index (host copy; the device recomputes them per index).
void host_bounds(int in_size, int out_size, int xx, int* xmin_out, int* xmax_out, int* ksize_out) {
  volatile double scale = (double)in_size / (double)out_size;
  volatile double filterscale = scale < 1.0 ? 1.0 : scale;
  volatile double support = 2.0 * filterscale;
  volatile double center = (xx + 0.5) * scale;
  volatile double lo = center - support;
  volatile double hi = center + support;
  int xmin = (int)(lo + 0.5);
  if (xmin < 0) xmin = 0;
  int xmax = (int)(hi + 0.5);
  if (xmax > in_size) xmax = in_size;
  *xmin_out = xmin;
  *xmax_out = xmax - xmin;
  *ksize_out = (int)ceil(support) * 2 + 1;
}

int make_plans(const pg_image* images, const pg_window* windows, int n, int size, std::vector<Plan>* plans,
               std::vector<Crop>* crops, Layout* lay) {
  if (!images || n <= 0 || size <= 0 || size > 1024) { set_last_error("preprocess: bad argument"); return 1; }
  plans->resize(n);
  crops->resize(windows ? n : 0);
  long long inter = 0;
  int ks = 0, max_rows = 0, max_row_bytes = 0;
  for (int i = 0; i < n; ++i) {
    const pg_image& im = images[i];
    Plan& p = (*plans)[i];
    if (!im.data || im.height <= 0 || im.width <= 0 || im.row_stride < (long long)im.width * 3) {
      set_last_error("preprocess: image %d has a bad descriptor", i);
      return 1;
    }
    p.data = im.data; p.row_stride = im.row_stride; p.height = im.height; p.width = im.width;
    if (windows) {
      const pg_window& w = windows[i];
      if (w.width <= 0 || w.height <= 0) {
        set_last_error("preprocess: window %d is empty (%dx%d)", i, w.width, w.height);
        return 1;
      }
      if (w.x0 < -(1 << 30) || w.x0 > (1 << 30) || w.y0 < -(1 << 30) || w.y0 > (1 << 30) || w.height > (1 << 30)) {
        set_last_error("preprocess: window %d (%d, %d, %dx%d) is out of range", i, w.x0, w.y0, w.width, w.height);
        return 1;
      }
      Crop& c = (*crops)[i];
      c.src_h = im.height; c.src_w = im.width; c.x0 = w.x0; c.y0 = w.y0;
      c.fill = (uint32_t)w.fill[0] | (uint32_t)w.fill[1] << 8 | (uint32_t)w.fill[2] << 16;
      p.height = w.height; p.width = w.width;
    }
    // transformers 4.23.1 image_utils.resize(default_to_square=False): int(size * long / short) in double
    const int shortest = p.width <= p.height ? p.width : p.height;
    const int longest = p.width <= p.height ? p.height : p.width;
    int new_short = size, new_long;
    if (shortest == size) new_long = longest;
    else { volatile double q = (double)size * (double)longest; q = q / (double)shortest; new_long = (int)q; }
    p.new_w = p.width <= p.height ? new_short : new_long;
    p.new_h = p.width <= p.height ? new_long : new_short;
    p.top = (p.new_h - size) / 2; p.left = (p.new_w - size) / 2;   // non-negative: both edges >= size
    int a0, a1, b0, b1, kv, kh, d0, d1;
    host_bounds(p.height, p.new_h, p.top, &a0, &a1, &kv);
    host_bounds(p.height, p.new_h, p.top + size - 1, &b0, &b1, &kv);
    host_bounds(p.width, p.new_w, p.left, &d0, &d1, &kh);
    p.first_row = a0; p.num_rows = b0 + b1 - a0;
    p.ksize_h = kh; p.ksize_v = kv;
    if (kh > MAX_KSIZE || kv > MAX_KSIZE || p.width * 3 > MAX_WIDTH_BYTES) {
      set_last_error("preprocess: image %d (%dx%d) exceeds the supported down-scaling factor / width", i, p.width, p.height);
      return 1;
    }
    p.inter_off = inter;
    inter += (long long)align_up((size_t)p.num_rows * size * 3, 256);
    ks = kh > ks ? kh : ks; ks = kv > ks ? kv : ks;
    max_rows = p.num_rows > max_rows ? p.num_rows : max_rows;
    max_row_bytes = p.width * 3 > max_row_bytes ? p.width * 3 : max_row_bytes;
  }
  lay->ks = ks; lay->max_rows = max_rows; lay->max_row_bytes = max_row_bytes;
  size_t off = 0;
  lay->plans = off; off += align_up((size_t)n * sizeof(Plan), 256);
  lay->crops = off; off += align_up((size_t)crops->size() * sizeof(Crop), 256);   // 0 without windows
  lay->coef = off; off += align_up((size_t)n * 2 * size * ks * sizeof(int), 256);
  lay->bounds = off; off += align_up((size_t)n * 2 * size * 2 * sizeof(int), 256);
  lay->inter = off; off += (size_t)inter;
  lay->total = off;
  return 0;
}

__device__ __forceinline__ double bicubic_filter(double x) {
  const double a = -0.5;
  if (x < 0.0) x = -x;
  if (x < 1.0) {   // ((a + 2.0) * x - (a + 3.0)) * x * x + 1
    double t = __dsub_rn(__dmul_rn(a + 2.0, x), a + 3.0);
    t = __dmul_rn(__dmul_rn(t, x), x);
    return __dadd_rn(t, 1.0);
  }
  if (x < 2.0) {   // (((x - 5) * x + 8) * x - 4) * a
    double t = __dadd_rn(__dmul_rn(__dsub_rn(x, 5.0), x), 8.0);
    t = __dsub_rn(__dmul_rn(t, x), 4.0);
    return __dmul_rn(t, a);
  }
  return 0.0;
}

// One thread per (image, axis, cropped output index): Resample.c precompute_coeffs + normalize_coeffs_8bpc.
__global__ void __launch_bounds__(128)
coeff_kernel(const Plan* __restrict__ plans, int n, int size, int ks, int* __restrict__ coef, int* __restrict__ bounds) {
  const int axis = blockIdx.z;
  const int o = blockIdx.x * 128 + threadIdx.x;
  if (o >= size) return;
  for (int img = blockIdx.y; img < n; img += gridDim.y) {
    const Plan p = plans[img];
    const int in_size = axis ? p.height : p.width, out_size = axis ? p.new_h : p.new_w;
    const int xx = o + (axis ? p.top : p.left);
    const double scale = __ddiv_rn((double)in_size, (double)out_size);
    const double filterscale = scale < 1.0 ? 1.0 : scale;
    const double support = __dmul_rn(2.0, filterscale);
    const double ss = __ddiv_rn(1.0, filterscale);
    const double center = __dmul_rn((double)xx + 0.5, scale);
    int xmin = __double2int_rz(__dadd_rn(__dsub_rn(center, support), 0.5));
    if (xmin < 0) xmin = 0;
    int xmax = __double2int_rz(__dadd_rn(__dadd_rn(center, support), 0.5));
    if (xmax > in_size) xmax = in_size;
    xmax -= xmin;
    int* k = coef + (((long)img * 2 + axis) * size + o) * ks;
    double ww = 0.0;
    for (int x = 0; x < xmax; ++x)
      ww = __dadd_rn(ww, bicubic_filter(__dmul_rn(__dadd_rn(__dsub_rn((double)(x + xmin), center), 0.5), ss)));
    for (int x = 0; x < xmax; ++x) {
      double w = bicubic_filter(__dmul_rn(__dadd_rn(__dsub_rn((double)(x + xmin), center), 0.5), ss));
      if (ww != 0.0) w = __ddiv_rn(w, ww);
      const double scaled = __dmul_rn(w, (double)(1 << PRECISION_BITS));
      k[x] = __double2int_rz(w < 0 ? __dadd_rn(-0.5, scaled) : __dadd_rn(0.5, scaled));
    }
    for (int x = xmax; x < ks; ++x) k[x] = 0;
    int* b = bounds + (((long)img * 2 + axis) * size + o) * 2;
    b[0] = xmin;
    b[1] = xmax;
  }
}

__device__ __forceinline__ int clip8(int v) {
  v >>= PRECISION_BITS;
  return v < 0 ? 0 : (v > 255 ? 255 : v);
}

// grid (max_rows, n): one input row -> `size` cropped output columns x 3 channels of the intermediate.
__global__ void __launch_bounds__(256)
horizontal_kernel(const Plan* __restrict__ plans, const Crop* __restrict__ crops, int n, int size, int ks,
                  const int* __restrict__ coef, const int* __restrict__ bounds, uint8_t* __restrict__ inter_base) {
  extern __shared__ uint8_t row[];
  const int r = blockIdx.x;
  for (int img = blockIdx.y; img < n; img += gridDim.y) {
    const Plan p = plans[img];
    if (r >= p.num_rows) continue;            // uniform per block: no thread reaches the barriers below
    const Crop c = crops ? crops[img] : Crop{p.height, p.width, 0, 0, 0u};
    const int sy = c.y0 + p.first_row + r;    // image row of this source-rectangle row
    const int nbytes = p.width * 3;
    const bool row_in = sy >= 0 && sy < c.src_h;
    if (row_in && c.x0 >= 0 && c.x0 + p.width <= c.src_w) {
      const uint8_t* src = p.data + (long long)sy * p.row_stride + (long long)c.x0 * 3;
      if ((((uintptr_t)src) & 3) == 0) {
        const int nw = nbytes >> 2;
        for (int i = threadIdx.x; i < nw; i += 256) reinterpret_cast<uint32_t*>(row)[i] = reinterpret_cast<const uint32_t*>(src)[i];
        for (int i = (nw << 2) + threadIdx.x; i < nbytes; i += 256) row[i] = src[i];
      } else {
        for (int i = threadIdx.x; i < nbytes; i += 256) row[i] = src[i];
      }
    } else {                                  // the rectangle leaves the image: samples outside it read the fill
      const uint8_t* src = p.data + (row_in ? (long long)sy * p.row_stride : 0);
      for (int i = threadIdx.x; i < nbytes; i += 256) {
        const int x = c.x0 + i / 3, ch = i - (i / 3) * 3;
        row[i] = row_in && x >= 0 && x < c.src_w ? src[(long long)x * 3 + ch] : (uint8_t)(c.fill >> (8 * ch));
      }
    }
    __syncthreads();
    const int* cbase = coef + ((long)img * 2 + 0) * size * ks;
    const int* bbase = bounds + ((long)img * 2 + 0) * size * 2;
    uint8_t* dst = inter_base + p.inter_off + (long long)r * size * 3;
    for (int o = threadIdx.x; o < size * 3; o += 256) {
      const int j = o / 3, ch = o - j * 3;
      const int xmin = bbase[2 * j], xmax = bbase[2 * j + 1];
      const int* k = cbase + (long)j * ks;
      const uint8_t* s = row + xmin * 3 + ch;
      int acc = 1 << (PRECISION_BITS - 1);
      for (int t = 0; t < xmax; ++t) acc += (int)s[t * 3] * k[t];
      dst[o] = (uint8_t)clip8(acc);
    }
    __syncthreads();                          // the next image's staging overwrites `row`
  }
}

// grid (size, n): one output row -> 3 x size normalised values, channel-first.
template <typename OutT>
__global__ void __launch_bounds__(256)
vertical_kernel(const Plan* __restrict__ plans, int n, int size, int ks, const int* __restrict__ coef,
                const int* __restrict__ bounds, const uint8_t* __restrict__ inter_base, float m0, float m1, float m2,
                float s0, float s1, float s2, OutT* __restrict__ out) {
  __shared__ int k[MAX_KSIZE];
  const int y = blockIdx.x;
  for (int img = blockIdx.y; img < n; img += gridDim.y) {
    const Plan p = plans[img];
    const int* kb = coef + (((long)img * 2 + 1) * size + y) * ks;
    const int ymin = bounds[(((long)img * 2 + 1) * size + y) * 2], ymax = bounds[(((long)img * 2 + 1) * size + y) * 2 + 1];
    for (int t = threadIdx.x; t < ymax; t += 256) k[t] = kb[t];
    __syncthreads();
    const uint8_t* src = inter_base + p.inter_off + (long long)(ymin - p.first_row) * size * 3;
    OutT* dst = out + (long long)img * 3 * size * size + (long long)y * size;
    for (int o = threadIdx.x; o < size * 3; o += 256) {
      const int c = o / size, j = o - c * size;
      const uint8_t* s = src + j * 3 + c;
      int acc = 1 << (PRECISION_BITS - 1);
      for (int t = 0; t < ymax; ++t) acc += (int)s[(long)t * size * 3] * k[t];
      // numpy: x.astype(float32) / 255.0, then (x - mean) / std, all in float32
      float v = __fdiv_rn((float)clip8(acc), 255.0f);
      const float m = c == 0 ? m0 : (c == 1 ? m1 : m2), sd = c == 0 ? s0 : (c == 1 ? s1 : s2);
      v = __fdiv_rn(__fsub_rn(v, m), sd);
      dst[(long long)c * size * size + j] = (OutT)v;
    }
    __syncthreads();                          // the next image's coefficients overwrite `k`
  }
}

}  // namespace

size_t preprocess_workspace_bytes(const pg_image* images, const pg_window* windows, int n, int size) {
  std::vector<Plan> plans;
  std::vector<Crop> crops;
  Layout lay;
  if (make_plans(images, windows, n, size, &plans, &crops, &lay)) return 0;
  return lay.total;
}

int preprocess_clip(const pg_image* images, const pg_window* windows, int n, int size, const float* mean,
                    const float* stdv, void* workspace, size_t workspace_bytes, void* out, int out_f16,
                    cudaStream_t stream) {
  std::vector<Plan> plans;
  std::vector<Crop> crops;
  Layout lay;
  if (make_plans(images, windows, n, size, &plans, &crops, &lay)) return 1;
  if (!workspace || workspace_bytes < lay.total || !out || !mean || !stdv) {
    set_last_error("preprocess: workspace too small (%zu < %zu) or null output", workspace_bytes, lay.total);
    return 1;
  }
  uint8_t* ws = reinterpret_cast<uint8_t*>(workspace);
  Plan* d_plans = reinterpret_cast<Plan*>(ws + lay.plans);
  int* d_coef = reinterpret_cast<int*>(ws + lay.coef);
  int* d_bounds = reinterpret_cast<int*>(ws + lay.bounds);
  uint8_t* d_inter = ws + lay.inter;
  // pageable source: the runtime stages the bytes before returning, so `plans` may go out of scope
  cudaError_t e = cudaMemcpyAsync(d_plans, plans.data(), (size_t)n * sizeof(Plan), cudaMemcpyHostToDevice, stream);
  if (e != cudaSuccess) { set_last_error("preprocess: plan upload: %s", cudaGetErrorString(e)); return 1; }
  Crop* d_crops = nullptr;
  if (windows) {
    d_crops = reinterpret_cast<Crop*>(ws + lay.crops);
    e = cudaMemcpyAsync(d_crops, crops.data(), (size_t)n * sizeof(Crop), cudaMemcpyHostToDevice, stream);
    if (e != cudaSuccess) { set_last_error("preprocess: window upload: %s", cudaGetErrorString(e)); return 1; }
  }
  ProfScope prof("preprocess_clip", stream);
  const int gy = n < MAX_GRID_IMAGES ? n : MAX_GRID_IMAGES;
  coeff_kernel<<<dim3((size + 127) / 128, gy, 2), 128, 0, stream>>>(d_plans, n, size, lay.ks, d_coef, d_bounds);
  const size_t smem = align_up((size_t)lay.max_row_bytes, 16);
  if (smem > 48 * 1024) {
    e = cudaFuncSetAttribute(horizontal_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) { set_last_error("preprocess: smem attr: %s", cudaGetErrorString(e)); return 1; }
  }
  horizontal_kernel<<<dim3(lay.max_rows, gy), 256, smem, stream>>>(d_plans, d_crops, n, size, lay.ks, d_coef, d_bounds,
                                                                   d_inter);
  if (out_f16)
    vertical_kernel<__half><<<dim3(size, gy), 256, 0, stream>>>(d_plans, n, size, lay.ks, d_coef, d_bounds, d_inter,
                                                                mean[0], mean[1], mean[2], stdv[0], stdv[1], stdv[2],
                                                                reinterpret_cast<__half*>(out));
  else
    vertical_kernel<float><<<dim3(size, gy), 256, 0, stream>>>(d_plans, n, size, lay.ks, d_coef, d_bounds, d_inter,
                                                               mean[0], mean[1], mean[2], stdv[0], stdv[1], stdv[2],
                                                               reinterpret_cast<float*>(out));
  e = cudaGetLastError();
  if (e != cudaSuccess) { set_last_error("preprocess launch: %s", cudaGetErrorString(e)); return 1; }
  return 0;
}

}  // namespace pg
