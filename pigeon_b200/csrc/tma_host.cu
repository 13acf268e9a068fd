#include "tma_host.h"

#include "prof.h"

#include <stdarg.h>
#include <stdio.h>
#include <string.h>

#include <map>
#include <string>
#include <vector>

namespace pg {

namespace {
thread_local char g_err[512] = "";

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*,
                                  CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion,
                                  CUtensorMapFloatOOBfill);

EncodeTiledFn get_encode() {
  static EncodeTiledFn fn = nullptr;
  static bool tried = false;
  if (!tried) {
    tried = true;
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q);
    if (e == cudaSuccess && q == cudaDriverEntryPointSuccess) fn = reinterpret_cast<EncodeTiledFn>(p);
  }
  return fn;
}
}  // namespace

void set_last_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

const char* last_error() { return g_err; }

int make_tmap_f16_2d(CUtensorMap* out, const void* base, uint64_t rows, uint64_t cols, uint64_t ld_elems,
                     uint32_t box_rows, uint32_t box_cols) {
  EncodeTiledFn enc = get_encode();
  if (!enc) {
    set_last_error("cuTensorMapEncodeTiled unavailable (no CUDA driver?)");
    return 1;
  }
  cuuint64_t gdim[2] = {cols, rows};
  cuuint64_t gstride[1] = {ld_elems * 2};
  cuuint32_t box[2] = {box_cols, box_rows};
  cuuint32_t estride[2] = {1, 1};
  CUresult r = enc(out, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, const_cast<void*>(base), gdim, gstride, box, estride,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_last_error("cuTensorMapEncodeTiled failed: CUresult %d (rows=%llu cols=%llu ld=%llu box=%ux%u)", (int)r,
                   (unsigned long long)rows, (unsigned long long)cols, (unsigned long long)ld_elems, box_rows,
                   box_cols);
    return 1;
  }
  return 0;
}

// 16-bit [views, rows_per_view, cols] (ld_elems elements per row, views contiguous): box [1, box_rows, box_cols].  A box that
// runs past a view's last row is zero-filled instead of reading the next view's rows.
int make_tmap_f16_3d(CUtensorMap* out, const void* base, uint64_t views, uint64_t rows_per_view, uint64_t cols, uint64_t ld_elems,
                     uint32_t box_rows, uint32_t box_cols) {
  EncodeTiledFn enc = get_encode();
  if (!enc) {
    set_last_error("cuTensorMapEncodeTiled unavailable (no CUDA driver?)");
    return 1;
  }
  cuuint64_t gdim[3] = {cols, rows_per_view, views};
  cuuint64_t gstride[2] = {ld_elems * 2, rows_per_view * ld_elems * 2};
  cuuint32_t box[3] = {box_cols, box_rows, 1};
  cuuint32_t estride[3] = {1, 1, 1};
  CUresult r = enc(out, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 3, const_cast<void*>(base), gdim, gstride, box, estride,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_last_error("cuTensorMapEncodeTiled (3-D) failed: CUresult %d (views=%llu rows=%llu cols=%llu ld=%llu box=%ux%u)", (int)r,
                   (unsigned long long)views, (unsigned long long)rows_per_view, (unsigned long long)cols,
                   (unsigned long long)ld_elems, box_rows, box_cols);
    return 1;
  }
  return 0;
}

// fp32 [rows, cols] row-major (ld_elems floats per row), box [box_rows, box_cols] with box_cols * 4 == 128 bytes, 128-byte swizzle.
int make_tmap_f32_2d(CUtensorMap* out, const void* base, uint64_t rows, uint64_t cols, uint64_t ld_elems,
                     uint32_t box_rows, uint32_t box_cols) {
  EncodeTiledFn enc = get_encode();
  if (!enc) {
    set_last_error("cuTensorMapEncodeTiled unavailable (no CUDA driver?)");
    return 1;
  }
  cuuint64_t gdim[2] = {cols, rows};
  cuuint64_t gstride[1] = {ld_elems * 4};
  cuuint32_t box[2] = {box_cols, box_rows};
  cuuint32_t estride[2] = {1, 1};
  CUresult r = enc(out, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<void*>(base), gdim, gstride, box, estride,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_last_error("cuTensorMapEncodeTiled (f32) failed: CUresult %d (rows=%llu cols=%llu ld=%llu box=%ux%u)", (int)r,
                   (unsigned long long)rows, (unsigned long long)cols, (unsigned long long)ld_elems, box_rows,
                   box_cols);
    return 1;
  }
  return 0;
}

// ------------------------------------------------------------------------------------------- profiler
namespace {
struct ProfRec { const char* name; cudaEvent_t e0, e1; };
bool g_prof_on = false;
std::vector<ProfRec> g_prof_recs;
std::vector<std::string> g_prof_names;
std::vector<float> g_prof_ms;
std::vector<int> g_prof_counts;
}  // namespace

bool prof_enabled() { return g_prof_on; }
void prof_record(const char* name, cudaEvent_t start, cudaEvent_t stop) { g_prof_recs.push_back({name, start, stop}); }

void prof_begin() {
  g_prof_recs.clear();
  g_prof_on = true;
}

int prof_end() {
  g_prof_on = false;
  cudaDeviceSynchronize();
  std::map<std::string, std::pair<float, int>> agg;
  for (auto& r : g_prof_recs) {
    float ms = 0.f;
    cudaEventElapsedTime(&ms, r.e0, r.e1);
    auto& a = agg[r.name];
    a.first += ms;
    a.second += 1;
    cudaEventDestroy(r.e0);
    cudaEventDestroy(r.e1);
  }
  g_prof_recs.clear();
  g_prof_names.clear(); g_prof_ms.clear(); g_prof_counts.clear();
  for (auto& kv : agg) {
    g_prof_names.push_back(kv.first);
    g_prof_ms.push_back(kv.second.first);
    g_prof_counts.push_back(kv.second.second);
  }
  return (int)g_prof_names.size();
}

void prof_read(const char** names, float* ms, int* counts, int n) {
  for (int i = 0; i < n && i < (int)g_prof_names.size(); ++i) {
    names[i] = g_prof_names[i].c_str();
    ms[i] = g_prof_ms[i];
    counts[i] = g_prof_counts[i];
  }
}

}  // namespace pg
