// Host-side CUtensorMap construction. The driver symbol is fetched through the runtime
// (cudaGetDriverEntryPoint) so the library does not link libcuda and still loads on a CPU-only box.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace pg {

// Encode a 2-D row-major fp16 matrix [rows, cols] (row stride `ld_elems` elements) with a
// [box_rows, box_cols] tile and 128-byte swizzle. box_cols * 2 must equal 128 bytes.
// Returns 0 on success, non-zero (and sets the last-error string) on failure.
int make_tmap_f16_2d(CUtensorMap* out, const void* base, uint64_t rows, uint64_t cols,
                     uint64_t ld_elems, uint32_t box_rows, uint32_t box_cols);

// 16-bit [views, rows_per_view, cols] with a [1, box_rows, box_cols] tile: rows past a view's end are zero-filled.
int make_tmap_f16_3d(CUtensorMap* out, const void* base, uint64_t views, uint64_t rows_per_view, uint64_t cols,
                     uint64_t ld_elems, uint32_t box_rows, uint32_t box_cols);

int make_tmap_f32_2d(CUtensorMap* out, const void* base, uint64_t rows, uint64_t cols,
                     uint64_t ld_elems, uint32_t box_rows, uint32_t box_cols);

void set_last_error(const char* fmt, ...);
const char* last_error();

void prof_begin();
int prof_end();
void prof_read(const char** names, float* ms, int* counts, int n);

}  // namespace pg
