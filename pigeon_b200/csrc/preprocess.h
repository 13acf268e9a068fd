// Internal (C++) interface of the image pre-processing kernels; see preprocess.cu.
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

struct pg_image;
struct pg_window;

namespace pg {

// `windows` may be NULL: every image is its own source rectangle (pg_preprocess_clip).
size_t preprocess_workspace_bytes(const pg_image* images, const pg_window* windows, int n, int size);
int preprocess_clip(const pg_image* images, const pg_window* windows, int n, int size, const float* mean,
                    const float* stdv, void* workspace, size_t workspace_bytes, void* out, int out_f16,
                    cudaStream_t stream);

}  // namespace pg
