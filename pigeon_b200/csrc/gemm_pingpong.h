// Launcher of the ping-pong GEMM kernel (gemm_pingpong.cu); gemm_wgmma.cu validates the problem, builds the tensor maps and
// picks this kernel, the 128 x 256 one (gemm_wide.cuh) or its own single-warpgroup one.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>

#include "gemm_epilogue.cuh"

namespace pg {

// K-major operands only (tensor-map boxes 128 x 64 for A and W).  `grid` persistent CTAs of 384 threads.
int gemm_pingpong_launch(int epi, bool bf16, const CUtensorMap& ta, const CUtensorMap& tb, const GemmArgs& args, int grid,
                         cudaStream_t stream);

}  // namespace pg
