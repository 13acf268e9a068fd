// Launcher of the 128 x 256 GEMM kernel (gemm_wide.cu); gemm_wgmma.cu validates the problem, builds the tensor maps and
// picks this kernel, the ping-pong one or its own single-warpgroup one.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>

#include "gemm_epilogue.cuh"

namespace pg {

constexpr int kWideBlockN = 256;   // output tile 128 x 256; W's tensor-map box is kWideBlockN x 64

// The epilogues the kernel implements: fp16 output, nothing written but the output.
constexpr bool gemm_wide_epilogue(int epi) {
  return epi == EPI_F16_BIAS || epi == EPI_F16_BIAS_QGELU || epi == EPI_F16_LN_BIAS || epi == EPI_F16_LN_BIAS_QGELU;
}

// K-major operands only: tensor-map boxes 128 x 64 for A, 256 x 64 for W, 64 x 64 for the fp16 output (128B swizzle).
// `grid` persistent CTAs of 384 threads over the 128 x 256 tiles.
int gemm_wide_launch(int epi, bool bf16, const CUtensorMap& ta, const CUtensorMap& tb, const CUtensorMap& tout,
                     const GemmArgs& args, int grid, cudaStream_t stream);

}  // namespace pg
