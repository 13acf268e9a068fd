// Launcher of the 128 x 256 GEMM kernel (gemm_wide.cuh, instantiated in gemm_wide.cu and gemm_wide_resid.cu); gemm_wgmma.cu
// validates the problem, builds the tensor maps and picks this kernel, the ping-pong one or its own single-warpgroup one.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>

#include "gemm_epilogue.cuh"

namespace pg {

constexpr int kWideBlockN = 256;   // output tile 128 x 256; W's tensor-map box is kWideBlockN x 64

// The epilogues the kernel implements: fp16 output with nothing written but the output, and the fp32 residual updates.
constexpr bool gemm_wide_epilogue(int epi) {
  return epi == EPI_F16_BIAS || epi == EPI_F16_BIAS_QGELU || epi == EPI_F16_LN_BIAS || epi == EPI_F16_LN_BIAS_QGELU ||
         epi == EPI_F32_BIAS_RESID || epi == EPI_F32_BIAS_RESID_STATS;
}

// K-major operands only: tensor-map boxes 128 x 64 for A, 256 x 64 for W (128B swizzle).  `tout`: the fp16 output in 64 x 64
// boxes, or for the residual epilogues the fp32 output in 64 x 32 boxes, `tres` the fp32 residual source in 64 x 32 boxes
// and `taux` the fp16 copy (EPI_F32_BIAS_RESID_STATS) in 64 x 64 boxes; a map the epilogue does not use is not read.
// `grid` persistent CTAs of 384 threads over the 128 x 256 tiles.
int gemm_wide_launch(int epi, bool bf16, const CUtensorMap& ta, const CUtensorMap& tb, const CUtensorMap& tout,
                     const CUtensorMap& tres, const CUtensorMap& taux, const GemmArgs& args, int grid, cudaStream_t stream);

}  // namespace pg
