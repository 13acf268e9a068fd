// 128 x 256 cooperative wgmma GEMM (gemm_wide.cuh) with the fp32 residual epilogues: out_proj and fc2 of the vision tower,
// EPI_F32_BIAS_RESID and EPI_F32_BIAS_RESID_STATS (the residual read and written by TMA in 64-column steps, see the header).
#include "gemm_wide.cuh"

namespace pg {

int gemm_wide_resid_launch(int epi, bool bf16, const CUtensorMap& ta, const CUtensorMap& tb, const CUtensorMap& tout,
                           const CUtensorMap& tres, const CUtensorMap& taux, const GemmArgs& a, int grid, cudaStream_t stream) {
  switch (epi) {
    case EPI_F32_BIAS_RESID:        return launch<EPI_F32_BIAS_RESID>(bf16, ta, tb, tout, tres, taux, a, grid, stream);
    case EPI_F32_BIAS_RESID_STATS:  return launch<EPI_F32_BIAS_RESID_STATS>(bf16, ta, tb, tout, tres, taux, a, grid, stream);
    default: set_last_error("gemm: epilogue %d is not a residual epilogue", epi); return 1;
  }
}

}  // namespace pg
