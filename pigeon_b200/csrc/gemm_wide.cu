// 128 x 256 cooperative wgmma GEMM (gemm_wide.cuh): the fp16-output epilogues (qkv and fc1 of the vision tower) are
// instantiated here; the fp32 residual epilogues (out_proj and fc2) in gemm_wide_resid.cu.
#include "gemm_wide.cuh"

namespace pg {

int gemm_wide_launch(int epi, bool bf16, const CUtensorMap& ta, const CUtensorMap& tb, const CUtensorMap& tout,
                     const CUtensorMap& tres, const CUtensorMap& taux, const GemmArgs& a, int grid, cudaStream_t stream) {
  switch (epi) {
    case EPI_F16_BIAS:              return launch<EPI_F16_BIAS>(bf16, ta, tb, tout, tres, taux, a, grid, stream);
    case EPI_F16_BIAS_QGELU:        return launch<EPI_F16_BIAS_QGELU>(bf16, ta, tb, tout, tres, taux, a, grid, stream);
    case EPI_F16_LN_BIAS:           return launch<EPI_F16_LN_BIAS>(bf16, ta, tb, tout, tres, taux, a, grid, stream);
    case EPI_F16_LN_BIAS_QGELU:     return launch<EPI_F16_LN_BIAS_QGELU>(bf16, ta, tb, tout, tres, taux, a, grid, stream);
    case EPI_F32_BIAS_RESID:
    case EPI_F32_BIAS_RESID_STATS:  return gemm_wide_resid_launch(epi, bf16, ta, tb, tout, tres, taux, a, grid, stream);
    default: set_last_error("gemm: epilogue %d has no 128 x 256 kernel", epi); return 1;
  }
}

}  // namespace pg
