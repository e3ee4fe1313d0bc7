// gemm_kernel instantiations with a row-major A operand (encoder linears, level-0 decoder input): the 128 x 256 direct-epilogue
// variants of WideRows (qkv, fc1) and the 128 x 128 staged ones.
#include "gemm_launch.cuh"

namespace mg {

int launch_gemm_rows(const GemmLaunch& g, int num_sms, cudaStream_t st) {
    if (g.bn == WideRows::kBN) return launch_gemm_wide(WideRows{}, g, num_sms, st);
#define INST(BN, EPI) \
    if (g.bn == BN && g.epi == EPI) return launch_gemm_variant<BN, MODE_GEMM, AMODE_ROWS, EPI>(g, num_sms, st);
    INST(128, EPI_STORE16)
    INST(128, EPI_GELU16)
    INST(128, EPI_RESID)
    INST(128, EPI_PATCH)
    INST(128, EPI_DEC)
#undef INST
    return set_error("no gemm_rows instantiation for bn=%d epi=%d", g.bn, g.epi);
}

}  // namespace mg
