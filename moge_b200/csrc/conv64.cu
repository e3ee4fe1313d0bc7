// gemm_kernel<MODE_CONV64> instantiations: 3x3 convs with C_in = 64, resident weights (gemm_kernel.cuh).
#include "gemm_launch.cuh"

namespace mg {

int launch_gemm_conv64(const GemmLaunch& g, int num_sms, cudaStream_t st) {
    // compile-time specialisations of the EPI_DEC variants the MoGe-2 decoder uses at levels 3/4 (Conv64DF, small hot loops)
    if (g.df >= 0) return launch_gemm_dec<MODE_CONV64, AMODE_TILES>(Conv64DF{}, g, num_sms, st);
#define INST(BN, EPI) \
    if (g.bn == BN && g.epi == EPI) return launch_gemm_variant<BN, MODE_CONV64, AMODE_TILES, EPI>(g, num_sms, st);
    INST(64, EPI_DEC)
    INST(16, EPI_HEADOUT)
    INST(32, EPI_NECKOUT)
#undef INST
    return set_error("no conv64 instantiation for bn=%d epi=%d", g.bn, g.epi);
}

}  // namespace mg
