// gemm_kernel instantiations with a pixel-tile A operand and the per-tap GEMM main loop (decoder implicit-GEMM convolutions).
// The EPI_DEC variants the MoGe-2 decoder actually uses at the 128-wide tiles are specialised at compile time (TilesDF) -- the
// generic run-time-flag epilogue is a much larger hot loop.
#include "gemm_launch.cuh"

namespace mg {

int launch_gemm_tiles(const GemmLaunch& g, int num_sms, cudaStream_t st) {
    if (g.df >= 0) return launch_gemm_dec<MODE_GEMM, AMODE_TILES>(TilesDF{}, g, num_sms, st);
#define INST(BN, EPI) \
    if (g.bn == BN && g.epi == EPI) return launch_gemm_variant<BN, MODE_GEMM, AMODE_TILES, EPI>(g, num_sms, st);
    INST(128, EPI_DEC) INST(64, EPI_DEC) INST(32, EPI_DEC)
    INST(16, EPI_HEADOUT)
    INST(32, EPI_NECKOUT)
#undef INST
    return set_error("no gemm_tiles instantiation for bn=%d epi=%d", g.bn, g.epi);
}

}  // namespace mg
