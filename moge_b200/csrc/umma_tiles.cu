// umma_kernel instantiations with a pixel-tile A operand (decoder implicit-GEMM convolutions).
// The EPI_DEC variants the MoGe-2 decoder actually uses at the 128-wide tiles are specialised at compile time
// (DF mask: raw / ReLU copies, skip, UV, pixel shuffle) -- the generic run-time-flag epilogue is a much larger hot loop.
#include "umma_launch.cuh"

namespace mg {

#define INST(BN, EPI)                                                                                       \
    if (bn == BN && epi == EPI)                                                                             \
        return bf16 ? launch_umma_inst<BN, MODE_GEMM, AMODE_TILES, EPI, true>(a, aux, b, p, num_sms, st)               \
                    : launch_umma_inst<BN, MODE_GEMM, AMODE_TILES, EPI, false>(a, aux, b, p, num_sms, st);
#define INST_DF(BN, DFV)                                                                                    \
    if (bn == BN && epi == EPI_DEC && df == (DFV))                                                          \
        return bf16 ? launch_umma_inst<BN, MODE_GEMM, AMODE_TILES, EPI_DEC, true, DFV>(a, aux, b, p, num_sms, st)      \
                    : launch_umma_inst<BN, MODE_GEMM, AMODE_TILES, EPI_DEC, false, DFV>(a, aux, b, p, num_sms, st);

int launch_umma_tiles(int bn, int epi, bool bf16, const CUtensorMap& a, const CUtensorMap& aux, const CUtensorMap& b,
                      const UmmaParams& p, int num_sms, cudaStream_t st) {
    const int df = (p.out0 ? DF_RAW : 0) | (p.out1 ? DF_RELU : 0) | (p.skip ? DF_SKIP : 0) | (p.vec1 ? DF_UV : 0) | (p.shuffle ? DF_SHUFFLE : 0);
    INST_DF(128, DF_RAW | DF_SHUFFLE)          // ConvTranspose2d k2s2
    INST_DF(128, DF_RAW)                       // 1x1 input block of a head
    INST_DF(128, DF_RELU)                      // residual block, first conv
    INST_DF(128, DF_RAW | DF_SKIP)             // residual block, second conv
    INST_DF(128, DF_RAW | DF_RELU | DF_SKIP)
    INST_DF(128, DF_RAW | DF_RELU)             // resampler conv (+ fused head input block)
    INST_DF(128, DF_RAW | DF_RELU | DF_UV)     // resampler conv of the neck (+ UV planes)
    INST(128, EPI_DEC) INST(64, EPI_DEC) INST(32, EPI_DEC)
    INST(16, EPI_HEADOUT)
    INST(32, EPI_NECKOUT)
    return set_error("no umma_tiles instantiation for bn=%d epi=%d", bn, epi);
}
#undef INST
#undef INST_DF

}  // namespace mg
