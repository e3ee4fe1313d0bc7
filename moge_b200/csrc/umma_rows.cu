// umma_kernel instantiations with a row-major A operand (encoder linears, level-0 decoder input).
#include "umma_launch.cuh"

namespace mg {

#define INST(BN, EPI)                                                                                       \
    if (bn == BN && epi == EPI)                                                                             \
        return bf16 ? launch_umma_inst<BN, MODE_GEMM, AMODE_ROWS, EPI, true>(a, aux, b, p, num_sms, st)                \
                    : launch_umma_inst<BN, MODE_GEMM, AMODE_ROWS, EPI, false>(a, aux, b, p, num_sms, st);

int launch_umma_rows(int bn, int epi, bool bf16, const CUtensorMap& a, const CUtensorMap& aux, const CUtensorMap& b,
                     const UmmaParams& p, int num_sms, cudaStream_t st) {
    INST(128, EPI_STORE16)
    INST(128, EPI_GELU16)
    INST(128, EPI_RESID)
    INST(128, EPI_PATCH)
    INST(128, EPI_DEC)
    return set_error("no umma_rows instantiation for bn=%d epi=%d", bn, epi);
}
#undef INST

int launch_umma(int bn, int amode, int epi, bool bf16, const CUtensorMap& a, const CUtensorMap& aux, const CUtensorMap& b,
                const UmmaParams& p, int num_sms, cudaStream_t st) {
    if (p.N % bn) return set_error("umma: N=%d not a multiple of the tile width %d", p.N, bn);
    if (amode == AMODE_ROWS) return launch_umma_rows(bn, epi, bf16, a, aux, b, p, num_sms, st);
    return launch_umma_tiles(bn, epi, bf16, a, aux, b, p, num_sms, st);
}

}  // namespace mg
