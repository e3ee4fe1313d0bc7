// umma_kernel<MODE_CONV64> instantiations + launcher: 3x3 convs with C_in = 64, resident weights (umma_kernel.cuh).
#include "umma_launch.cuh"

namespace mg {

int launch_conv64(int bn, int epi, bool bf16, const CUtensorMap& a, const CUtensorMap& aux, const CUtensorMap& w, const UmmaParams& p,
                  int num_sms, cudaStream_t st) {
    if (p.ntaps != 9 || p.kb_main != 1 || p.kb_aux > 1) return set_error("conv64: needs a 3x3 conv with C_in = 64");
    if (p.N % bn) return set_error("conv64: N=%d not a multiple of %d", p.N, bn);
    // compile-time specialisations of the EPI_DEC variants the MoGe-2 decoder uses at levels 3/4 (small hot loops);
    // anything else runs the generic run-time-flag variant.
    int df = -1;
    if (epi == EPI_DEC) df = (p.out0 ? DF_RAW : 0) | (p.out1 ? DF_RELU : 0) | (p.skip ? DF_SKIP : 0) | (p.vec1 ? DF_UV : 0) | (p.shuffle ? DF_SHUFFLE : 0);
#define INST(BN, EPI, DFV)                                                                                       \
    if (bn == BN && epi == EPI && df == (DFV))                                                                   \
        return bf16 ? launch_umma_inst<BN, MODE_CONV64, AMODE_TILES, EPI, true, DFV>(a, aux, w, p, num_sms, st)  \
                    : launch_umma_inst<BN, MODE_CONV64, AMODE_TILES, EPI, false, DFV>(a, aux, w, p, num_sms, st);
    INST(64, EPI_DEC, DF_RELU)
    INST(64, EPI_DEC, DF_RAW | DF_SKIP)
    INST(64, EPI_DEC, DF_RAW | DF_RELU | DF_SKIP)
    INST(64, EPI_DEC, DF_RAW | DF_RELU)
    INST(64, EPI_DEC, DF_RAW | DF_RELU | DF_UV)
    INST(64, EPI_DEC, DF_RAW | DF_UV | DF_SHUFFLE)
    df = -1;
    INST(64, EPI_DEC, -1)
    INST(16, EPI_HEADOUT, -1)
    INST(32, EPI_NECKOUT, -1)
#undef INST
    return set_error("no conv64 instantiation for bn=%d epi=%d", bn, epi);
}

}  // namespace mg
