// umma_kernel<MODE_CONVH> instantiations + launcher: 3x3 convs with C_in >= 128, halo boxes + streamed weights (umma_kernel.cuh).
#include "umma_launch.cuh"

namespace mg {

bool convh_supports(int bn, const UmmaParams& p) {
    if (p.ntaps != 9 || p.kb_main < 1 || bn != 128 || p.N % bn) return false;      // 256-wide stages do not fit beside the tile
    const int df = (p.out0 ? DF_RAW : 0) | (p.out1 ? DF_RELU : 0) | (p.skip ? DF_SKIP : 0) | (p.vec1 ? DF_UV : 0) | (p.shuffle ? DF_SHUFFLE : 0);
    return df == DF_RELU || df == (DF_RAW | DF_SKIP) || df == (DF_RAW | DF_RELU | DF_SKIP) || df == (DF_RAW | DF_RELU) ||
           df == (DF_RAW | DF_RELU | DF_UV);
}

int launch_convh(int bn, bool bf16, const CUtensorMap& a, const CUtensorMap& aux, const CUtensorMap& w, const UmmaParams& p,
                 int num_sms, cudaStream_t st) {
    if (!convh_supports(bn, p)) return set_error("convh: unsupported configuration (bn=%d taps=%d)", bn, p.ntaps);
    const int df = (p.out0 ? DF_RAW : 0) | (p.out1 ? DF_RELU : 0) | (p.skip ? DF_SKIP : 0) | (p.vec1 ? DF_UV : 0) | (p.shuffle ? DF_SHUFFLE : 0);
#define INST(BN, DFV)                                                                                            \
    if (bn == BN && df == (DFV))                                                                                 \
        return bf16 ? launch_umma_inst<BN, MODE_CONVH, AMODE_TILES, EPI_DEC, true, DFV>(a, aux, w, p, num_sms, st)        \
                    : launch_umma_inst<BN, MODE_CONVH, AMODE_TILES, EPI_DEC, false, DFV>(a, aux, w, p, num_sms, st);
    INST(128, DF_RELU)
    INST(128, DF_RAW | DF_SKIP)
    INST(128, DF_RAW | DF_RELU | DF_SKIP)
    INST(128, DF_RAW | DF_RELU)
    INST(128, DF_RAW | DF_RELU | DF_UV)
#undef INST
    return set_error("no convh instantiation for bn=%d df=%d", bn, df);
}

}  // namespace mg
