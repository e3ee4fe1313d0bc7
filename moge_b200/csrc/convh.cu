// gemm_kernel<MODE_CONVH> instantiations: 3x3 convs with C_in >= 128, halo boxes + streamed weights (gemm_kernel.cuh).
// Only the EPI_DEC variants of ConvHDF exist; gemm_conv takes this mode for those alone.
#include "gemm_launch.cuh"

namespace mg {

int launch_gemm_convh(const GemmLaunch& g, int num_sms, cudaStream_t st) {
    return launch_gemm_dec<MODE_CONVH, AMODE_TILES>(ConvHDF{}, g, num_sms, st);
}

}  // namespace mg
