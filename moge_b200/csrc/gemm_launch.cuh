// Host-side launch helpers shared by the instantiation units of gemm_kernel (gemm_rows.cu, gemm_tiles.cu, conv64.cu, convh.cu).
#pragma once
#include "gemm_kernel.cuh"
#include "host_api.h"

namespace mg {

// The EPI_DEC variants a main-loop mode specialises at compile time (DF mask), all at tile width BN; every other EPI_DEC launch of
// the mode runs the run-time-flag variant (DF = -1).  The mode's instantiation unit instantiates exactly this list and gemm_conv
// selects from it, so the two cannot drift apart.
template <int BN, int... M> struct DecFlagList {
    static constexpr bool has(int bn, int df) { return bn == BN && ((df == M) || ...); }
};
using TilesDF = DecFlagList<128,                     // MODE_GEMM with pixel tiles (per-tap GEMM)
                            DF_RAW | DF_SHUFFLE,     // ConvTranspose2d k2s2
                            DF_RAW,                  // 1x1 input block of a head
                            DF_RELU,                 // residual block, first conv
                            DF_RAW | DF_SKIP,        // residual block, second conv
                            DF_RAW | DF_RELU | DF_SKIP,
                            DF_RAW | DF_RELU,        // resampler conv (+ fused head input block)
                            DF_RAW | DF_RELU | DF_UV>;   // resampler conv of the neck (+ UV planes)
using Conv64DF = DecFlagList<64, DF_RELU, DF_RAW | DF_SKIP, DF_RAW | DF_RELU | DF_SKIP, DF_RAW | DF_RELU, DF_RAW | DF_RELU | DF_UV,
                             DF_RAW | DF_UV | DF_SHUFFLE>;
using ConvHDF = DecFlagList<128, DF_RELU, DF_RAW | DF_SKIP, DF_RAW | DF_RELU | DF_SKIP, DF_RAW | DF_RELU, DF_RAW | DF_RELU | DF_UV>;

// Persistent grid: one CTA per SM (at most one per tile).  MODE_CONV64 keeps the weights of one output-channel tile resident, so
// its grid is a multiple of num_n_tiles (every CTA then sees one fixed nt).
template <int BN, int MODE, int AMODE, int EPI, bool BF16, int DF>
int launch_gemm_inst(const GemmLaunch& g, int num_sms, cudaStream_t st) {
    using Cfg = GemmCfg<BN, MODE, gemm_direct(BN, MODE, AMODE, EPI, DF)>;
    const GemmParams& p = g.p;
    auto kern = gemm_kernel<BN, MODE, AMODE, EPI, BF16, DF>;
    MG_SET_SMEM_ONCE(kern, Cfg::kSmemBytes);
    const int tiles = p.num_m_tiles * p.num_n_tiles;
    if (tiles <= 0) return 0;
    int grid = tiles < num_sms ? tiles : num_sms;
    if (MODE == MODE_CONV64) grid = (num_sms / p.num_n_tiles) * p.num_n_tiles < tiles ? (num_sms / p.num_n_tiles) * p.num_n_tiles : tiles;
    if (grid <= 0) return set_error("gemm: %d output-channel tiles exceed the %d SMs", p.num_n_tiles, num_sms);
    CUDA_TRY(launch_pdl(kern, dim3(grid), dim3(Cfg::kThreads), Cfg::kSmemBytes, st, g.a, g.aux, g.b, g.o0, g.o1, p));
    return 0;
}

template <int BN, int MODE, int AMODE, int EPI, int DF = -1>
int launch_gemm_variant(const GemmLaunch& g, int num_sms, cudaStream_t st) {
    return g.bf16 ? launch_gemm_inst<BN, MODE, AMODE, EPI, true, DF>(g, num_sms, st)
                  : launch_gemm_inst<BN, MODE, AMODE, EPI, false, DF>(g, num_sms, st);
}

// The WideRows variant of epilogue g.epi (instantiates every epilogue of the list).
template <int BN, int... E>
int launch_gemm_wide(RowEpiList<BN, E...>, const GemmLaunch& g, int num_sms, cudaStream_t st) {
    int rc = 0;
    const bool found = ((g.bn == BN && g.epi == E && ((rc = launch_gemm_variant<BN, MODE_GEMM, AMODE_ROWS, E>(g, num_sms, st)), true)) || ...);
    return found ? rc : set_error("gemm: no %d-wide row variant for epi=%d", BN, g.epi);
}

// The specialised EPI_DEC variant g.df of a mode's list (instantiates every mask of the list).
template <int MODE, int AMODE, int BN, int... M>
int launch_gemm_dec(DecFlagList<BN, M...>, const GemmLaunch& g, int num_sms, cudaStream_t st) {
    int rc = 0;
    const bool found = ((g.bn == BN && g.df == M && ((rc = launch_gemm_variant<BN, MODE, AMODE, EPI_DEC, M>(g, num_sms, st)), true)) || ...);
    return found ? rc : set_error("gemm: no mode-%d variant for bn=%d df=%d", MODE, g.bn, g.df);
}

// one per instantiation unit
int launch_gemm_rows(const GemmLaunch& g, int num_sms, cudaStream_t st);
int launch_gemm_tiles(const GemmLaunch& g, int num_sms, cudaStream_t st);
int launch_gemm_conv64(const GemmLaunch& g, int num_sms, cudaStream_t st);
int launch_gemm_convh(const GemmLaunch& g, int num_sms, cudaStream_t st);

}  // namespace mg
