// Host-side launch helper shared by the instantiation units of umma_kernel.
#pragma once
#include "umma_kernel.cuh"
#include "host_api.h"

namespace mg {

// Persistent grid: one CTA per SM (at most one per tile).  MODE_CONV64 keeps the weights of one output-channel tile resident, so
// its grid is a multiple of num_n_tiles (every CTA then sees one fixed nt).
template <int BN, int MODE, int AMODE, int EPI, bool BF16, int DF = -1>
int launch_umma_inst(const CUtensorMap& a, const CUtensorMap& aux, const CUtensorMap& b, const UmmaParams& p, int num_sms,
                     cudaStream_t st) {
    using Cfg = UmmaCfg<BN, MODE>;
    auto kern = umma_kernel<BN, MODE, AMODE, EPI, BF16, DF>;
    MG_SET_SMEM_ONCE(kern, Cfg::kSmemBytes);
    const int tiles = p.num_m_tiles * p.num_n_tiles;
    if (tiles <= 0) return 0;
    int grid = tiles < num_sms ? tiles : num_sms;
    if (MODE == MODE_CONV64) grid = (num_sms / p.num_n_tiles) * p.num_n_tiles < tiles ? (num_sms / p.num_n_tiles) * p.num_n_tiles : tiles;
    if (grid <= 0) return set_error("umma: %d output-channel tiles exceed the %d SMs", p.num_n_tiles, num_sms);
    CUDA_TRY(launch_pdl(kern, dim3(grid), dim3(Cfg::kThreads), Cfg::kSmemBytes, st, a, aux, b, p));
    return 0;
}

int launch_umma_rows(int bn, int epi, bool bf16, const CUtensorMap& a, const CUtensorMap& aux, const CUtensorMap& b,
                     const UmmaParams& p, int num_sms, cudaStream_t st);
int launch_umma_tiles(int bn, int epi, bool bf16, const CUtensorMap& a, const CUtensorMap& aux, const CUtensorMap& b,
                      const UmmaParams& p, int num_sms, cudaStream_t st);

}  // namespace mg
