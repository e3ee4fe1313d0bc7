// The one way into gemm_kernel: launch builders for linears and convs (kernel variant, params, tensor maps) and launch_gemm.
#include "gemm_launch.cuh"

namespace mg {

int gemm_linear(GemmLaunch* g, bool bf16, const void* A, int M, int K, const void* W, int ldw, int N, int epi, void* out, int ldo,
                const float* bias, const float* v1, const LnIO* ln, const Level* grid, void* out_relu, const float* v2, float su, float sv) {
    constexpr int bn = 128;
    if (N % bn) return set_error("linear: N=%d must be a multiple of %d", N, bn);
    if ((epi == EPI_PATCH || epi == EPI_DEC) && grid == nullptr) return set_error("linear: epilogue %d needs the token grid", epi);
    GemmParams p{};
    p.M = M; p.N = N; p.ntaps = 1; p.kb_main = (K + 63) / 64; p.kb_aux = 0;
    p.num_m_tiles = (M + TILE_M - 1) / TILE_M;
    p.num_n_tiles = N / bn;
    p.out0 = out; p.out1 = out_relu; p.bias = bias; p.vec1 = v1; p.vec2 = v2; p.ldo = ldo;
    if (grid) { p.T = grid->H * grid->W; p.W = grid->W; }
    if (epi == EPI_DEC) {
        p.B = M / p.T; p.H = grid->H;
        p.Ho = grid->H; p.Wo = grid->W; p.Hop = grid->Hp; p.Wop = grid->Wp; p.su = su; p.sv = sv;
    }
    if (ln) {
        const int parts = N / (bn / 2);             // every ROWS kernel has 8 epilogue warps: column groups of BN/2
        p.stats_ld = kStatsLd;
        if (ln->x16) {
            if (parts > kStatsLd) return set_error("linear: %d statistics groups per row > %d", parts, kStatsLd);
            p.x16 = ln->x16; p.stats_out = ln->stats_out;
            if (ln->parts_out) *ln->parts_out = parts;
        }
        p.ln_rstd = ln->ln_rstd;
    }
    g->bn = bn; g->mode = MODE_GEMM; g->amode = AMODE_ROWS; g->epi = epi; g->df = -1; g->bf16 = bf16; g->p = p;
    MG_TRY(make_map_2d(&g->a, A, K, M, K, TILE_M));
    MG_TRY(make_map_2d(&g->b, W, K, N, ldw, bn));
    g->aux = g->a;
    return 0;
}

int gemm_conv(GemmLaunch* g, bool bf16, const ConvW& cw, const void* src, const void* aux, const Level& gs, int B, int epi,
              void* out_raw, void* out_relu, const void* skip, const Level& go, int out_ch, bool shuffle, bool uv, float su, float sv,
              int ncomp, void* out2) {
    GemmParams p{};
    p.N = cw.N; p.ntaps = cw.taps; p.kb_main = cw.cin / 64; p.kb_aux = cw.caux / 64;
    p.B = B; p.H = gs.H; p.W = gs.W;
    p.tiles_x = (gs.W + TILE_PW - 1) / TILE_PW; p.tiles_y = (gs.H + TILE_PH - 1) / TILE_PH;
    p.num_m_tiles = B * p.tiles_x * p.tiles_y;
    p.out0 = out_raw; p.out1 = out_relu; p.out2 = out2; p.bias = cw.bias;
    p.vec1 = uv ? cw.wu : nullptr; p.vec2 = uv ? cw.wv : nullptr;
    p.skip = skip; p.ldo = out_ch;
    p.Ho = go.H; p.Wo = go.W; p.Hop = go.Hp; p.Wop = go.Wp;
    p.shuffle = shuffle ? 1 : 0; p.su = su; p.sv = sv;
    if (epi == EPI_HEADOUT) p.ncomp = ncomp;
    // tile width: fixed for the folded head / neck outputs, else the widest that divides N
    int bn = (epi == EPI_HEADOUT) ? 16 : (epi == EPI_NECKOUT) ? 32 : (cw.N % 128 == 0) ? 128 : (cw.N % 64 == 0) ? 64 : (cw.N % 32 == 0) ? 32 : 0;
    if (!bn) return set_error("conv: N=%d has no tile width", cw.N);
    const int df = (epi == EPI_DEC) ? dec_flags(p) : -1;
    // main loop: the halo modes read 3x3 taps from 10-row boxes (8 output rows + 2), so the padded map must be that tall
    const bool halo = cw.taps == 9 && gs.Hp >= 10;
    int mode = MODE_GEMM;
    if (halo && cw.cin == 64 && (cw.caux == 0 || cw.caux == 64) &&
        ((epi == EPI_HEADOUT && cw.N == 16) || (epi == EPI_NECKOUT && cw.N == 32) || (epi == EPI_DEC && cw.N % 64 == 0))) {
        mode = MODE_CONV64;      // resident weights + one halo box per horizontal tap
        if (epi == EPI_DEC) bn = 64;
    } else if (halo && epi == EPI_DEC && cw.cin >= 128 && cw.cin % 64 == 0 && cw.caux % 64 == 0 && ConvHDF::has(bn, df)) {
        mode = MODE_CONVH;       // halo boxes + streamed weights
    }
    p.num_n_tiles = cw.N / bn;
    const bool specialised = (mode == MODE_CONV64) ? Conv64DF::has(bn, df) : (mode == MODE_CONVH) ? ConvHDF::has(bn, df) : TilesDF::has(bn, df);
    g->bn = bn; g->mode = mode; g->amode = AMODE_TILES; g->epi = epi; g->df = specialised ? df : -1; g->bf16 = bf16; g->p = p;
    MG_TRY(make_map_nhwc(&g->a, src, cw.cin, gs.Wp, gs.Hp, B, mode == MODE_GEMM ? 8 : 10));
    if (cw.caux) MG_TRY(make_map_nhwc(&g->aux, aux, cw.caux, gs.Wp, gs.Hp, B, 8));
    else g->aux = g->a;
    MG_TRY(make_map_2d(&g->b, cw.w, cw.Ktot, cw.N, cw.Ktot, bn));
    return 0;
}

int launch_gemm(const GemmLaunch& g, int num_sms, cudaStream_t st) {
    if (g.mode == MODE_CONV64) return launch_gemm_conv64(g, num_sms, st);
    if (g.mode == MODE_CONVH) return launch_gemm_convh(g, num_sms, st);
    return (g.amode == AMODE_ROWS) ? launch_gemm_rows(g, num_sms, st) : launch_gemm_tiles(g, num_sms, st);
}

}  // namespace mg
