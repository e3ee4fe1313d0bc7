// The one way into gemm_kernel: launch builders for linears and convs (kernel variant, params, tensor maps) and launch_gemm.
#include "gemm_launch.cuh"

namespace mg {

int gemm_linear(GemmLaunch* g, bool bf16, const LinearArgs& a) {
    const int M = a.M, N = a.N, K = a.K, epi = a.epi;
    const Level* grid = a.grid;
    const LnIO* ln = a.ln;
    // 128 x 256 tiles with the direct epilogue where the variant exists, N allows it and there are at least four such tiles per SM;
    // else 128 x 128 staged tiles.  At one or two wide tiles per SM (batch 1, 1370 rows) the wide tiles were the slower ones
    // (batch-1 p50 about 0.25 ms longer on an H100): there the staged tiles' epilogue warpgroup still overlaps a CTA's later tiles,
    // while the direct epilogue runs behind each tile's main loop.
    bool wide = WideRows::has(epi) && N % WideRows::kBN == 0;
    if (wide) {
        int sms = 0;
        MG_TRY(check_device("linear", &sms));
        wide = static_cast<long>((M + TILE_M - 1) / TILE_M) * (N / WideRows::kBN) >= 4L * sms;
    }
    const int bn = wide ? WideRows::kBN : 128;
    if (N % bn) return set_error("linear: N=%d must be a multiple of %d", N, bn);
    if ((epi == EPI_PATCH || epi == EPI_DEC) && grid == nullptr) return set_error("linear: epilogue %d needs the token grid", epi);
    GemmParams p{};
    p.M = M; p.N = N; p.ntaps = 1; p.kb_main = (K + 63) / 64; p.kb_aux = 0;
    p.num_m_tiles = (M + TILE_M - 1) / TILE_M;
    p.num_n_tiles = N / bn;
    p.out0 = a.out; p.out1 = a.out_relu; p.bias = a.bias; p.vec1 = a.v1; p.vec2 = a.v2; p.ldo = N;
    if (grid) { p.T = grid->H * grid->W; p.W = grid->W; }
    if (epi == EPI_DEC) {
        p.B = M / p.T; p.H = grid->H;
        p.Ho = grid->H; p.Wo = grid->W; p.Hop = grid->Hp; p.Wop = grid->Wp; p.su = a.su; p.sv = a.sv;
    }
    if (ln) {
        const int parts = N / (bn / 2);             // the ROWS epilogues run in column groups of BN/2 (GemmCfg::kEpiCols)
        p.stats_ld = kStatsLd;
        if (ln->x16) {
            if (parts > kStatsLd) return set_error("linear: %d statistics groups per row > %d", parts, kStatsLd);
            p.x16 = ln->x16; p.stats_out = ln->stats_out;
            if (ln->parts_out) *ln->parts_out = parts;
        }
        p.ln_rstd = ln->ln_rstd;
    }
    g->bn = bn; g->mode = MODE_GEMM; g->amode = AMODE_ROWS; g->epi = epi; g->df = -1; g->bf16 = bf16; g->p = p;
    MG_TRY(make_map_2d(&g->a, a.A, K, M, K, TILE_M));
    MG_TRY(make_map_2d(&g->b, a.W, K, N, K, bn));
    g->aux = g->o0 = g->o1 = g->a;
    if (wide) MG_TRY(make_map_2d(&g->o0, a.out, N, M, N, 64));       // the epilogue's TMA stores: 64 columns x 64 rows
    return 0;
}

int gemm_conv(GemmLaunch* g, bool bf16, const ConvArgs& a) {
    const ConvW& cw = a.cw;
    const Level &gs = a.gs, &go = a.go;
    const int B = a.B, epi = a.epi;
    GemmParams p{};
    p.N = cw.N; p.ntaps = cw.taps; p.kb_main = cw.cin / 64; p.kb_aux = cw.caux / 64;
    p.B = B; p.H = gs.H; p.W = gs.W;
    p.tiles_x = (gs.W + TILE_PW - 1) / TILE_PW; p.tiles_y = (gs.H + TILE_PH - 1) / TILE_PH;
    p.num_m_tiles = B * p.tiles_x * p.tiles_y;
    p.out0 = a.out_raw; p.out1 = a.out_relu; p.out2 = a.out2; p.bias = cw.bias;
    p.vec1 = a.uv ? cw.wu : nullptr; p.vec2 = a.uv ? cw.wv : nullptr;
    p.skip = a.skip; p.ldo = a.out_ch;
    p.Ho = go.H; p.Wo = go.W; p.Hop = go.Hp; p.Wop = go.Wp;
    p.shuffle = a.shuffle ? 1 : 0; p.su = a.su; p.sv = a.sv;
    if (epi == EPI_HEADOUT) p.ncomp = a.ncomp;
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
    MG_TRY(make_map_nhwc(&g->a, a.src, cw.cin, gs.Wp, gs.Hp, B, mode == MODE_GEMM ? 8 : 10));
    if (cw.caux) MG_TRY(make_map_nhwc(&g->aux, a.aux, cw.caux, gs.Wp, gs.Hp, B, 8));
    else g->aux = g->a;
    MG_TRY(make_map_2d(&g->b, cw.w, cw.Ktot, cw.N, cw.Ktot, bn));
    g->o0 = g->o1 = g->a;
    if (dec_direct(mode, epi, g->df)) {        // the epilogue's TMA stores: one box = 64 channels x 16 px x 4 rows
        if (a.out_raw) MG_TRY(make_map_nhwc(&g->o0, a.out_raw, a.out_ch, go.Wp, go.Hp, B, 4));
        if (a.out_relu) MG_TRY(make_map_nhwc(&g->o1, a.out_relu, a.out_ch, go.Wp, go.Hp, B, 4));
    }
    return 0;
}

Level level_geom(int h, int w, int l) {
    Level g;
    g.H = h << l; g.W = w << l;
    g.Hp = std::max(g.H + 2, TILE_PH);
    g.Wp = std::max(g.W + 2, TILE_PW);
    return g;
}

int launch_gemm(const GemmLaunch& g, int num_sms, cudaStream_t st) {
    if (g.mode == MODE_CONV64) return launch_gemm_conv64(g, num_sms, st);
    if (g.mode == MODE_CONVH) return launch_gemm_convh(g, num_sms, st);
    return (g.amode == AMODE_ROWS) ? launch_gemm_rows(g, num_sms, st) : launch_gemm_tiles(g, num_sms, st);
}

}  // namespace mg
