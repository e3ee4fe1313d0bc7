// Operator-level entry points of libmoge_b200.so (include/moge_b200.h): single kernels of the engine's forward, each run the way
// the engine runs it, for tests and inspection.
#include "moge_b200.h"
#include "gemm_kernel.cuh"
#include "host_api.h"

namespace mg {

static_assert(kStatsLd == MOGE_STATS_LD, "the statistics pitch of the C ABI is the engine's");

// Device scratch of one operator call.  alloc() reports the first failed cudaMalloc through set_error; the destructor waits for
// the stream, whose launches read the buffers, then frees them all.
struct Scratch {
    const char* op;
    cudaStream_t st;
    std::vector<void*> bufs;
    ~Scratch() { cudaStreamSynchronize(st); for (void* p : bufs) cudaFree(p); }
    template <typename T>
    int alloc(T** p, size_t bytes) {
        if (cudaMalloc(reinterpret_cast<void**>(p), bytes) != cudaSuccess)
            return set_error("%s: cudaMalloc of %zu bytes failed", op, bytes);
        bufs.push_back(*p);
        return 0;
    }
};

}  // namespace mg

using namespace mg;

extern "C" {

int moge_op_linear(const void* x, const void* w, const float* bias, const float* gamma, void* out, int M, int N, int K, int epi,
                   int dtype, void* stream) {
    if (K % 8) return set_error("op_linear: K must be a multiple of 8");
    if (epi < 0 || epi > 2) return set_error("op_linear: epi must be 0..2");
    LinearArgs a; a.A = x; a.M = M; a.K = K; a.W = w; a.N = N; a.epi = epi; a.out = out; a.bias = bias; a.v1 = gamma;
    GemmLaunch g;
    MG_TRY(gemm_linear(&g, dtype == MOGE_BF16, a));
    int sms; MG_TRY(check_device("op_linear", &sms));
    return launch_gemm(g, sms, static_cast<cudaStream_t>(stream));
}

int moge_op_attention(const void* qkv, void* out, int B, int N, int D, int heads, int dtype, void* stream) {
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    if (B <= 0 || N <= 0) return set_error("op_attention: bad shape B=%d N=%d", B, N);
    CUtensorMap mq;
    MG_TRY(make_map_2d(&mq, qkv, 3 * static_cast<uint64_t>(D), static_cast<uint64_t>(B) * N, 3 * static_cast<uint64_t>(D), 128));
    int sms; MG_TRY(check_device("op_attention", &sms));
    AttnWork work;
    Scratch s{"op_attention", st};
    MG_TRY(upload_attention_work(std::vector<int>(B, N), heads, sms, [&s](void** p, size_t bytes) { return s.alloc(p, bytes); }, st, &work));
    return launch_attention(mq, out, work.items_dev, work.ranges_dev, static_cast<int>(work.ranges.size()), D, heads, dtype == MOGE_BF16, st);
}

int moge_attention_work_list(const int* n_tokens, int n_images, int heads, int n_ctas, int* items, int items_cap, int* ranges, int* n_items,
                             int* n_ranges) {
    // host only: the work list the engine uploads for the persistent attention kernel (plan time), for inspection and tests
    if (n_images < 0 || heads <= 0 || n_ctas <= 0 || !n_tokens) return set_error("attention_work_list: bad arguments");
    for (int i = 0; i < n_images; ++i)
        if (n_tokens[i] <= 0) return set_error("attention_work_list: image %d has %d tokens", i, n_tokens[i]);
    std::vector<AttnItem> it;
    std::vector<int2> rg;
    attention_work_list(n_tokens, n_images, heads, n_ctas, &it, &rg);
    if (n_items) *n_items = static_cast<int>(it.size());
    if (n_ranges) *n_ranges = static_cast<int>(rg.size());
    if (items) {
        if (items_cap < static_cast<int>(it.size())) return set_error("attention_work_list: items_cap %d < %zu", items_cap, it.size());
        for (size_t i = 0; i < it.size(); ++i) { items[4 * i] = it[i].row0; items[4 * i + 1] = it[i].n; items[4 * i + 2] = it[i].q0; items[4 * i + 3] = it[i].head; }
    }
    if (ranges) for (size_t i = 0; i < rg.size(); ++i) { ranges[2 * i] = rg[i].x; ranges[2 * i + 1] = rg[i].y; }
    return 0;
}

int moge_op_linear_ln_rows(const void* x16, const float* rstd, const float* ln_gamma, const float* ln_beta, const float* w, const float* bias,
                           void* out, int M, int N, int K, int epi, int dtype, void* stream) {
    // the engine's LayerNorm consumer (qkv, fc1): the load-time weight fold, then one GEMM on the rounded rows scaled by rstd[row]
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const bool bf16 = dtype == MOGE_BF16;
    if (!x16 || !rstd || !ln_gamma || !ln_beta || !w || !out) return set_error("null argument");
    if (M <= 0 || K % 64) return set_error("op_linear_ln_rows: M > 0 and K a multiple of 64 required");
    if (epi != EPI_STORE16 && epi != EPI_GELU16) return set_error("op_linear_ln_rows: epi must be 0 (store) or 1 (GELU)");
    Scratch s{"op_linear_ln_rows", st};
    void* w16; float* b2;
    MG_TRY(s.alloc(&w16, static_cast<size_t>(N) * K * 2));
    MG_TRY(s.alloc(&b2, static_cast<size_t>(N) * 4));
    LnIO cons; cons.ln_rstd = rstd;
    LinearArgs a; a.A = x16; a.M = M; a.K = K; a.W = w16; a.N = N; a.epi = epi; a.out = out; a.bias = b2; a.ln = &cons;
    GemmLaunch g;
    MG_TRY(gemm_linear(&g, bf16, a));
    MG_TRY(launch_ln_fold(w, ln_gamma, ln_beta, bias, N, K, K, w16, b2, bf16, st));
    int sms; MG_TRY(check_device("op_linear_ln_rows", &sms));
    return launch_gemm(g, sms, st);
}

int moge_op_linear_ln(const float* x, const float* ln_gamma, const float* ln_beta, const float* w, const float* bias, void* out, int M,
                      int N, int K, int epi, int dtype, void* stream) {
    // out = epi(LayerNorm(x) W^T + bias) the way the engine computes it: rounded rows + row statistics, folded weights, one GEMM
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const bool bf16 = dtype == MOGE_BF16;
    if (M <= 0 || K % 64) return set_error("op_linear_ln: M > 0 and K a multiple of 64 required");
    if (epi != EPI_STORE16 && epi != EPI_GELU16) return set_error("op_linear_ln: epi must be 0 (store) or 1 (GELU)");
    Scratch s{"op_linear_ln", st};
    void* x16; float2* stats; float* rstd;
    MG_TRY(s.alloc(&x16, static_cast<size_t>(M) * K * 2));
    MG_TRY(s.alloc(&stats, static_cast<size_t>(M) * kStatsLd * 8));
    MG_TRY(s.alloc(&rstd, static_cast<size_t>(M) * 4));
    MG_TRY(launch_ln_prepare(x, M, K, K, x16, K, stats, kStatsLd, 1, bf16, st));
    MG_TRY(launch_ln_rstd(stats, kStatsLd, 1, M, K, rstd, st));
    return moge_op_linear_ln_rows(x16, rstd, ln_gamma, ln_beta, w, bias, out, M, N, K, epi, dtype, stream);
}

int moge_op_linear_resid_ln(const void* a, const void* w, const float* bias, const float* gamma, float* x, void* x16, float* stats, int* parts,
                            int M, int N, int K, int dtype, void* stream) {
    // the engine's proj / fc2: x += gamma * (a W^T + bias), with the LayerNorm producer side (x16 and per-group partial sums)
    if (!a || !w || !bias || !gamma || !x || !x16 || !stats || !parts) return set_error("null argument");
    if (M <= 0 || K % 8) return set_error("op_linear_resid_ln: M > 0 and K a multiple of 8 required");
    LnIO prod; prod.x16 = x16; prod.stats_out = reinterpret_cast<float2*>(stats); prod.parts_out = parts;
    LinearArgs la; la.A = a; la.M = M; la.K = K; la.W = w; la.N = N; la.epi = EPI_RESID; la.out = x; la.bias = bias; la.v1 = gamma; la.ln = &prod;
    GemmLaunch g;
    MG_TRY(gemm_linear(&g, dtype == MOGE_BF16, la));
    int sms; MG_TRY(check_device("op_linear_resid_ln", &sms));
    return launch_gemm(g, sms, static_cast<cudaStream_t>(stream));
}

int moge_op_ln_rstd(const float* stats, int parts, int rows, int D, float* rstd, void* stream) {
    if (!stats || !rstd) return set_error("null argument");
    if (parts < 1 || parts > kStatsLd || rows < 0 || D <= 0) return set_error("op_ln_rstd: bad arguments parts=%d rows=%d D=%d", parts, rows, D);
    return launch_ln_rstd(reinterpret_cast<const float2*>(stats), kStatsLd, parts, rows, D, rstd, static_cast<cudaStream_t>(stream));
}

int moge_op_preprocess(const void* image, int image_dtype, int B, int H, int W, int h, int w, void* patches, int dtype, void* stream) {
    if (!image || !patches) return set_error("null argument");
    if (image_dtype != MOGE_F32 && image_dtype != MOGE_F16 && image_dtype != MOGE_BF16) return set_error("op_preprocess: unsupported image dtype %d", image_dtype);
    if (B <= 0 || H <= 0 || W <= 0 || h <= 0 || w <= 0) return set_error("op_preprocess: bad shape");
    return launch_preprocess(image, image_dtype, B, H, W, h, w, patches, 592, dtype == MOGE_BF16, static_cast<cudaStream_t>(stream));
}

int moge_op_pos_table(const float* pos_embed, const float* cls_token, const float* patch_bias, int D, int h, int w, float* table, float* cls_row,
                      void* stream) {
    if (!pos_embed || !cls_token || !patch_bias || !table || !cls_row) return set_error("null argument");
    if (D <= 0 || h <= 0 || w <= 0) return set_error("op_pos_table: bad shape");
    return launch_pos_table(pos_embed, cls_token, patch_bias, D, h, w, table, cls_row, static_cast<cudaStream_t>(stream));
}

int moge_op_patch_embed(const void* image, int image_dtype, int B, int H, int W, int h, int w, const float* w_patch, const float* b_patch,
                        const float* pos_embed, const float* cls_token, int D, float* x, void* x16, float* stats, int* parts, int dtype,
                        void* stream) {
    // the engine's front end of one group (get_plan, build_plan): pos table, preprocess, the EPI_PATCH GEMM with the LayerNorm
    // producer side, the cls rows, and their rounded copies and statistics
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const bool bf16 = dtype == MOGE_BF16;
    if (!image || !w_patch || !b_patch || !pos_embed || !cls_token || !x || !x16 || !stats || !parts) return set_error("null argument");
    if (B <= 0 || H <= 0 || W <= 0 || h <= 0 || w <= 0 || D <= 0) return set_error("op_patch_embed: bad shape");
    const int T = h * w, N = T + 1;
    Scratch s{"op_patch_embed", st};
    float *table, *cls_row; void *patches, *w16;
    MG_TRY(s.alloc(&table, static_cast<size_t>(T) * D * 4));
    MG_TRY(s.alloc(&cls_row, static_cast<size_t>(D) * 4));
    MG_TRY(s.alloc(&patches, static_cast<size_t>(B) * T * 592 * 2));
    MG_TRY(s.alloc(&w16, static_cast<size_t>(D) * 592 * 2));
    float2* st2 = reinterpret_cast<float2*>(stats);
    LnIO prod; prod.x16 = x16; prod.stats_out = st2; prod.parts_out = parts;
    const Level grid = level_geom(h, w, 0);
    LinearArgs a; a.A = patches; a.M = B * T; a.K = 592; a.W = w16; a.N = D; a.epi = EPI_PATCH;
    a.out = x; a.v1 = table; a.ln = &prod; a.grid = &grid;
    GemmLaunch g;
    MG_TRY(gemm_linear(&g, bf16, a));
    int sms; MG_TRY(check_device("op_patch_embed", &sms));
    MG_TRY(launch_pos_table(pos_embed, cls_token, b_patch, D, h, w, table, cls_row, st));
    MG_TRY(launch_preprocess(image, image_dtype, B, H, W, h, w, patches, 592, bf16, st));
    MG_TRY(launch_cast_2d(w_patch, MOGE_F32, w16, bf16, D, 588, 588, 592, st));
    MG_TRY(launch_gemm(g, sms, st));
    MG_TRY(launch_init_cls(x, cls_row, B, N, D, st));
    return launch_ln_prepare(x, B, static_cast<long>(N) * D, D, x16, static_cast<long>(N) * D, st2, static_cast<long>(N) * kStatsLd, *parts, bf16, st);
}

int moge_op_layernorm(const float* x, const float* gamma, const float* beta, void* out, int rows, int D, int dtype, void* stream) {
    return launch_layernorm(x, gamma, beta, out, rows, D, D, 0, 0, 1, nullptr, dtype == MOGE_BF16, static_cast<cudaStream_t>(stream));
}

int moge_op_layernorm_taps(const float* x, const float* gamma, const float* beta, void* out, float* cls_out, int B, int N, int D, int ld_out,
                           int col_off, int dtype, void* stream) {
    // the engine's tap LayerNorm: patch token (b, t) -> out[(b*(N-1) + t) * ld_out + col_off ..], cls rows fp32 to cls_out (or skipped)
    if (!x || !gamma || !beta || !out) return set_error("null argument");
    if (B <= 0 || N < 2 || col_off < 0 || col_off + D > ld_out) return set_error("op_layernorm_taps: bad shape");
    return launch_layernorm(x, gamma, beta, out, B * N, D, ld_out, col_off, 1, N, cls_out, dtype == MOGE_BF16, static_cast<cudaStream_t>(stream));
}

int moge_op_conv(const void* x, const float* w, const float* bias, const void* skip, void* out_raw, void* out_relu, int B, int H, int W,
                 int Cin, int Cout, int taps, int shuffle, int dtype, void* stream) {
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const bool bf16 = dtype == MOGE_BF16;
    if (Cin % 64) return set_error("op_conv: Cin must be a multiple of 64");
    if (taps != 1 && taps != 9) return set_error("op_conv: taps must be 1 or 9");
    if (shuffle && taps != 1) return set_error("op_conv: shuffle requires taps=1");
    ConvArgs a;
    ConvW& cw = a.cw; cw.N = shuffle ? 4 * Cout : Cout; cw.Ktot = taps * Cin; cw.cin = Cin; cw.taps = taps; cw.bias = const_cast<float*>(bias);
    Scratch s{"op_conv", st};
    MG_TRY(s.alloc(&cw.w, static_cast<size_t>(cw.N) * cw.Ktot * 2));
    MG_TRY(shuffle ? launch_pack_convT(w, cw.w, bf16, Cin, Cout, st) : launch_pack_conv(w, cw.w, bf16, Cout, Cin, taps, cw.Ktot, 0, st));
    a.src = x; a.gs = level_geom(H, W, 0); a.go = level_geom(H, W, shuffle ? 1 : 0); a.B = B; a.out_ch = Cout; a.epi = EPI_DEC;
    a.out_raw = out_raw; a.out_relu = out_relu; a.skip = skip; a.shuffle = shuffle != 0;
    GemmLaunch g;
    MG_TRY(gemm_conv(&g, bf16, a));
    int sms; MG_TRY(check_device("op_conv", &sms));
    return launch_gemm(g, sms, st);
}

int moge_op_resize_bicubic_aa(const void* x, int dtype, int B, int C, int H, int W, int Ho, int Wo, float* out, void* stream) {
    if (!x || !out) return set_error("null argument");
    if (dtype != MOGE_F32 && dtype != MOGE_F16 && dtype != MOGE_BF16) return set_error("op_resize_bicubic_aa: unsupported dtype %d", dtype);
    if (B <= 0 || C <= 0 || H <= 0 || W <= 0 || Ho <= 0 || Wo <= 0) return set_error("op_resize_bicubic_aa: bad shape");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    Scratch s{"op_resize_bicubic_aa", st};
    float* tmp;
    MG_TRY(s.alloc(&tmp, static_cast<size_t>(B) * C * H * Wo * 4));
    return launch_resize_bicubic_aa(x, dtype, B, C, H, W, Ho, Wo, tmp, out, st);
}

int moge_op_groupnorm_relu(const void* x, void* out, const float* gamma, const float* beta, int B, int H, int W, int C, int G, int dtype,
                           void* stream) {
    if (!x || !out || !gamma || !beta) return set_error("null argument");
    if (B <= 0 || H <= 0 || W <= 0 || C <= 0 || C % 8) return set_error("op_groupnorm_relu: bad shape");
    if (G <= 0) return set_error("op_groupnorm_relu: G=%d / cudaMalloc failed", G);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const bool bf16 = dtype == MOGE_BF16;
    const Level g = level_geom(H, W, 0);
    Scratch s{"op_groupnorm_relu", st};
    double2* part;
    float2* stats;
    MG_TRY(s.alloc(&part, static_cast<size_t>(B) * gn_tiles(H, W, C) * G * 16));
    MG_TRY(s.alloc(&stats, static_cast<size_t>(B) * G * 8));
    MG_TRY(launch_gn_stats(x, g, B, C, G, part, stats, bf16, st));
    return launch_gn_relu(x, out, g, B, C, G, stats, gamma, beta, bf16, st);
}

int moge_op_conv_transpose_uv(const void* x, const float* w, const float* bias, void* out, int B, int H, int W, int Cin, int Cout, float su, float sv,
                     int dtype, void* stream) {
    // the engine's MoGe-1 upsampling ConvTranspose: moge_op_conv's pixel-shuffle GEMM over the feature rows of w, then the
    // input-grid UV term of its last two rows
    if (!x || !w || !bias || !out) return set_error("null argument");
    if (B <= 0 || H <= 0 || W <= 0) return set_error("op_conv_transpose_uv: bad shape");
    if (Cin % 64 || Cout <= 0 || Cout % 32) return set_error("op_conv_transpose_uv: Cin %% 64 and Cout %% 32 must be 0");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    Scratch s{"op_conv_transpose_uv", st};
    float* wuv;
    MG_TRY(s.alloc(&wuv, static_cast<size_t>(8) * Cout * 4));
    MG_TRY(launch_pack_convT_uv(w, Cin, Cout, wuv, st));
    MG_TRY(moge_op_conv(x, w, bias, nullptr, out, nullptr, B, H, W, Cin, Cout, 1, 1, dtype, stream));
    return launch_uv_convT(out, level_geom(H, W, 1), B, Cout, wuv, su, sv, dtype == MOGE_BF16, st);
}

int moge_bicubic_aa_weights(int in, int out, int i, int* lo, float* w, int cap) {
    if (!lo) return set_error("null argument");
    if (in <= 0 || out <= 0 || i < 0 || i >= out) return set_error("bicubic_aa_weights: bad arguments in=%d out=%d i=%d", in, out, i);
    return bicubic_aa_taps(in, out, i, lo, w, cap);
}

}  // extern "C"
