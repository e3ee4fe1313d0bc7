// Load path of libmoge_b200.so: the fp32 staging registry behind moge_engine_set_weight, and moge_engine_finalize, which checks each
// weight's shape, packs the weights into the engine's 16-bit GEMM operands and folds consecutive linear maps at load time.
#include "engine.h"

#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <algorithm>
#include <initializer_list>
#include <string>
#include <vector>

namespace mg {

__global__ void to_f32_kernel(const void* src, int dtype, float* dst, size_t n) {
    for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < n; i += static_cast<size_t>(gridDim.x) * blockDim.x) {
        if (dtype == MOGE_F32) dst[i] = static_cast<const float*>(src)[i];
        else if (dtype == MOGE_F16) dst[i] = __half2float(static_cast<const __half*>(src)[i]);
        else dst[i] = __bfloat162float(static_cast<const __nv_bfloat16*>(src)[i]);
    }
}
// dst[i] = a[i*lda] + (b ? b[i] : 0)
__global__ void vec_combine_kernel(float* dst, const float* a, int lda, const float* b, int n) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) dst[i] = a[static_cast<size_t>(i) * lda] + (b ? b[i] : 0.f);
}

// ------------------------------------------------------------------------------------------------ the folds' vocabulary
// An fp32 device matrix: rows x cols, consecutive rows ld floats apart.  A vector is a column, n x 1 (ld 1 when contiguous).
struct Mat {
    float* p = nullptr;
    int rows = 0, cols = 0, ld = 0;
    Mat row_block(int r0, int n) const { return Mat{p + static_cast<size_t>(r0) * ld, n, cols, ld}; }
    Mat col_block(int c0, int n) const { return Mat{p + c0, rows, n, ld}; }
    Mat col(int c) const { return col_block(c, 1); }
};

// One finalize: the shape-checked weight accessors, the fp32 buffers of the folds and the operations on them, all on one stream.
// Temporaries are zero-filled on allocation and freed with the loader, at the end of finalize or of a failed one.
struct Loader {
    moge_engine* e;
    cudaStream_t st;
    std::vector<void*> temps;
    Loader(moge_engine* e_, cudaStream_t st_) : e(e_), st(st_) {}
    ~Loader() {
        cudaStreamSynchronize(st);          // queued folds may still read them
        for (void* t : temps) cudaFree(t);
    }

    // The staging weight `key` of exactly `shape`, as a shape[0] x (the rest) matrix.
    int get(const std::string& key, std::initializer_list<int64_t> shape, Mat* out) {
        RawWeight* w;
        MG_TRY(find(key, shape, &w));
        const int rows = static_cast<int>(*shape.begin()), cols = rows ? static_cast<int>(w->numel / rows) : 0;
        *out = Mat{w->p, rows, cols, cols};
        return 0;
    }
    // `prefix`.weight of exactly `shape` and `prefix`.bias of shape[0]
    int layer(const std::string& prefix, std::initializer_list<int64_t> shape, Mat* w, Mat* b) {
        MG_TRY(get(prefix + ".weight", shape, w));
        return get(prefix + ".bias", {*shape.begin()}, b);
    }
    // The same for a weight a kernel reads at run time: finalize keeps its staging copy.
    int keep(const std::string& key, std::initializer_list<int64_t> shape, const float** out) {
        RawWeight* w;
        MG_TRY(find(key, shape, &w));
        w->keep = true;
        *out = w->p;
        return 0;
    }
    // Zero-filled fp32 buffers: a rows x cols temporary, or an engine-owned n-vector at *field (m: its view, optional).
    int temp(Mat* m, int rows, int cols = 1) {
        void* p;
        CUDA_TRY(cudaMalloc(&p, std::max<size_t>(static_cast<size_t>(rows) * cols * 4, 16)));
        temps.push_back(p);
        return zero(m, p, rows, cols);
    }
    int owned(float** field, int n, Mat* m = nullptr) {
        Mat v;
        MG_TRY(e->alloc(reinterpret_cast<void**>(field), static_cast<size_t>(n) * 4));
        return zero(m ? m : &v, *field, n, 1);
    }

    // C = A B
    int mm(Mat C, Mat A, Mat B) {
        if (A.cols != B.rows || C.rows != A.rows || C.cols != B.cols)
            return set_error("fold: (%d x %d) = (%d x %d) (%d x %d)", C.rows, C.cols, A.rows, A.cols, B.rows, B.cols);
        return launch_sgemm(A.p, A.ld, B.p, B.ld, C.p, C.ld, A.rows, B.cols, A.cols, 0, st);
    }
    // dst = a + b over n-vectors; without b a copy of a, which may be a column of a matrix
    int add(Mat dst, Mat a, Mat b = Mat()) {
        if (dst.cols != 1 || dst.ld != 1 || a.cols != 1 || dst.rows != a.rows || (b.p && (b.cols != 1 || b.ld != 1 || b.rows != a.rows)))
            return set_error("fold: vector sum over %d x %d and %d x %d into %d x %d", a.rows, a.cols, b.rows, b.cols, dst.rows, dst.cols);
        vec_combine_kernel<<<(a.rows + 255) / 256, 256, 0, st>>>(dst.p, a.p, a.ld, b.p, a.rows);
        CUDA_TRY(cudaGetLastError());
        return 0;
    }
    // *field = a + b in a new engine-owned vector
    int sum(float** field, Mat a, Mat b = Mat()) { Mat v; MG_TRY(owned(field, a.rows, &v)); return add(v, a, b); }
    int upload(Mat dst, const std::vector<float>& v) { CUDA_TRY(cudaMemcpyAsync(dst.p, v.data(), v.size() * 4, cudaMemcpyHostToDevice, st)); return 0; }
    // dst = up2(w): w a 3x3 conv (Cout, Cin, 3, 3) as Cout x 9Cin, dst its first 4 Cout rows (phase, channel) with the bilinear x2
    // before the conv folded in (pack.cu)
    int up2(Mat dst, Mat w) {
        if (dst.rows < 4 * w.rows || dst.cols != w.cols || w.ld != w.cols || dst.ld != dst.cols)
            return set_error("fold: up2 of %d x %d into %d x %d", w.rows, w.cols, dst.rows, dst.cols);
        return launch_up2_expand(w.p, dst.p, w.rows, w.cols / 9, st);
    }

    // ---- the 16-bit operands
    // dst [w.rows, dst_ld] = w, zero past w's columns
    int cast(void* dst, Mat w, int dst_ld) { return launch_cast_2d(w.p, MOGE_F32, dst, e->bf16, w.rows, w.cols, w.ld, dst_ld, st); }
    // cw: an engine-owned [N, taps * cin + caux] operand
    int conv(ConvW* cw, int N, int cin, int taps, int caux = 0) {
        cw->N = N; cw->cin = cin; cw->taps = taps; cw->caux = caux; cw->Ktot = taps * cin + caux;
        return e->alloc(&cw->w, static_cast<size_t>(N) * cw->Ktot * 2);
    }
    // cw's columns [k_off, k_off + w.cols) from a conv weight (N, C, taps) as N x (C * taps)
    int pack_conv(const ConvW& cw, Mat w, int taps, int k_off) {
        if (w.rows != cw.N || w.ld != w.cols || k_off + w.cols > cw.Ktot) return set_error("fold: conv weight %d x %d into [%d, %d]", w.rows, w.cols, cw.N, cw.Ktot);
        return launch_pack_conv(w.p, cw.w, e->bf16, w.rows, w.cols / taps, taps, cw.Ktot, k_off, st);
    }
    // cw from a k2s2 ConvTranspose2d weight (Cin, Cout, 2, 2) as Cin x 4Cout
    int pack_convT(const ConvW& cw, Mat w) {
        if (w.rows != cw.Ktot || w.cols != cw.N || w.ld != w.cols) return set_error("fold: convT weight %d x %d into [%d, %d]", w.rows, w.cols, cw.N, cw.Ktot);
        return launch_pack_convT(w.p, cw.w, e->bf16, w.rows, w.cols / 4, st);
    }

  private:
    int find(const std::string& key, std::initializer_list<int64_t> shape, RawWeight** out) {
        auto it = e->raw.find(key);
        if (it == e->raw.end()) return set_error("missing weight '%s'", key.c_str());
        if (!std::equal(shape.begin(), shape.end(), it->second.shape.begin(), it->second.shape.end())) {
            std::string got, want;
            for (auto d : it->second.shape) got += std::to_string(d) + ",";
            for (auto d : shape) want += std::to_string(d) + ",";
            return set_error("weight '%s' has shape (%s) expected (%s)", key.c_str(), got.c_str(), want.c_str());
        }
        *out = &it->second;
        return 0;
    }
    int zero(Mat* m, void* p, int rows, int cols) {
        CUDA_TRY(cudaMemsetAsync(p, 0, static_cast<size_t>(rows) * cols * 4, st));
        *m = Mat{static_cast<float*>(p), rows, cols, cols};
        return 0;
    }
};

// ------------------------------------------------------------------------------------------------ finalize
// a linear's weight of `shape` (N, K...) -> engine-owned 16-bit [N, Kpad]
static int pack_linear(Loader& ctx, const std::string& key, std::initializer_list<int64_t> shape, int Kpad, void** out) {
    Mat w;
    MG_TRY(ctx.get(key, shape, &w));
    MG_TRY(ctx.e->alloc(out, static_cast<size_t>(w.rows) * Kpad * 2));
    return ctx.cast(*out, w, Kpad);
}

// 3x3 conv (Cout,Cin,3,3) [+ aux 1x1 (Cout,Caux,1,1)] [+ UV 1x1 (Cout,2,1,1)] -> ConvW; up2: a bilinear x2 before the conv, folded
// in as 4 output phases that run on the low-resolution grid
static int pack_conv3(Loader& ctx, const std::string& wkey, int Cout, int Cin, const std::string& in_key, int Caux, bool uv, ConvW* cw,
                      bool up2 = false) {
    Mat w, b, wi, b_in;
    MG_TRY(ctx.layer(wkey, {Cout, Cin, 3, 3}, &w, &b));
    if (Cin % 64) return set_error("conv '%s': C_in=%d must be a multiple of 64", wkey.c_str(), Cin);
    if (up2) {
        Mat wexp;
        MG_TRY(ctx.temp(&wexp, 4 * Cout, 9 * Cin));
        MG_TRY(ctx.up2(wexp, w));
        w = wexp;
    }
    MG_TRY(ctx.conv(cw, w.rows, Cin, 9, Caux));
    MG_TRY(ctx.pack_conv(*cw, w, 9, 0));
    if (!in_key.empty()) {
        if (uv) {
            MG_TRY(ctx.layer(in_key, {Cout, 2, 1, 1}, &wi, &b_in));
            MG_TRY(ctx.sum(&cw->wu, wi.col(0)));
            MG_TRY(ctx.sum(&cw->wv, wi.col(1)));
        } else {
            if (Caux % 64) return set_error("input block '%s': C=%d must be a multiple of 64", in_key.c_str(), Caux);
            MG_TRY(ctx.layer(in_key, {Cout, Caux, 1, 1}, &wi, &b_in));
            MG_TRY(ctx.pack_conv(*cw, wi, 1, 9 * Cin));
        }
    }
    return ctx.sum(&cw->bias, b, b_in);
}

// waux: the [8, 32] map from the neck's last-level map to the heads' output components (points xyz | normal xyz | mask logit |
// pad).  A head gets its own rows and writes [ncomp, 32] (output block o last-level input block) there; the neck reads all 8 rows.
static int pack_stack(Loader& ctx, const std::string& name, const moge_stack_config_t& sc, bool is_neck, StackW* sw, Mat waux) {
    const int L = sc.num_levels;
    sw->res.assign(L, {});
    sw->convT.assign(L, ConvW());
    sw->post.assign(L, ConvW());
    const int* C = sc.dim_res_blocks;
    if (!is_neck) {
        // level-0 input block: 1x1 conv C0 -> C0 on the neck's level-0 output
        if (sc.dim_in[0] <= 0) return set_error("%s: level-0 input block required", name.c_str());
        Mat w, b;
        MG_TRY(ctx.layer(name + ".input_blocks.0", {C[0], sc.dim_in[0], 1, 1}, &w, &b));
        if (sc.dim_in[0] % 64) return set_error("%s: level-0 C_in=%d must be a multiple of 64", name.c_str(), sc.dim_in[0]);
        MG_TRY(ctx.conv(&sw->in0, C[0], sc.dim_in[0], 1));
        MG_TRY(ctx.pack_conv(sw->in0, w, 1, 0));
        MG_TRY(ctx.sum(&sw->in0.bias, b));
    }
    for (int l = 0; l < L; ++l) {
        const bool last = (l == L - 1);
        if (sc.dim_out[l] > 0 && !(last && !is_neck)) return set_error("%s: output block at level %d unsupported", name.c_str(), l);
        for (int r = 0; r < sc.num_res_blocks[l]; ++r) {
            if (last && !is_neck) return set_error("%s: residual blocks at the last head level unsupported", name.c_str());
            for (int k : {2, 5}) {
                ConvW cw;
                MG_TRY(pack_conv3(ctx, name + ".res_blocks." + std::to_string(l) + "." + std::to_string(r) + ".layers." + std::to_string(k),
                                  C[l], C[l], "", 0, false, &cw));
                sw->res[l].push_back(cw);
            }
        }
        if (last) break;
        const std::string rs = name + ".resamplers." + std::to_string(l);
        const std::string in_key = sc.dim_in[l + 1] > 0 ? name + ".input_blocks." + std::to_string(l + 1) : std::string();
        const bool fold_head_out = !is_neck && (l + 1 == L - 1);
        int conv_cin;
        if (sc.resamplers[l] == MOGE_RESAMPLE_CONV_TRANSPOSE) {
            Mat w, b;
            MG_TRY(ctx.get(rs + ".0.weight", {C[l], C[l + 1], 2, 2}, &w));
            MG_TRY(ctx.get(rs + ".0.bias", {C[l + 1]}, &b));
            if (C[l] % 64 || C[l + 1] % 32) return set_error("%s: convT %d->%d channel counts unsupported", name.c_str(), C[l], C[l + 1]);
            ConvW& ct = sw->convT[l];
            MG_TRY(ctx.conv(&ct, 4 * C[l + 1], C[l], 1));
            MG_TRY(ctx.pack_convT(ct, w));
            MG_TRY(ctx.sum(&ct.bias, b));
            conv_cin = C[l + 1];
        } else if (sc.resamplers[l] == MOGE_RESAMPLE_BILINEAR) {
            conv_cin = C[l];
        } else {
            return set_error("%s: resampler type %d unsupported", name.c_str(), sc.resamplers[l]);
        }
        if (!fold_head_out) {
            if (is_neck) {
                if (sc.dim_in[l + 1] != 2) return set_error("neck: dim_in[%d] must be 2 (UV planes)", l + 1);
                if (l + 1 == L - 1) {
                    // Last neck level folded through the heads (EPI_NECKOUT).  The level-(L-1) neck map m = conv3x3(up2(x)) + b + Wuv uv
                    // is consumed ONLY by the heads' last-level input blocks and, with no nonlinearity in between, by their output
                    // blocks: head k-th component += waux[k, :] m.  Push waux through the (linear) conv: a 3x3 conv with
                    // 4 phases x 8 components on the low-resolution grid; the 32-channel map at the 16x grid is never materialised.
                    //   W[phase] = waux W_up2[phase],  b = waux (b_conv + b_in),  wu / wv = waux W_in[:, 0 / 1]
                    const int Cn = C[l + 1];
                    Mat wc, bc, wi, bi, wexp, wfold, bsum, bias, wu, wv;
                    MG_TRY(ctx.layer(rs + ".1", {Cn, conv_cin, 3, 3}, &wc, &bc));
                    MG_TRY(ctx.layer(in_key, {Cn, 2, 1, 1}, &wi, &bi));
                    MG_TRY(ctx.temp(&wexp, 4 * Cn, 9 * conv_cin));
                    MG_TRY(ctx.up2(wexp, wc));                                                  // rows (phase, channel)
                    MG_TRY(ctx.temp(&wfold, 32, 9 * conv_cin));                                 // rows (phase, component)
                    for (int ph = 0; ph < 4; ++ph) MG_TRY(ctx.mm(wfold.row_block(8 * ph, 8), waux, wexp.row_block(Cn * ph, Cn)));
                    ConvW& no = sw->neckout;
                    MG_TRY(ctx.conv(&no, 32, conv_cin, 9));
                    MG_TRY(ctx.pack_conv(no, wfold, 9, 0));
                    MG_TRY(ctx.temp(&bsum, Cn));
                    MG_TRY(ctx.add(bsum, bc, bi));
                    MG_TRY(ctx.owned(&no.bias, 8, &bias));
                    MG_TRY(ctx.mm(bias, waux, bsum));
                    MG_TRY(ctx.owned(&no.wu, 8, &wu));
                    MG_TRY(ctx.owned(&no.wv, 8, &wv));
                    MG_TRY(ctx.mm(wu, waux, wi.col(0)));
                    MG_TRY(ctx.mm(wv, waux, wi.col(1)));
                    continue;
                }
                MG_TRY(pack_conv3(ctx, rs + ".1", C[l + 1], conv_cin, in_key, 0, true, &sw->post[l], sc.resamplers[l] == MOGE_RESAMPLE_BILINEAR));
            } else {
                if (sc.dim_in[l + 1] <= 0) return set_error("%s: input block at level %d required", name.c_str(), l + 1);
                if (sc.resamplers[l] == MOGE_RESAMPLE_BILINEAR) return set_error("%s: a bilinear resampler is supported at the last level only", name.c_str());
                MG_TRY(pack_conv3(ctx, rs + ".1", C[l + 1], conv_cin, in_key, sc.dim_in[l + 1], false, &sw->post[l]));
            }
        } else {
            // head tail: conv3x3 (conv_cin -> 32) + in_block(neck_last 32 -> 32) then output block 32 -> ncomp, no
            // nonlinearity in between  =>  one 3x3 conv conv_cin -> ncomp plus a [ncomp,32] map of the neck map:
            //   W = up2(W_out W_conv),  b = W_out (b_conv + b_in) + b_out,  waux = W_out W_in
            const int Cl = C[L - 1], nc = sc.dim_out[L - 1];
            if (Cl != 32 || sc.dim_in[L - 1] != 32 || nc <= 0 || nc > 3 || nc > waux.rows || conv_cin % 64)
                return set_error("%s: last level must be 32 channels with a 1..3 channel output block", name.c_str());
            if (sc.resamplers[l] != MOGE_RESAMPLE_BILINEAR) return set_error("%s: the last resampler must be bilinear", name.c_str());
            const std::string ob = name + ".output_blocks." + std::to_string(L - 1);
            Mat wc, bc, w4, b4, wo, bo, wnc, wexp, bsum, bias;
            MG_TRY(ctx.layer(rs + ".1", {Cl, conv_cin, 3, 3}, &wc, &bc));
            MG_TRY(ctx.layer(in_key, {Cl, 32, 1, 1}, &w4, &b4));
            MG_TRY(ctx.layer(ob, {nc, Cl, 1, 1}, &wo, &bo));
            MG_TRY(ctx.temp(&wnc, nc, 9 * conv_cin));
            MG_TRY(ctx.mm(wnc, wo, wc));                                                        // (nc, Cin, 3, 3)
            MG_TRY(ctx.temp(&wexp, 16, 9 * conv_cin));                                          // rows (phase, component), zero past 4 nc
            MG_TRY(ctx.up2(wexp, wnc));
            ConvW& ho = sw->headout;
            MG_TRY(ctx.conv(&ho, 16, conv_cin, 9));
            MG_TRY(ctx.pack_conv(ho, wexp, 9, 0));
            MG_TRY(ctx.mm(waux.row_block(0, nc), wo, w4));
            MG_TRY(ctx.temp(&bsum, Cl));
            MG_TRY(ctx.add(bsum, bc, b4));
            MG_TRY(ctx.owned(&ho.bias, 16, &bias));
            MG_TRY(ctx.mm(bias.row_block(0, nc), wo, bsum));
            MG_TRY(ctx.add(bias.row_block(0, nc), bias.row_block(0, nc), bo));
            sw->ncomp = nc;
        }
    }
    return 0;
}

static int finalize_encoder(Loader& ctx) {
    moge_engine* e = ctx.e;
    const moge_config_t& c = e->cfg;
    const int D = c.embed_dim;
    const std::string bb = e->dino ? "" : e->v1 ? "backbone." : "encoder.backbone.";
    MG_TRY(pack_linear(ctx, bb + "patch_embed.proj.weight", {D, 3, 14, 14}, 592, &e->w_patch));
    MG_TRY(ctx.keep(bb + "patch_embed.proj.bias", {D}, &e->patch_bias));
    MG_TRY(ctx.keep(bb + "pos_embed", {1, 1 + 37 * 37, D}, &e->pos_embed));
    MG_TRY(ctx.keep(bb + "cls_token", {1, 1, D}, &e->cls_token));
    MG_TRY(ctx.keep(bb + "norm.weight", {D}, &e->norm_g));
    MG_TRY(ctx.keep(bb + "norm.bias", {D}, &e->norm_b));
    e->blk.resize(c.depth);
    for (int i = 0; i < c.depth; ++i) {
        const std::string p = bb + "blocks." + std::to_string(i) + ".";
        moge_engine::Blk& b = e->blk[i];
        MG_TRY(pack_linear(ctx, p + "attn.proj.weight", {D, D}, D, &b.wproj));
        MG_TRY(pack_linear(ctx, p + "mlp.fc2.weight", {D, 4 * D}, 4 * D, &b.wfc2));
        Mat wq, bqkv, wf, bfc1, ln1g, ln1b, ln2g, ln2b;
        MG_TRY(ctx.keep(p + "attn.proj.bias", {D}, &b.bproj));
        MG_TRY(ctx.keep(p + "mlp.fc2.bias", {D}, &b.bfc2));
        MG_TRY(ctx.keep(p + "ls1.gamma", {D}, &b.g1));
        MG_TRY(ctx.keep(p + "ls2.gamma", {D}, &b.g2));
        MG_TRY(ctx.layer(p + "norm1", {D}, &ln1g, &ln1b));
        MG_TRY(ctx.layer(p + "norm2", {D}, &ln2g, &ln2b));
        MG_TRY(ctx.layer(p + "attn.qkv", {3 * D, D}, &wq, &bqkv));
        MG_TRY(ctx.layer(p + "mlp.fc1", {4 * D, D}, &wf, &bfc1));
        MG_TRY(e->alloc(&b.wqkv_ln, static_cast<size_t>(3 * D) * D * 2));
        MG_TRY(e->alloc(&b.wfc1_ln, static_cast<size_t>(4 * D) * D * 2));
        MG_TRY(ctx.owned(&b.b_qkv_ln, 3 * D));
        MG_TRY(ctx.owned(&b.b_fc1_ln, 4 * D));
        MG_TRY(launch_ln_fold(wq.p, ln1g.p, ln1b.p, bqkv.p, 3 * D, D, D, b.wqkv_ln, b.b_qkv_ln, e->bf16, ctx.st));
        MG_TRY(launch_ln_fold(wf.p, ln2g.p, ln2b.p, bfc1.p, 4 * D, D, D, b.wfc1_ln, b.b_fc1_ln, e->bf16, ctx.st));
    }
    return 0;
}

static int finalize_v2_decoder(Loader& ctx) {
    moge_engine* e = ctx.e;
    const moge_config_t& c = e->cfg;
    const int D = c.embed_dim;
    // ---- fold: neck.input_blocks.0 o (sum_j output_projections.j)  ->  one GEMM over the concatenated taps:
    //   W[:, tap j] = W_0 P_j,  b = W_0 (sum_j b_j) + b_0,  wu / wv = W_0[:, Do / Do + 1] (the UV planes)
    {
        const int C0 = c.neck.dim_res_blocks[0], Do = c.dim_out, nt = c.num_taps;
        if (c.neck.dim_in[0] != Do + 2) return set_error("neck.dim_in[0]=%d must be encoder.dim_out+2=%d", c.neck.dim_in[0], Do + 2);
        Mat w0, b0, wf, bp, bias;
        MG_TRY(ctx.layer("neck.input_blocks.0", {C0, Do + 2, 1, 1}, &w0, &b0));
        const Mat w0x = w0.col_block(0, Do);          // the columns applied to the projected taps
        MG_TRY(ctx.temp(&wf, C0, nt * D));
        MG_TRY(ctx.temp(&bp, Do));
        for (int j = 0; j < nt; ++j) {
            Mat w, b;
            MG_TRY(ctx.layer("encoder.output_projections." + std::to_string(j), {Do, D, 1, 1}, &w, &b));
            MG_TRY(ctx.mm(wf.col_block(j * D, D), w0x, w));
            MG_TRY(ctx.add(bp, bp, b));
        }
        ConvW& f = e->fold0;
        MG_TRY(ctx.owned(&f.bias, C0, &bias));
        MG_TRY(ctx.mm(bias, w0x, bp));
        MG_TRY(ctx.add(bias, bias, b0));
        MG_TRY(ctx.conv(&f, C0, nt * D, 1));
        MG_TRY(ctx.cast(f.w, wf, f.Ktot));
        MG_TRY(ctx.sum(&f.wu, w0.col(Do)));
        MG_TRY(ctx.sum(&f.wv, w0.col(Do + 1)));
    }
    // the heads' last levels first: they give the map through which the neck's last level is folded (EPI_NECKOUT)
    Mat waux;
    MG_TRY(ctx.temp(&waux, 8, 32));
    const int row_of[4] = {0, 3, 6, 8};          // points xyz | normal xyz | mask logit | pad
    for (int i = 0; i < 3; ++i)
        if (head_cfg(e, i)->present)
            MG_TRY(pack_stack(ctx, head_name(i), *head_cfg(e, i), false, &e->heads[i], waux.row_block(row_of[i], row_of[i + 1] - row_of[i])));
    MG_TRY(pack_stack(ctx, "neck", c.neck, true, &e->neck, waux));
    for (int l = 0; l < c.scale_head_layers; ++l) {
        const std::string k = "scale_head." + std::to_string(2 * l);
        const float *w, *b;
        MG_TRY(ctx.keep(k + ".weight", {c.scale_head_dims[l + 1], c.scale_head_dims[l]}, &w));
        MG_TRY(ctx.keep(k + ".bias", {c.scale_head_dims[l + 1]}, &b));
        e->mlp_w.push_back(w);
        e->mlp_b.push_back(b);
    }
    return 0;
}

// ---- MoGe-1 decoder (keys head.*, v1.py:61-142).  The output blocks' small folds are done on the host from copies of the fp32
// staging weights.
static int to_host(Mat w, std::vector<float>* out) {
    out->resize(static_cast<size_t>(w.rows) * w.cols);
    CUDA_TRY(cudaMemcpy(out->data(), w.p, out->size() * 4, cudaMemcpyDeviceToHost));
    return 0;
}

static int finalize_v1(Loader& ctx) {
    moge_engine* e = ctx.e;
    const moge_v1_config_t& c = e->v1cfg;
    const int D = c.embed_dim, nt = c.num_taps, P = c.dim_proj;
    CUDA_TRY(cudaStreamSynchronize(ctx.st));       // the staging copies are written on st; the host reads some of them below
    V1W& v = e->v1w;
    // V4: sum_j projects.j(tap_j) = one GEMM over the concatenated taps [B*T, nt*D]:  W = [W_0 | W_1 | ...],  b = sum_j b_j
    {
        ConvW& pj = v.proj;
        Mat wcat, bias;
        MG_TRY(ctx.conv(&pj, P, nt * D, 1));
        MG_TRY(ctx.owned(&pj.bias, P, &bias));
        MG_TRY(ctx.temp(&wcat, P, nt * D));
        for (int j = 0; j < nt; ++j) {
            Mat w, b;
            MG_TRY(ctx.layer("head.projects." + std::to_string(j), {P, D, 1, 1}, &w, &b));
            const Mat dst = wcat.col_block(j * D, D);
            CUDA_TRY(cudaMemcpy2DAsync(dst.p, dst.ld * 4, w.p, w.ld * 4, w.cols * 4, w.rows, cudaMemcpyDeviceToDevice, ctx.st));
            MG_TRY(ctx.add(bias, bias, b));
        }
        MG_TRY(ctx.cast(pj.w, wcat, pj.Ktot));
    }
    int cin = P;
    v.lv.assign(c.num_levels, V1Level());
    for (int l = 0; l < c.num_levels; ++l) {
        const int Co = c.dim_upsample[l], Hd = c.hidden_mult * Co;
        const std::string pre = "head.upsample_blocks." + std::to_string(l) + ".";
        V1Level& L = v.lv[l];
        // V5: ConvTranspose2d(cin + 2 -> Co): rows 0..cin-1 through the GEMM, the two UV rows as the input-grid term
        Mat wt, bt;
        MG_TRY(ctx.get(pre + "0.0.weight", {cin + 2, Co, 2, 2}, &wt));
        MG_TRY(ctx.get(pre + "0.0.bias", {Co}, &bt));
        MG_TRY(ctx.conv(&L.convT, 4 * Co, cin, 1));
        MG_TRY(ctx.pack_convT(L.convT, wt.row_block(0, cin)));
        MG_TRY(ctx.sum(&L.convT.bias, bt));
        MG_TRY(ctx.owned(&L.wuv, 8 * Co));
        MG_TRY(launch_pack_convT_uv(wt.p, cin, Co, L.wuv, ctx.st));
        MG_TRY(pack_conv3(ctx, pre + "0.1", Co, Co, "", 0, false, &L.conv));
        for (int r = 0; r < c.num_res_blocks; ++r) {
            const std::string rp = pre + std::to_string(1 + r) + ".layers.";
            V1Res R;
            MG_TRY(ctx.keep(rp + "0.weight", {Co}, &R.g1));
            MG_TRY(ctx.keep(rp + "0.bias", {Co}, &R.b1));
            MG_TRY(pack_conv3(ctx, rp + "2", Hd, Co, "", 0, false, &R.c1));
            MG_TRY(ctx.keep(rp + "3.weight", {Hd}, &R.g2));
            MG_TRY(ctx.keep(rp + "3.bias", {Hd}, &R.b2));
            MG_TRY(pack_conv3(ctx, rp + "5", Co, Hd, "", 0, false, &R.c2));
            R.G2 = c.hidden_norm == MOGE_V1_GROUP_NORM ? Hd / 32 : 1;
            L.res.push_back(R);
        }
        cin = Co;
    }
    // V7: output blocks k = 0 (points, 3) and 1 (mask, 1): conv3x3 (cin + 2 -> 32), ReLU, conv1x1 (32 -> n_k)
    const int lc = c.last_conv_channels, nout[2] = {3, 1};
    std::vector<float> wcat(static_cast<size_t>(2) * lc * cin * 9), bcat(2 * lc), params(64 * 6 + 4 * 64 + 4, 0.f);
    for (int k = 0; k < 2; ++k) {
        const std::string ob = "head.output_block." + std::to_string(k) + ".";
        Mat wc, bc, wo, bo;
        MG_TRY(ctx.layer(ob + "0", {lc, cin + 2, 3, 3}, &wc, &bc));
        MG_TRY(ctx.layer(ob + "2", {nout[k], lc, 1, 1}, &wo, &bo));
        std::vector<float> hw, hb, hwo, hbo;
        MG_TRY(to_host(wc, &hw));
        MG_TRY(to_host(bc, &hb));
        MG_TRY(to_host(wo, &hwo));
        MG_TRY(to_host(bo, &hbo));
        for (int co = 0; co < lc; ++co) {
            const int n = k * lc + co;
            const float* src = hw.data() + static_cast<size_t>(co) * (cin + 2) * 9;
            std::copy(src, src + static_cast<size_t>(cin) * 9, wcat.begin() + static_cast<size_t>(n) * cin * 9);
            bcat[n] = hb[co];
            // UV part of the replicate-padded 3x3 conv: u depends on x only, v on y only -> six folded weights
            const float* wu = src + static_cast<size_t>(cin) * 9;
            const float* wv = wu + 9;
            for (int d = 0; d < 3; ++d) {
                params[n * 6 + d] = wu[0 * 3 + d] + wu[1 * 3 + d] + wu[2 * 3 + d];          // sum over dy, tap dx = d - 1
                params[n * 6 + 3 + d] = wv[d * 3 + 0] + wv[d * 3 + 1] + wv[d * 3 + 2];      // sum over dx, tap dy = d - 1
            }
            for (int o = 0; o < nout[k]; ++o) params[64 * 6 + (k == 0 ? o : 3) * 64 + n] = hwo[static_cast<size_t>(o) * lc + co];
        }
        for (int o = 0; o < nout[k]; ++o) params[64 * 6 + 4 * 64 + (k == 0 ? o : 3)] = hbo[o];
    }
    Mat wout, wcat_dev, bias;
    MG_TRY(ctx.owned(&v.wout, static_cast<int>(params.size()), &wout));
    MG_TRY(ctx.upload(wout, params));
    MG_TRY(ctx.temp(&wcat_dev, 2 * lc, 9 * cin));
    MG_TRY(ctx.upload(wcat_dev, wcat));
    ConvW& oc = v.out;
    MG_TRY(ctx.conv(&oc, 2 * lc, cin, 9));
    MG_TRY(ctx.pack_conv(oc, wcat_dev, 9, 0));
    MG_TRY(ctx.owned(&oc.bias, 2 * lc, &bias));
    return ctx.upload(bias, bcat);
}

static int finalize(moge_engine* e, cudaStream_t st) {
    Loader ctx(e, st);
    MG_TRY(finalize_encoder(ctx));
    if (!e->dino) MG_TRY(e->v1 ? finalize_v1(ctx) : finalize_v2_decoder(ctx));
    CUDA_TRY(cudaStreamSynchronize(st));
    // release the staging copies no kernel reads at run time
    for (auto& kv : e->raw)
        if (!kv.second.keep && kv.second.p) { cudaFree(kv.second.p); kv.second.p = nullptr; }
    e->finalized = true;
    return 0;
}

}  // namespace mg

using namespace mg;

extern "C" {

int moge_engine_set_weight(moge_engine_t* e, const char* key, const void* dev_ptr, const int64_t* shape, int ndim, int dtype, void* stream) {
    if (!e || !key || !dev_ptr) return set_error("null argument");
    if (e->finalized) return set_error("engine already finalized");
    if (dtype != MOGE_F32 && dtype != MOGE_F16 && dtype != MOGE_BF16) return set_error("weight '%s': unsupported dtype %d", key, dtype);
    CUDA_TRY(cudaSetDevice(e->device));
    RawWeight rw;
    rw.numel = 1;
    for (int i = 0; i < ndim; ++i) { rw.shape.push_back(shape[i]); rw.numel *= static_cast<size_t>(shape[i]); }
    CUDA_TRY(cudaMalloc(reinterpret_cast<void**>(&rw.p), std::max<size_t>(rw.numel, 4) * 4));
    const int blocks = static_cast<int>(std::min<size_t>((rw.numel + 255) / 256, 132 * 8));
    to_f32_kernel<<<std::max(blocks, 1), 256, 0, static_cast<cudaStream_t>(stream)>>>(dev_ptr, dtype, rw.p, rw.numel);
    CUDA_TRY(cudaGetLastError());
    auto it = e->raw.find(key);
    if (it != e->raw.end() && it->second.p) cudaFree(it->second.p);
    e->raw[key] = rw;
    return 0;
}

int moge_engine_finalize(moge_engine_t* e, void* stream) {
    if (!e) return set_error("null engine");
    if (e->finalized) return 0;
    CUDA_TRY(cudaSetDevice(e->device));
    return finalize(e, static_cast<cudaStream_t>(stream));
}

}  // extern "C"
