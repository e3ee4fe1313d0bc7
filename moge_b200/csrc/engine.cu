// Host runtime of libmoge_b200.so: weight registry + load-time repacking, per-shape execution plans (workspace
// layout, TMA descriptors, launch list), and the extern "C" ABI declared in include/moge_b200.h.
#include "moge_b200.h"
#include "gemm_kernel.cuh"
#include "host_api.h"

#include <algorithm>
#include <functional>
#include <map>
#include <memory>
#include <string>
#include <vector>
#include <math.h>

namespace mg {

const char* last_error();

// ------------------------------------------------------------------------------------------------ helpers
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

struct RawWeight {
    float* p = nullptr;
    std::vector<int64_t> shape;
    size_t numel = 0;
};

struct StackW {
    ConvW in0;                                  // heads: 1x1 input block at level 0
    std::vector<std::vector<ConvW>> res;        // [level][2*r + {0,1}]
    std::vector<ConvW> convT;                   // [level] (conv_transpose resampler)
    std::vector<ConvW> post;                    // [level] 3x3 after the resampler (writes level l+1), fused in-block / UV
    // folded last level of a head
    ConvW headout;
    int ncomp = 0;
    // neck only: its last level folded through the heads' last-level input + output blocks (EPI_NECKOUT): N = 4 phases x 8 components
    ConvW neckout;
};

struct Op {
    std::function<int(cudaStream_t)> fn;
    std::string name;      // kernel class + role, e.g. "gemm.qkv", "conv3x3.neck.l2", "attention"
    double flops = 0;      // algorithmic flops (2*MAC) of this launch
    double bytes = 0;      // algorithmic HBM bytes of this launch (each operand/result once)
    int phase = 1;         // 0: reads a caller-bound input (preprocess)   1: touches the workspace only (graph-capturable with a
                           // key that is just the workspace)   2: writes a caller-bound output (scale head, head output)
};

struct OpList : std::vector<Op> {
    void add(std::function<int(cudaStream_t)> fn, const std::string& name, double flops = 0, double bytes = 0, int phase = 1) {
        Op o; o.fn = std::move(fn); o.name = name; o.flops = flops; o.bytes = bytes; o.phase = phase;
        push_back(std::move(o));
    }
};

// One shape group of a forward call: B images of H x W pixels on an h x w token grid.  A call may carry several groups
// (mixed-aspect batches): the encoder runs ONCE over the token rows of all groups packed back to back, everything that
// depends on the pixel geometry (preprocess, patch/pos embed, taps, decoder, output resize) runs per group.
struct Group {
    int B = 0, H = 0, W = 0, h = 0, w = 0;
    int rh = 0, rw = 0;           // MoGe-1: the resized image the encoder and decoder see (0 for MoGe-2)
    int img0 = 0;                 // index of the group's first image among all images of the call
    long row0 = 0;                // first row of the group in the packed token matrices
    float* pos_table = nullptr;   // plan-owned, [h*w, D] (bicubic-resampled pos embed + patch bias)
    // bindings (set per forward)
    const void* image = nullptr; int image_dtype = 0;
    float* points = nullptr; float* normal = nullptr; float* mask = nullptr; float* scale = nullptr;
};

struct Plan {
    std::vector<Group> groups;
    void* ws = nullptr;
    size_t ws_bytes = 0;
    OpList ops;                    // in launch order: all phase-0 ops, then phase 1, then phase 2
    std::vector<void*> owned;      // device buffers that live and die with the plan (pos tables, cls row, attention work list)
    float* cls_row = nullptr;
    std::vector<AttnItem> att_items; std::vector<int2> att_ranges;     // host copies (source of the async upload)
    // ONE CUDA graph of the phase-1 launches (they touch nothing but the workspace the plan is keyed on, so the graph never
    // goes stale when the caller passes fresh input / output tensors): the launch list of a single image is ~240 kernels of a
    // few microseconds each and replaying a graph removes the per-launch CPU cost.  Phase 0 / 2 launches run eagerly around it.
    cudaGraphExec_t exec = nullptr;
    int eager_runs = 0;
    bool same_shape(const moge_group_t* g, int n, int rh, int rw) const {
        if (static_cast<int>(groups.size()) != n) return false;
        for (int i = 0; i < n; ++i)
            if (groups[i].B != g[i].B || groups[i].H != g[i].H || groups[i].W != g[i].W || groups[i].h != g[i].h || groups[i].w != g[i].w ||
                groups[i].rh != rh || groups[i].rw != rw) return false;
        return true;
    }
    ~Plan() {
        if (exec) cudaGraphExecDestroy(exec);
        for (void* p : owned) cudaFree(p);
    }
};

// MoGe-1 decoder weights (v1.py:61-142)
struct V1Res {            // ResidualConvBlock: GN(1, C) -> ReLU -> conv C->Hd -> GN(G2, Hd) -> ReLU -> conv Hd->C, identity skip
    ConvW c1, c2;
    const float *g1 = nullptr, *b1 = nullptr, *g2 = nullptr, *b2 = nullptr;
    int G2 = 1;
};
struct V1Level {
    ConvW convT, conv;      // ConvTranspose2d k2s2 over the feature channels (pixel shuffle), 3x3 replicate conv
    float* wuv = nullptr;   // [2][4 phases][C]: the convT's UV rows, applied on the input grid
    std::vector<V1Res> res;
};
struct V1W {
    ConvW proj;             // the summed 1x1 projections of the taps as one GEMM over the concatenated taps
    std::vector<V1Level> lv;
    ConvW out;              // both output blocks' 3x3 convs over the feature channels: N = 32 points + 32 mask
    float* wout = nullptr;  // launch_v1_output parameters: folded UV weights, block-diagonal 64 -> 4 map, biases
};

}  // namespace mg

using namespace mg;

struct moge_engine {
    moge_config_t cfg;
    bool v1 = false;                  // created by moge_engine_create_v1: cfg holds the encoder only, v1cfg the rest
    moge_v1_config_t v1cfg{};
    V1W v1w;
    int device = 0, num_sms = 132;
    bool bf16 = false, finalized = false;
    std::map<std::string, RawWeight> raw;
    std::vector<void*> owned;         // cudaMalloc'd, freed at destroy
    // packed encoder
    void* w_patch = nullptr;
    struct Blk {
        // qkv / fc1 with norm1 / norm2 folded in: centred W diag(gamma) in 16 bit, b + W beta
        void *wqkv_ln, *wfc1_ln;
        float *b_qkv_ln, *b_fc1_ln;
        void *wproj, *wfc2;
        const float *bproj, *bfc2, *g1, *g2;     // g1, g2: LayerScale gamma
    };
    std::vector<Blk> blk;
    const float *norm_g = nullptr, *norm_b = nullptr, *pos_embed = nullptr, *cls_token = nullptr, *patch_bias = nullptr;
    ConvW fold0;                      // taps-concat GEMM: (output projections folded into neck.input_blocks.0)
    StackW neck, heads[3];            // heads: points, normal, mask
    std::vector<const float*> mlp_w, mlp_b;
    std::vector<std::unique_ptr<Plan>> plans;      // LRU order (most recently used last), at most kMaxPlans
    Plan* last_plan = nullptr;
    std::vector<void*> temps;         // load-time scratch (fp32 folds), freed at the end of finalize
    cudaStream_t own_stream = nullptr;
    cudaEvent_t ev_in = nullptr, ev_out = nullptr;

    int alloc(void** p, size_t bytes) {
        CUDA_TRY(cudaMalloc(p, bytes ? bytes : 16));
        owned.push_back(*p);
        return 0;
    }
    int alloc_temp(void** p, size_t bytes) {
        CUDA_TRY(cudaMalloc(p, bytes ? bytes : 16));
        temps.push_back(*p);
        return 0;
    }
};

namespace mg {

static const moge_stack_config_t* head_cfg(const moge_engine* e, int i) {
    return i == 0 ? &e->cfg.points_head : i == 1 ? &e->cfg.normal_head : &e->cfg.mask_head;
}
static const char* head_name(int i) { return i == 0 ? "points_head" : i == 1 ? "normal_head" : "mask_head"; }

static int get_raw(moge_engine* e, const std::string& key, const RawWeight** out, std::initializer_list<int64_t> shape) {
    auto it = e->raw.find(key);
    if (it == e->raw.end()) return set_error("missing weight '%s'", key.c_str());
    if (shape.size()) {
        if (it->second.shape.size() != shape.size() || !std::equal(shape.begin(), shape.end(), it->second.shape.begin())) {
            std::string got;
            for (auto d : it->second.shape) got += std::to_string(d) + ",";
            std::string want;
            for (auto d : shape) want += std::to_string(d) + ",";
            return set_error("weight '%s' has shape (%s) expected (%s)", key.c_str(), got.c_str(), want.c_str());
        }
    }
    *out = &it->second;
    return 0;
}

// ------------------------------------------------------------------------------------------------ finalize
static int pack_linear(moge_engine* e, const std::string& key, int N, int K, int Kpad, void** out, cudaStream_t st) {
    const RawWeight* w;
    MG_TRY(get_raw(e, key, &w, {}));
    if (static_cast<int64_t>(w->numel) != static_cast<int64_t>(N) * K) return set_error("weight '%s': numel %zu != %d*%d", key.c_str(), w->numel, N, K);
    MG_TRY(e->alloc(out, static_cast<size_t>(N) * Kpad * 2));
    return launch_cast_2d(w->p, MOGE_F32, *out, e->bf16, N, K, K, Kpad, st);
}
static int vec(moge_engine* e, const std::string& key, int n, const float** out) {
    const RawWeight* w;
    MG_TRY(get_raw(e, key, &w, {}));
    if (static_cast<int>(w->numel) != n) return set_error("weight '%s': numel %zu != %d", key.c_str(), w->numel, n);
    *out = w->p;
    return 0;
}
// bias = a + b (b optional), engine-owned
static int sum_bias(moge_engine* e, const float* a, const float* b, int n, float** out, cudaStream_t st) {
    MG_TRY(e->alloc(reinterpret_cast<void**>(out), static_cast<size_t>(n) * 4));
    vec_combine_kernel<<<(n + 255) / 256, 256, 0, st>>>(*out, a, 1, b, n);
    CUDA_TRY(cudaGetLastError());
    return 0;
}

// 3x3 conv (Cout,Cin,3,3) [+ aux 1x1 (Cout,Caux,1,1)] [+ UV 1x1 (Cout,2,1,1)] -> ConvW
static int pack_conv3(moge_engine* e, const std::string& wkey, int Cout, int Cin, const std::string& in_key, int Caux,
                      bool uv, ConvW* cw, cudaStream_t st, bool up2 = false) {
    const RawWeight* w;
    MG_TRY(get_raw(e, wkey + ".weight", &w, {Cout, Cin, 3, 3}));
    const float* b;
    MG_TRY(vec(e, wkey + ".bias", Cout, &b));
    if (Cin % 64) return set_error("conv '%s': C_in=%d must be a multiple of 64", wkey.c_str(), Cin);
    const float* wsrc = w->p;
    int Nrows = Cout;
    if (up2) {      // bilinear x2 folded into the conv: 4 output phases, run on the low-resolution grid (pack.cu)
        float* wexp;
        MG_TRY(e->alloc_temp(reinterpret_cast<void**>(&wexp), static_cast<size_t>(4) * Cout * Cin * 9 * 4));
        MG_TRY(launch_up2_expand(w->p, wexp, Cout, Cin, st));
        wsrc = wexp;
        Nrows = 4 * Cout;
    }
    cw->N = Nrows; cw->cin = Cin; cw->caux = Caux; cw->taps = 9;
    cw->Ktot = 9 * Cin + Caux;
    MG_TRY(e->alloc(&cw->w, static_cast<size_t>(Nrows) * cw->Ktot * 2));
    MG_TRY(launch_pack_conv(wsrc, cw->w, e->bf16, Nrows, Cin, 9, cw->Ktot, 0, st));
    const float* b_in = nullptr;
    if (!in_key.empty()) {
        const RawWeight* wi;
        if (uv) {
            MG_TRY(get_raw(e, in_key + ".weight", &wi, {Cout, 2, 1, 1}));
            MG_TRY(e->alloc(reinterpret_cast<void**>(&cw->wu), Cout * 4));
            MG_TRY(e->alloc(reinterpret_cast<void**>(&cw->wv), Cout * 4));
            vec_combine_kernel<<<(Cout + 255) / 256, 256, 0, st>>>(cw->wu, wi->p, 2, nullptr, Cout);
            vec_combine_kernel<<<(Cout + 255) / 256, 256, 0, st>>>(cw->wv, wi->p + 1, 2, nullptr, Cout);
        } else {
            if (Caux % 64) return set_error("input block '%s': C=%d must be a multiple of 64", in_key.c_str(), Caux);
            MG_TRY(get_raw(e, in_key + ".weight", &wi, {Cout, Caux, 1, 1}));
            MG_TRY(launch_pack_conv(wi->p, cw->w, e->bf16, Cout, Caux, 1, cw->Ktot, 9 * Cin, st));
        }
        MG_TRY(vec(e, in_key + ".bias", Cout, &b_in));
    }
    return sum_bias(e, b, b_in, Cout, &cw->bias, st);
}

// waux: the [8, 32] map from the neck's last-level map to the heads' output components (points xyz | normal xyz | mask logit |
// pad).  A head writes its [ncomp, 32] rows (output block o last-level input block) at `waux`; the neck reads all 8 rows.
static int pack_stack(moge_engine* e, const std::string& name, const moge_stack_config_t& sc, bool is_neck, StackW* sw,
                      cudaStream_t st, float* waux) {
    const int L = sc.num_levels;
    sw->res.assign(L, {});
    sw->convT.assign(L, ConvW());
    sw->post.assign(L, ConvW());
    const int* C = sc.dim_res_blocks;
    if (!is_neck) {
        // level-0 input block: 1x1 conv C0 -> C0 on the neck's level-0 output
        if (sc.dim_in[0] <= 0) return set_error("%s: level-0 input block required", name.c_str());
        const RawWeight* w;
        MG_TRY(get_raw(e, name + ".input_blocks.0.weight", &w, {C[0], sc.dim_in[0], 1, 1}));
        if (sc.dim_in[0] % 64) return set_error("%s: level-0 C_in=%d must be a multiple of 64", name.c_str(), sc.dim_in[0]);
        ConvW& cw = sw->in0;
        cw.N = C[0]; cw.cin = sc.dim_in[0]; cw.taps = 1; cw.Ktot = sc.dim_in[0];
        MG_TRY(e->alloc(&cw.w, static_cast<size_t>(cw.N) * cw.Ktot * 2));
        MG_TRY(launch_pack_conv(w->p, cw.w, e->bf16, cw.N, cw.cin, 1, cw.Ktot, 0, st));
        const float* b;
        MG_TRY(vec(e, name + ".input_blocks.0.bias", C[0], &b));
        MG_TRY(sum_bias(e, b, nullptr, C[0], &cw.bias, st));
    }
    for (int l = 0; l < L; ++l) {
        const bool last = (l == L - 1);
        if (sc.dim_out[l] > 0 && !(last && !is_neck)) return set_error("%s: output block at level %d unsupported", name.c_str(), l);
        for (int r = 0; r < sc.num_res_blocks[l]; ++r) {
            if (last && !is_neck) return set_error("%s: residual blocks at the last head level unsupported", name.c_str());
            for (int k : {2, 5}) {
                ConvW cw;
                MG_TRY(pack_conv3(e, name + ".res_blocks." + std::to_string(l) + "." + std::to_string(r) + ".layers." + std::to_string(k),
                                  C[l], C[l], "", 0, false, &cw, st));
                sw->res[l].push_back(cw);
            }
        }
        if (last) break;
        const std::string rs = name + ".resamplers." + std::to_string(l);
        const std::string in_key = sc.dim_in[l + 1] > 0 ? name + ".input_blocks." + std::to_string(l + 1) : std::string();
        const bool fold_head_out = !is_neck && (l + 1 == L - 1);
        int conv_cin;
        if (sc.resamplers[l] == MOGE_RESAMPLE_CONV_TRANSPOSE) {
            const RawWeight* w;
            MG_TRY(get_raw(e, rs + ".0.weight", &w, {C[l], C[l + 1], 2, 2}));
            if (C[l] % 64 || C[l + 1] % 32) return set_error("%s: convT %d->%d channel counts unsupported", name.c_str(), C[l], C[l + 1]);
            ConvW& ct = sw->convT[l];
            ct.N = 4 * C[l + 1]; ct.cin = C[l]; ct.taps = 1; ct.Ktot = C[l];
            MG_TRY(e->alloc(&ct.w, static_cast<size_t>(ct.N) * ct.Ktot * 2));
            MG_TRY(launch_pack_convT(w->p, ct.w, e->bf16, C[l], C[l + 1], st));
            const float* b;
            MG_TRY(vec(e, rs + ".0.bias", C[l + 1], &b));
            MG_TRY(sum_bias(e, b, nullptr, C[l + 1], &ct.bias, st));
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
                    const int Cn = C[l + 1], K9 = conv_cin * 9;
                    const RawWeight *wc, *wi;
                    const float *bc, *bi;
                    MG_TRY(get_raw(e, rs + ".1.weight", &wc, {Cn, conv_cin, 3, 3}));
                    MG_TRY(vec(e, rs + ".1.bias", Cn, &bc));
                    MG_TRY(get_raw(e, in_key + ".weight", &wi, {Cn, 2, 1, 1}));
                    MG_TRY(vec(e, in_key + ".bias", Cn, &bi));
                    float *wexp, *wfold, *bsum, *wuv;
                    MG_TRY(e->alloc_temp(reinterpret_cast<void**>(&wexp), static_cast<size_t>(4) * Cn * K9 * 4));
                    MG_TRY(launch_up2_expand(wc->p, wexp, Cn, conv_cin, st));                    // rows (phase, channel)
                    MG_TRY(e->alloc_temp(reinterpret_cast<void**>(&wfold), static_cast<size_t>(32) * K9 * 4));
                    for (int ph = 0; ph < 4; ++ph)
                        MG_TRY(launch_sgemm(waux, Cn, wexp + static_cast<size_t>(ph) * Cn * K9, K9, wfold + static_cast<size_t>(ph) * 8 * K9, K9, 8, K9, Cn, 0, st));
                    ConvW& no = sw->neckout;
                    no.N = 32; no.cin = conv_cin; no.taps = 9; no.Ktot = K9;
                    MG_TRY(e->alloc(&no.w, static_cast<size_t>(32) * K9 * 2));
                    MG_TRY(launch_pack_conv(wfold, no.w, e->bf16, 32, conv_cin, 9, K9, 0, st));
                    MG_TRY(sum_bias(e, bc, bi, Cn, &bsum, st));
                    MG_TRY(e->alloc(reinterpret_cast<void**>(&no.bias), 8 * 4));
                    MG_TRY(launch_sgemm(waux, Cn, bsum, 1, no.bias, 1, 8, 1, Cn, 0, st));
                    MG_TRY(e->alloc_temp(reinterpret_cast<void**>(&wuv), 2 * Cn * 4));
                    vec_combine_kernel<<<(Cn + 255) / 256, 256, 0, st>>>(wuv, wi->p, 2, nullptr, Cn);
                    vec_combine_kernel<<<(Cn + 255) / 256, 256, 0, st>>>(wuv + Cn, wi->p + 1, 2, nullptr, Cn);
                    CUDA_TRY(cudaGetLastError());
                    MG_TRY(e->alloc(reinterpret_cast<void**>(&no.wu), 8 * 4));
                    MG_TRY(e->alloc(reinterpret_cast<void**>(&no.wv), 8 * 4));
                    MG_TRY(launch_sgemm(waux, Cn, wuv, 1, no.wu, 1, 8, 1, Cn, 0, st));
                    MG_TRY(launch_sgemm(waux, Cn, wuv + Cn, 1, no.wv, 1, 8, 1, Cn, 0, st));
                    continue;
                }
                MG_TRY(pack_conv3(e, rs + ".1", C[l + 1], conv_cin, in_key, 0, true, &sw->post[l], st, sc.resamplers[l] == MOGE_RESAMPLE_BILINEAR));
            } else {
                if (sc.dim_in[l + 1] <= 0) return set_error("%s: input block at level %d required", name.c_str(), l + 1);
                if (sc.resamplers[l] == MOGE_RESAMPLE_BILINEAR) return set_error("%s: a bilinear resampler is supported at the last level only", name.c_str());
                MG_TRY(pack_conv3(e, rs + ".1", C[l + 1], conv_cin, in_key, sc.dim_in[l + 1], false, &sw->post[l], st));
            }
        } else {
            // head tail: conv3x3 (conv_cin -> 32) + in_block(neck_last 32 -> 32) then output block 32 -> ncomp, no
            // nonlinearity in between  =>  one 3x3 conv conv_cin -> ncomp plus a [ncomp,32] map of the neck map.
            const int Cl = C[L - 1], nc = sc.dim_out[L - 1];
            if (Cl != 32 || sc.dim_in[L - 1] != 32 || nc <= 0 || nc > 3 || conv_cin % 64)
                return set_error("%s: last level must be 32 channels with a 1..3 channel output block", name.c_str());
            const RawWeight *wc, *w4, *wo;
            const float *bc, *b4, *bo;
            MG_TRY(get_raw(e, rs + ".1.weight", &wc, {Cl, conv_cin, 3, 3}));
            MG_TRY(vec(e, rs + ".1.bias", Cl, &bc));
            MG_TRY(get_raw(e, in_key + ".weight", &w4, {Cl, 32, 1, 1}));
            MG_TRY(vec(e, in_key + ".bias", Cl, &b4));
            MG_TRY(get_raw(e, name + ".output_blocks." + std::to_string(L - 1) + ".weight", &wo, {nc, Cl, 1, 1}));
            MG_TRY(vec(e, name + ".output_blocks." + std::to_string(L - 1) + ".bias", nc, &bo));
            float *tmpw, *bsum, *bfold;
            const int K9 = conv_cin * 9;
            MG_TRY(e->alloc_temp(reinterpret_cast<void**>(&tmpw), static_cast<size_t>(16) * K9 * 4));
            CUDA_TRY(cudaMemsetAsync(tmpw, 0, static_cast<size_t>(16) * K9 * 4, st));
            if (sc.resamplers[l] != MOGE_RESAMPLE_BILINEAR) return set_error("%s: the last resampler must be bilinear", name.c_str());
            MG_TRY(launch_sgemm(wo->p, Cl, wc->p, K9, tmpw, K9, nc, K9, Cl, 0, st));          // [nc, (ci,tap)] = (nc,Cin,3,3)
            float* wexp;                                                                       // (4*nc,Cin,3,3), rows (phase, comp)
            MG_TRY(e->alloc_temp(reinterpret_cast<void**>(&wexp), static_cast<size_t>(16) * K9 * 4));
            CUDA_TRY(cudaMemsetAsync(wexp, 0, static_cast<size_t>(16) * K9 * 4, st));
            MG_TRY(launch_up2_expand(tmpw, wexp, nc, conv_cin, st));
            ConvW& ho = sw->headout;
            ho.N = 16; ho.cin = conv_cin; ho.taps = 9; ho.Ktot = K9;
            MG_TRY(e->alloc(&ho.w, static_cast<size_t>(16) * K9 * 2));
            MG_TRY(launch_pack_conv(wexp, ho.w, e->bf16, 16, conv_cin, 9, K9, 0, st));
            MG_TRY(launch_sgemm(wo->p, Cl, w4->p, 32, waux, 32, nc, 32, Cl, 0, st));            // [nc, 32]
            MG_TRY(sum_bias(e, bc, b4, Cl, &bsum, st));
            MG_TRY(e->alloc(reinterpret_cast<void**>(&bfold), 16 * 4));
            CUDA_TRY(cudaMemsetAsync(bfold, 0, 16 * 4, st));
            MG_TRY(launch_sgemm(wo->p, Cl, bsum, 1, bfold, 1, nc, 1, Cl, 0, st));
            vec_combine_kernel<<<1, 32, 0, st>>>(bfold, bfold, 1, bo, nc);
            CUDA_TRY(cudaGetLastError());
            ho.bias = bfold;
            sw->ncomp = nc;
        }
    }
    return 0;
}

static int finalize_encoder(moge_engine* e, cudaStream_t st) {
    const moge_config_t& c = e->cfg;
    const int D = c.embed_dim;
    const std::string bb = e->v1 ? "backbone." : "encoder.backbone.";
    MG_TRY(pack_linear(e, bb + "patch_embed.proj.weight", D, 588, 592, &e->w_patch, st));
    MG_TRY(vec(e, bb + "patch_embed.proj.bias", D, &e->patch_bias));
    MG_TRY(vec(e, bb + "pos_embed", (1 + 37 * 37) * D, &e->pos_embed));
    MG_TRY(vec(e, bb + "cls_token", D, &e->cls_token));
    MG_TRY(vec(e, bb + "norm.weight", D, &e->norm_g));
    MG_TRY(vec(e, bb + "norm.bias", D, &e->norm_b));
    e->blk.resize(c.depth);
    for (int i = 0; i < c.depth; ++i) {
        const std::string p = bb + "blocks." + std::to_string(i) + ".";
        moge_engine::Blk& b = e->blk[i];
        MG_TRY(pack_linear(e, p + "attn.proj.weight", D, D, D, &b.wproj, st));
        MG_TRY(pack_linear(e, p + "mlp.fc2.weight", D, 4 * D, 4 * D, &b.wfc2, st));
        const float *bqkv, *bfc1, *ln1g, *ln1b, *ln2g, *ln2b;
        MG_TRY(vec(e, p + "attn.qkv.bias", 3 * D, &bqkv));
        MG_TRY(vec(e, p + "attn.proj.bias", D, &b.bproj));
        MG_TRY(vec(e, p + "mlp.fc1.bias", 4 * D, &bfc1));
        MG_TRY(vec(e, p + "mlp.fc2.bias", D, &b.bfc2));
        MG_TRY(vec(e, p + "ls1.gamma", D, &b.g1));
        MG_TRY(vec(e, p + "ls2.gamma", D, &b.g2));
        MG_TRY(vec(e, p + "norm1.weight", D, &ln1g));
        MG_TRY(vec(e, p + "norm1.bias", D, &ln1b));
        MG_TRY(vec(e, p + "norm2.weight", D, &ln2g));
        MG_TRY(vec(e, p + "norm2.bias", D, &ln2b));
        const RawWeight *wq, *wf;
        MG_TRY(get_raw(e, p + "attn.qkv.weight", &wq, {}));
        MG_TRY(get_raw(e, p + "mlp.fc1.weight", &wf, {}));
        MG_TRY(e->alloc(&b.wqkv_ln, static_cast<size_t>(3 * D) * D * 2));
        MG_TRY(e->alloc(&b.wfc1_ln, static_cast<size_t>(4 * D) * D * 2));
        MG_TRY(e->alloc(reinterpret_cast<void**>(&b.b_qkv_ln), static_cast<size_t>(3 * D) * 4));
        MG_TRY(e->alloc(reinterpret_cast<void**>(&b.b_fc1_ln), static_cast<size_t>(4 * D) * 4));
        MG_TRY(launch_ln_fold(wq->p, ln1g, ln1b, bqkv, 3 * D, D, D, b.wqkv_ln, b.b_qkv_ln, e->bf16, st));
        MG_TRY(launch_ln_fold(wf->p, ln2g, ln2b, bfc1, 4 * D, D, D, b.wfc1_ln, b.b_fc1_ln, e->bf16, st));
    }
    return 0;
}

static int finalize_v2_decoder(moge_engine* e, cudaStream_t st) {
    const moge_config_t& c = e->cfg;
    const int D = c.embed_dim;
    // ---- fold: neck.input_blocks.0 o (sum_j output_projections.j)  ->  one GEMM over the concatenated taps
    {
        const int C0 = c.neck.dim_res_blocks[0], Do = c.dim_out, nt = c.num_taps;
        if (c.neck.dim_in[0] != Do + 2) return set_error("neck.dim_in[0]=%d must be encoder.dim_out+2=%d", c.neck.dim_in[0], Do + 2);
        const RawWeight* w0;
        MG_TRY(get_raw(e, "neck.input_blocks.0.weight", &w0, {C0, Do + 2, 1, 1}));
        const float* b0;
        MG_TRY(vec(e, "neck.input_blocks.0.bias", C0, &b0));
        float *wf, *bf, *bp;
        MG_TRY(e->alloc_temp(reinterpret_cast<void**>(&wf), static_cast<size_t>(C0) * nt * D * 4));
        MG_TRY(e->alloc(reinterpret_cast<void**>(&bf), C0 * 4));
        MG_TRY(e->alloc_temp(reinterpret_cast<void**>(&bp), Do * 4));
        CUDA_TRY(cudaMemsetAsync(bp, 0, Do * 4, st));
        for (int j = 0; j < nt; ++j) {
            const RawWeight* pj;
            MG_TRY(get_raw(e, "encoder.output_projections." + std::to_string(j) + ".weight", &pj, {Do, D, 1, 1}));
            const float* bj;
            MG_TRY(vec(e, "encoder.output_projections." + std::to_string(j) + ".bias", Do, &bj));
            MG_TRY(launch_sgemm(w0->p, Do + 2, pj->p, D, wf + static_cast<size_t>(j) * D, nt * D, C0, D, Do, 0, st));
            vec_combine_kernel<<<(Do + 255) / 256, 256, 0, st>>>(bp, bp, 1, bj, Do);
        }
        MG_TRY(launch_sgemm(w0->p, Do + 2, bp, 1, bf, 1, C0, 1, Do, 0, st));
        vec_combine_kernel<<<(C0 + 255) / 256, 256, 0, st>>>(bf, bf, 1, b0, C0);
        ConvW& f = e->fold0;
        f.N = C0; f.Ktot = nt * D; f.taps = 1; f.cin = nt * D;
        MG_TRY(e->alloc(&f.w, static_cast<size_t>(C0) * f.Ktot * 2));
        MG_TRY(launch_cast_2d(wf, MOGE_F32, f.w, e->bf16, C0, f.Ktot, f.Ktot, f.Ktot, st));
        f.bias = bf;
        MG_TRY(e->alloc(reinterpret_cast<void**>(&f.wu), C0 * 4));
        MG_TRY(e->alloc(reinterpret_cast<void**>(&f.wv), C0 * 4));
        vec_combine_kernel<<<(C0 + 255) / 256, 256, 0, st>>>(f.wu, w0->p + Do, Do + 2, nullptr, C0);
        vec_combine_kernel<<<(C0 + 255) / 256, 256, 0, st>>>(f.wv, w0->p + Do + 1, Do + 2, nullptr, C0);
        CUDA_TRY(cudaGetLastError());
    }
    // the heads' last levels first: they give the map through which the neck's last level is folded (EPI_NECKOUT)
    float* waux;
    MG_TRY(e->alloc_temp(reinterpret_cast<void**>(&waux), 8 * 32 * 4));
    CUDA_TRY(cudaMemsetAsync(waux, 0, 8 * 32 * 4, st));
    const int row_of[3] = {0, 3, 6};          // points xyz | normal xyz | mask logit | pad
    for (int i = 0; i < 3; ++i)
        if (head_cfg(e, i)->present) MG_TRY(pack_stack(e, head_name(i), *head_cfg(e, i), false, &e->heads[i], st, waux + row_of[i] * 32));
    MG_TRY(pack_stack(e, "neck", c.neck, true, &e->neck, st, waux));
    for (int l = 0; l < c.scale_head_layers; ++l) {
        const float *w, *b;
        MG_TRY(vec(e, "scale_head." + std::to_string(2 * l) + ".weight", c.scale_head_dims[l] * c.scale_head_dims[l + 1], &w));
        MG_TRY(vec(e, "scale_head." + std::to_string(2 * l) + ".bias", c.scale_head_dims[l + 1], &b));
        e->mlp_w.push_back(w);
        e->mlp_b.push_back(b);
    }
    return 0;
}

// ---- MoGe-1 decoder (keys head.*, v1.py:61-142).  The small folds are done on the host from copies of the fp32 staging weights.
static int to_host(const RawWeight* w, size_t off, size_t n, std::vector<float>* out) {
    out->resize(n);
    CUDA_TRY(cudaMemcpy(out->data(), w->p + off, n * 4, cudaMemcpyDeviceToHost));
    return 0;
}
static int to_dev(moge_engine* e, const std::vector<float>& v, float** out) {
    MG_TRY(e->alloc(reinterpret_cast<void**>(out), v.size() * 4));
    CUDA_TRY(cudaMemcpy(*out, v.data(), v.size() * 4, cudaMemcpyHostToDevice));
    return 0;
}

static int finalize_v1(moge_engine* e, cudaStream_t st) {
    const moge_v1_config_t& c = e->v1cfg;
    const int D = c.embed_dim, nt = c.num_taps, P = c.dim_proj;
    CUDA_TRY(cudaStreamSynchronize(st));       // the staging copies are written on st; the host reads some of them below
    V1W& v = e->v1w;
    // V4: sum_j projects.j(tap_j) = one GEMM over the concatenated taps [B*T, nt*D] with the summed bias
    ConvW& pj = v.proj;
    pj.N = P; pj.cin = nt * D; pj.taps = 1; pj.Ktot = nt * D;
    MG_TRY(e->alloc(&pj.w, static_cast<size_t>(P) * pj.Ktot * 2));
    MG_TRY(e->alloc(reinterpret_cast<void**>(&pj.bias), P * 4));
    CUDA_TRY(cudaMemsetAsync(pj.bias, 0, P * 4, st));
    float* wcat32;                             // [P, nt*D] fp32: tap j's weight in columns j*D ..
    MG_TRY(e->alloc_temp(reinterpret_cast<void**>(&wcat32), static_cast<size_t>(P) * pj.Ktot * 4));
    for (int j = 0; j < nt; ++j) {
        const std::string k = "head.projects." + std::to_string(j);
        const RawWeight* w;
        const float* b;
        MG_TRY(get_raw(e, k + ".weight", &w, {P, D, 1, 1}));
        MG_TRY(vec(e, k + ".bias", P, &b));
        CUDA_TRY(cudaMemcpy2DAsync(wcat32 + static_cast<size_t>(j) * D, static_cast<size_t>(pj.Ktot) * 4, w->p, static_cast<size_t>(D) * 4,
                                   static_cast<size_t>(D) * 4, P, cudaMemcpyDeviceToDevice, st));
        vec_combine_kernel<<<(P + 255) / 256, 256, 0, st>>>(pj.bias, pj.bias, 1, b, P);
        CUDA_TRY(cudaGetLastError());
    }
    MG_TRY(launch_cast_2d(wcat32, MOGE_F32, pj.w, e->bf16, P, pj.Ktot, pj.Ktot, pj.Ktot, st));
    int cin = P;
    v.lv.assign(c.num_levels, V1Level());
    for (int l = 0; l < c.num_levels; ++l) {
        const int Co = c.dim_upsample[l], Hd = c.hidden_mult * Co;
        const std::string pre = "head.upsample_blocks." + std::to_string(l) + ".";
        V1Level& L = v.lv[l];
        // V5: ConvTranspose2d(cin + 2 -> Co): rows 0..cin-1 through the GEMM, the two UV rows as the input-grid term
        const RawWeight* wt;
        const float* bt;
        MG_TRY(get_raw(e, pre + "0.0.weight", &wt, {cin + 2, Co, 2, 2}));
        MG_TRY(vec(e, pre + "0.0.bias", Co, &bt));
        L.convT.N = 4 * Co; L.convT.cin = cin; L.convT.taps = 1; L.convT.Ktot = cin;
        MG_TRY(e->alloc(&L.convT.w, static_cast<size_t>(4) * Co * cin * 2));
        MG_TRY(launch_pack_convT(wt->p, L.convT.w, e->bf16, cin, Co, st));
        MG_TRY(sum_bias(e, bt, nullptr, Co, &L.convT.bias, st));
        MG_TRY(e->alloc(reinterpret_cast<void**>(&L.wuv), static_cast<size_t>(8) * Co * 4));
        MG_TRY(launch_pack_convT_uv(wt->p, cin, Co, L.wuv, st));
        MG_TRY(pack_conv3(e, pre + "0.1", Co, Co, "", 0, false, &L.conv, st));
        for (int r = 0; r < c.num_res_blocks; ++r) {
            const std::string rp = pre + std::to_string(1 + r) + ".layers.";
            V1Res R;
            MG_TRY(vec(e, rp + "0.weight", Co, &R.g1));
            MG_TRY(vec(e, rp + "0.bias", Co, &R.b1));
            MG_TRY(pack_conv3(e, rp + "2", Hd, Co, "", 0, false, &R.c1, st));
            MG_TRY(vec(e, rp + "3.weight", Hd, &R.g2));
            MG_TRY(vec(e, rp + "3.bias", Hd, &R.b2));
            MG_TRY(pack_conv3(e, rp + "5", Co, Hd, "", 0, false, &R.c2, st));
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
        const RawWeight *wc, *bc, *wo, *bo;
        MG_TRY(get_raw(e, ob + "0.weight", &wc, {lc, cin + 2, 3, 3}));
        MG_TRY(get_raw(e, ob + "0.bias", &bc, {lc}));
        MG_TRY(get_raw(e, ob + "2.weight", &wo, {nout[k], lc, 1, 1}));
        MG_TRY(get_raw(e, ob + "2.bias", &bo, {nout[k]}));
        std::vector<float> hw, hb, hwo, hbo;
        MG_TRY(to_host(wc, 0, wc->numel, &hw));
        MG_TRY(to_host(bc, 0, bc->numel, &hb));
        MG_TRY(to_host(wo, 0, wo->numel, &hwo));
        MG_TRY(to_host(bo, 0, bo->numel, &hbo));
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
    MG_TRY(to_dev(e, params, &v.wout));
    float* wcat_dev;
    MG_TRY(e->alloc_temp(reinterpret_cast<void**>(&wcat_dev), wcat.size() * 4));
    CUDA_TRY(cudaMemcpy(wcat_dev, wcat.data(), wcat.size() * 4, cudaMemcpyHostToDevice));
    ConvW& oc = v.out;
    oc.N = 2 * lc; oc.cin = cin; oc.taps = 9; oc.Ktot = 9 * cin;
    MG_TRY(e->alloc(&oc.w, static_cast<size_t>(oc.N) * oc.Ktot * 2));
    MG_TRY(launch_pack_conv(wcat_dev, oc.w, e->bf16, oc.N, cin, 9, oc.Ktot, 0, st));
    MG_TRY(to_dev(e, bcat, &oc.bias));
    return 0;
}

static int finalize(moge_engine* e, cudaStream_t st) {
    MG_TRY(finalize_encoder(e, st));
    MG_TRY(e->v1 ? finalize_v1(e, st) : finalize_v2_decoder(e, st));
    CUDA_TRY(cudaStreamSynchronize(st));
    for (void* t : e->temps) cudaFree(t);
    e->temps.clear();
    // release the fp32 staging copies of the big matrices (vectors stay: kernels read them directly)
    for (auto& kv : e->raw) {
        const bool keep = kv.second.shape.size() <= 1 || kv.first.find("pos_embed") != std::string::npos ||
                          kv.first.find("cls_token") != std::string::npos || kv.first.rfind("scale_head.", 0) == 0;
        if (!keep && kv.second.p) { cudaFree(kv.second.p); kv.second.p = nullptr; }
    }
    e->finalized = true;
    return 0;
}

// ------------------------------------------------------------------------------------------------ planning
struct WsAlloc {
    uint8_t* base; size_t off = 0;
    explicit WsAlloc(void* b) : base(static_cast<uint8_t*>(b)) {}
    void* take(size_t bytes) {
        off = (off + 1023) & ~static_cast<size_t>(1023);
        void* p = base ? base + off : nullptr;
        off += bytes;
        return p;
    }
};

static Level level_geom(int h, int w, int l) {
    Level g;
    g.H = h << l; g.W = w << l;
    g.Hp = std::max(g.H + 2, TILE_PH);
    g.Wp = std::max(g.W + 2, TILE_PW);
    return g;
}
static size_t map_bytes(const Level& g, int B, int C) { return static_cast<size_t>(B) * g.Hp * g.Wp * C * 2; }

// conv-type launch on padded NHWC maps. src/aux/skip/out buffers live in the workspace.
static int add_conv(moge_engine* e, Plan* pl, const ConvW& cw, const void* src, const void* aux, const Level& gs, int B,
                    int epi, void* out_raw, void* out_relu, const void* skip, const Level& go, int out_ch, bool shuffle,
                    bool uv, float su, float sv, const std::string& name, int ncomp = 0, void* out2 = nullptr) {
    GemmLaunch g;
    MG_TRY(gemm_conv(&g, e->bf16, cw, src, aux, gs, B, epi, out_raw, out_relu, skip, go, out_ch, shuffle, uv, su, sv, ncomp, out2));
    const double px = static_cast<double>(B) * gs.H * gs.W;
    const double flops = 2.0 * px * cw.N * cw.Ktot;
    double bytes = px * cw.cin * 2 + px * cw.caux * 2 + static_cast<double>(cw.N) * cw.Ktot * 2;
    // 4 output pixels per low-res pixel, each read (the neck's part) and written
    if (epi == EPI_HEADOUT) bytes += 2 * (4 * px * (ncomp == 1 ? 4 : 16));
    else if (epi == EPI_NECKOUT) bytes += 4 * px * ((out_raw ? 16 : 0) + (out_relu ? 16 : 0) + (out2 ? 4 : 0));
    else bytes += px * cw.N * 2 * ((out_raw ? 1 : 0) + (out_relu ? 1 : 0)) + (skip ? px * cw.N * 2 : 0);
    const int sms = e->num_sms;
    pl->ops.add([=](cudaStream_t st) { return launch_gemm(g, sms, st); }, name, flops, bytes);
    return 0;
}

// Linear over row-major A [M, K] with the engine's packed (dense [N, K]) weight W; trailing arguments as in gemm_linear.
static int add_linear(moge_engine* e, Plan* pl, const void* A, int M, int K, const void* W, int N, int epi, void* out, const float* bias,
                      const float* v1, int ldo, const std::string& name, const LnIO* ln = nullptr, const Level* grid = nullptr,
                      void* out_relu = nullptr, const float* v2 = nullptr, float su = 0.f, float sv = 0.f) {
    GemmLaunch g;
    MG_TRY(gemm_linear(&g, e->bf16, A, M, K, W, K, N, epi, out, ldo, bias, v1, ln, grid, out_relu, v2, su, sv));
    const double flops = 2.0 * M * static_cast<double>(N) * K;
    double bytes = static_cast<double>(M) * K * 2 + static_cast<double>(N) * K * 2;
    bytes += (epi == EPI_RESID) ? static_cast<double>(M) * N * 8 : (epi == EPI_PATCH) ? static_cast<double>(M) * N * 4 + static_cast<double>(g.p.T) * N * 4
                                                                                      : static_cast<double>(M) * N * 2;
    if (ln && ln->x16) bytes += static_cast<double>(M) * N * 2;
    const int sms = e->num_sms;
    pl->ops.add([=](cudaStream_t st) { return launch_gemm(g, sms, st); }, name, flops, bytes);
    return 0;
}

struct StackBufs {     // per-level scratch maps of one ConvStack
    std::vector<void*> x_raw, x_relu, y_relu, t_up;
};

static int plan_stack(moge_engine* e, Plan* pl, const char* sname, const moge_stack_config_t& sc, const StackW& sw, bool is_neck, int B, int h,
                      int w, float su, float sv, const StackBufs& sb, const std::vector<void*>& neck_out, void* x0_raw, void* x0_relu,
                      void* lowres_out, void* const* neck_lowres = nullptr) {
    const int L = sc.num_levels;
    const int* C = sc.dim_res_blocks;
    void* x_raw = x0_raw;
    void* x_relu = x0_relu;
    auto nm = [&](const char* kind, int l) { return std::string(kind) + "." + sname + ".l" + std::to_string(l); };
    for (int l = 0; l < L; ++l) {
        const Level g = level_geom(h, w, l);
        const int nres = sc.num_res_blocks[l];
        for (int r = 0; r < nres; ++r) {
            // y = conv3(relu(x)) -> only relu(y) is ever consumed
            MG_TRY(add_conv(e, pl, sw.res[l][2 * r], x_relu, nullptr, g, B, EPI_DEC, nullptr, sb.y_relu[l], nullptr, g, C[l], false, false, 0, 0, nm("conv3x3.res_a", l)));
            // x = x + conv3(relu(y))
            void* nraw = (x_raw == sb.x_raw[l]) ? sb.t_up[l] : sb.x_raw[l];     // ping-pong between two raw maps
            MG_TRY(add_conv(e, pl, sw.res[l][2 * r + 1], sb.y_relu[l], nullptr, g, B, EPI_DEC, nraw, (r + 1 < nres) ? x_relu : nullptr, x_raw, g, C[l], false, false, 0, 0, nm("conv3x3.res_b", l)));
            x_raw = nraw;
        }
        if (is_neck) const_cast<std::vector<void*>&>(neck_out)[l] = x_raw;
        if (l == L - 1) break;
        const Level gn = level_geom(h, w, l + 1);
        const bool tail = !is_neck && (l + 1 == L - 1);
        const void* conv_src;
        if (sc.resamplers[l] == MOGE_RESAMPLE_CONV_TRANSPOSE) {
            MG_TRY(add_conv(e, pl, sw.convT[l], x_raw, nullptr, g, B, EPI_DEC, sb.t_up[l + 1], nullptr, nullptr, gn, C[l + 1], true, false, 0, 0, nm("convT", l)));
            conv_src = sb.t_up[l + 1];
        } else {
            // bilinear x2 + 3x3 conv run as ONE low-resolution conv with 4 output phases (weights expanded at load time)
            const bool need_relu_b = sc.num_res_blocks[l + 1] > 0;
            if (tail) {
                MG_TRY(add_conv(e, pl, sw.headout, x_raw, nullptr, g, B, EPI_HEADOUT, lowres_out, nullptr, nullptr, gn, 0, false,
                                false, 0, 0, nm("conv3x3up2.headout", l + 1), sw.ncomp));
                break;
            }
            if (is_neck && l + 1 == L - 1) {
                // the neck's last level goes straight into the heads' output maps (folded through their last input/output blocks)
                MG_TRY(add_conv(e, pl, sw.neckout, x_raw, nullptr, g, B, EPI_NECKOUT, neck_lowres[0], neck_lowres[1], nullptr, gn, 0, false, true, su, sv,
                                nm("conv3x3up2.neckout", l + 1), 0, neck_lowres[2]));
                break;
            }
            MG_TRY(add_conv(e, pl, sw.post[l], x_raw, nullptr, g, B, EPI_DEC, sb.x_raw[l + 1], need_relu_b ? sb.x_relu[l + 1] : nullptr, nullptr, gn,
                            C[l + 1], true, is_neck, su, sv, nm("conv3x3up2.post", l + 1)));
            x_raw = sb.x_raw[l + 1];
            x_relu = sb.x_relu[l + 1];
            continue;
        }
        if (tail) return set_error("%s: the last resampler must be bilinear", sname);
        const bool need_relu = sc.num_res_blocks[l + 1] > 0;
        MG_TRY(add_conv(e, pl, sw.post[l], conv_src, is_neck ? nullptr : neck_out[l + 1], gn, B, EPI_DEC, sb.x_raw[l + 1],
                        need_relu ? sb.x_relu[l + 1] : nullptr, nullptr, gn, C[l + 1], false, is_neck, su, sv, nm("conv3x3.post", l + 1)));
        x_raw = sb.x_raw[l + 1];
        x_relu = sb.x_relu[l + 1];
    }
    return 0;
}

// ---- MoGe-1 decoder (one shape group): workspace maps and launch list
struct V1Bufs {
    float *rs_tmp = nullptr, *rs_img = nullptr;     // bicubic row pass (B,3,H,rw), resized image (B,3,rh,rw)
    void* x0 = nullptr;                             // projected taps, level 0
    struct Lv { void *m0, *m1, *relu, *hraw, *hrelu; };
    std::vector<Lv> lv;                             // per upsampling level (its output grid): ping-pong maps, ReLU maps
    double2* gn_part = nullptr;
    float2* gn_stats = nullptr;
    void *full = nullptr, *fout = nullptr;          // last map resized to (rh, rw); the output conv's 64 channels there
    float4* pts = nullptr;                          // (rh, rw) points before the resize to (H, W)
    float* msk = nullptr;
};

static Level full_geom(int rh, int rw) { return Level{rh, rw, std::max(rh + 2, TILE_PH), std::max(rw + 2, TILE_PW)}; }

static void v1_alloc(moge_engine* e, const Group& g, WsAlloc& ws, V1Bufs* vb) {
    const moge_v1_config_t& c = e->v1cfg;
    const int B = g.B;
    vb->rs_tmp = static_cast<float*>(ws.take(static_cast<size_t>(B) * 3 * g.H * g.rw * 4));
    vb->rs_img = static_cast<float*>(ws.take(static_cast<size_t>(B) * 3 * g.rh * g.rw * 4));
    vb->x0 = ws.take(map_bytes(level_geom(g.h, g.w, 0), B, c.dim_proj));
    size_t part = 0, stats = 0;
    vb->lv.resize(c.num_levels);
    for (int l = 0; l < c.num_levels; ++l) {
        const Level go = level_geom(g.h, g.w, l + 1);
        const int Co = c.dim_upsample[l], Hd = c.hidden_mult * Co;
        const int G2 = c.hidden_norm == MOGE_V1_GROUP_NORM ? Hd / 32 : 1;
        V1Bufs::Lv& L = vb->lv[l];
        L.m0 = ws.take(map_bytes(go, B, Co));
        L.m1 = ws.take(map_bytes(go, B, Co));
        L.relu = ws.take(map_bytes(go, B, Co));
        L.hraw = ws.take(map_bytes(go, B, Hd));
        L.hrelu = ws.take(map_bytes(go, B, Hd));
        part = std::max({part, static_cast<size_t>(B) * gn_tiles(go.H, go.W, Co), static_cast<size_t>(B) * gn_tiles(go.H, go.W, Hd) * G2});
        stats = std::max(stats, static_cast<size_t>(B) * G2);
    }
    vb->gn_part = static_cast<double2*>(ws.take(part * 16));
    vb->gn_stats = static_cast<float2*>(ws.take(stats * 8));
    const Level gr = full_geom(g.rh, g.rw);
    vb->full = ws.take(map_bytes(gr, B, c.dim_upsample[c.num_levels - 1]));
    vb->fout = ws.take(map_bytes(gr, B, 2 * c.last_conv_channels));
    vb->pts = static_cast<float4*>(ws.take(static_cast<size_t>(B) * g.rh * g.rw * 16));
    vb->msk = static_cast<float*>(ws.take(static_cast<size_t>(B) * g.rh * g.rw * 4));
}

static int plan_v1_decoder(moge_engine* e, Plan* pl, const void* taps, const V1Bufs& vb) {
    const moge_v1_config_t& c = e->v1cfg;
    const V1W& v = e->v1w;
    const Group& g = pl->groups[0];
    const int B = g.B, H = g.H, W = g.W, h = g.h, w = g.w, rh = g.rh, rw = g.rw;
    const bool bf16 = e->bf16;
    // every UV plane of the head has the aspect of the resized image (v1.py:125, 133)
    const float aspect = static_cast<float>(rw) / rh;
    const float su = aspect / sqrtf(1.f + aspect * aspect), sv = 1.f / sqrtf(1.f + aspect * aspect);
    const Level g0 = level_geom(h, w, 0);
    MG_TRY(add_linear(e, pl, taps, B * h * w, v.proj.Ktot, v.proj.w, v.proj.N, EPI_DEC, vb.x0, v.proj.bias, nullptr, v.proj.N, "gemm.projects",
                      nullptr, &g0));
    const void* x = vb.x0;
    double2* part = vb.gn_part;
    float2* stats = vb.gn_stats;
    auto nm = [](const char* kind, int l) { return std::string(kind) + ".l" + std::to_string(l); };
    auto add_gn = [&](const void* src, void* dst, const Level& gl, int C, int G, const float* gamma, const float* beta, int l) {
        const double px = static_cast<double>(B) * gl.H * gl.W;
        pl->ops.add([=](cudaStream_t st) { return launch_gn_stats(src, gl, B, C, G, part, stats, bf16, st); }, nm("groupnorm_stats", l), 0, px * C * 2);
        pl->ops.add([=](cudaStream_t st) { return launch_gn_relu(src, dst, gl, B, C, G, stats, gamma, beta, bf16, st); }, nm("groupnorm_relu", l), 0,
                    px * C * 4);
    };
    for (int l = 0; l < c.num_levels; ++l) {
        const V1Level& L = v.lv[l];
        const V1Bufs::Lv& m = vb.lv[l];
        const int Co = c.dim_upsample[l], Hd = c.hidden_mult * Co;
        const Level gi = level_geom(h, w, l), go = level_geom(h, w, l + 1);
        MG_TRY(add_conv(e, pl, L.convT, x, nullptr, gi, B, EPI_DEC, m.m1, nullptr, nullptr, go, Co, true, false, 0, 0, nm("convT", l)));
        const float* wuv = L.wuv;
        void* t = m.m1;
        pl->ops.add([=](cudaStream_t st) { return launch_uv_convT(t, go, B, Co, wuv, su, sv, bf16, st); }, nm("uv_convT", l), 0,
                    static_cast<double>(B) * go.H * go.W * Co * 4);
        MG_TRY(add_conv(e, pl, L.conv, m.m1, nullptr, go, B, EPI_DEC, m.m0, nullptr, nullptr, go, Co, false, false, 0, 0, nm("conv3x3", l)));
        void* xr = m.m0;
        void* other = m.m1;
        for (const V1Res& R : L.res) {
            add_gn(xr, m.relu, go, Co, 1, R.g1, R.b1, l);
            MG_TRY(add_conv(e, pl, R.c1, m.relu, nullptr, go, B, EPI_DEC, m.hraw, nullptr, nullptr, go, Hd, false, false, 0, 0, nm("conv3x3.res_a", l)));
            add_gn(m.hraw, m.hrelu, go, Hd, R.G2, R.g2, R.b2, l);
            MG_TRY(add_conv(e, pl, R.c2, m.hrelu, nullptr, go, B, EPI_DEC, other, nullptr, xr, go, Co, false, false, 0, 0, nm("conv3x3.res_b", l)));
            std::swap(xr, other);
        }
        x = xr;
    }
    // V7: bilinear resize to the resized-image grid, both output blocks' 3x3 conv, then their UV part, ReLU and 1x1 convs
    const int Cl = c.dim_upsample[c.num_levels - 1];
    const Level gl = level_geom(h, w, c.num_levels), gr = full_geom(rh, rw);
    const double pxr = static_cast<double>(B) * rh * rw;
    void* full = vb.full;
    pl->ops.add([=](cudaStream_t st) { return launch_resize_bilinear_nhwc(x, gl, full, gr, B, Cl, bf16, st); }, "resize_bilinear", 0,
                static_cast<double>(B) * gl.H * gl.W * Cl * 2 + pxr * Cl * 2);
    MG_TRY(add_conv(e, pl, v.out, vb.full, nullptr, gr, B, EPI_DEC, vb.fout, nullptr, nullptr, gr, v.out.N, false, false, 0, 0, "conv3x3.output"));
    const void* fout = vb.fout;
    const float* wout = v.wout;
    float4* pts = vb.pts;
    float* msk = vb.msk;
    pl->ops.add([=](cudaStream_t st) { return launch_v1_output(fout, gr, B, wout, su, sv, pts, msk, bf16, st); }, "output_block", 2.0 * pxr * 64 * 10,
                pxr * (64 * 2 + 20));
    // V8 (phase 2: the caller's outputs): bilinear resize to (H, W), remap; the mask stays a raw logit
    const int remap = c.remap_output;
    Plan* P = pl;
    pl->ops.add([=](cudaStream_t st) {
        return launch_head_output(pts, nullptr, msk, B, rh, rw, H, W, remap, P->groups[0].points, nullptr, P->groups[0].mask, st, false);
    }, "head_output", 0, static_cast<double>(B) * H * W * 16 + pxr * 20, 2);
    return 0;
}

// MoGe-2 decoder maps: the groups run one after the other through ONE set of maps sized for the largest group
struct V2Bufs {
    StackBufs nb, hb;                               // neck, heads
    std::vector<float4*> pts_lr, nrm_lr;            // low-resolution fp32 head outputs, per group
    std::vector<float*> msk_lr;
};

static void alloc_v2_decoder(moge_engine* e, Plan* pl, WsAlloc& ws, V2Bufs* v) {
    const moge_config_t& c = e->cfg;
    const int G = static_cast<int>(pl->groups.size());
    const int L = c.neck.num_levels;
    auto alloc_stack = [&](const moge_stack_config_t& sc, StackBufs& sb) {
        sb.x_raw.assign(L, nullptr); sb.x_relu.assign(L, nullptr); sb.y_relu.assign(L, nullptr); sb.t_up.assign(L, nullptr);
        // no level-(L-1) map: the last levels are folded into EPI_NECKOUT / EPI_HEADOUT, which write the fp32 head outputs
        for (int l = 0; l < L - 1; ++l) {
            const int Cl = sc.dim_res_blocks[l];
            // t_up[l]: resampler output feeding the 3x3 conv of level l (channels: convT -> C[l], bilinear -> C[l-1]);
            // doubles as the second raw map of the residual ping-pong.
            int ct = Cl;
            if (l > 0 && sc.resamplers[l - 1] == MOGE_RESAMPLE_BILINEAR) ct = std::max(Cl, sc.dim_res_blocks[l - 1]);
            size_t sz = 0, szt = 0;
            for (const auto& g : pl->groups) {
                const Level lg = level_geom(g.h, g.w, l);
                sz = std::max(sz, map_bytes(lg, g.B, Cl));
                szt = std::max(szt, map_bytes(lg, g.B, ct));
            }
            sb.x_raw[l] = ws.take(sz);
            if (sc.num_res_blocks[l] > 0) {
                sb.x_relu[l] = ws.take(sz);
                sb.y_relu[l] = ws.take(sz);
            }
            sb.t_up[l] = ws.take(szt);
        }
    };
    alloc_stack(c.neck, v->nb);
    // neck outputs must survive all heads: the neck's final x per level is whichever ping-pong map holds it (kept).
    alloc_stack(*head_cfg(e, c.points_head.present ? 0 : c.normal_head.present ? 1 : 2), v->hb);     // validate_cfg: at least one head
    // low-resolution fp32 head outputs, PER GROUP (read by the phase-2 output kernels after every group's decoder has run)
    v->pts_lr.assign(G, nullptr); v->nrm_lr.assign(G, nullptr); v->msk_lr.assign(G, nullptr);
    for (int gi = 0; gi < G; ++gi) {
        const Group& g = pl->groups[gi];
        const Level gl = level_geom(g.h, g.w, L - 1);
        const size_t px = static_cast<size_t>(g.B) * gl.H * gl.W;
        if (c.points_head.present) v->pts_lr[gi] = static_cast<float4*>(ws.take(px * 16));
        if (c.normal_head.present) v->nrm_lr[gi] = static_cast<float4*>(ws.take(px * 16));
        if (c.mask_head.present) v->msk_lr[gi] = static_cast<float*>(ws.take(px * 4));
    }
}

// MoGe-2 decoder launch list: neck and heads group by group, then every group's scale head and output resize (phase 2).
// Group gi's encoder taps start at row prow0[gi] of `taps`; `cls` / `mlp_scratch`: the scale head's input rows and scratch, per image.
static int plan_v2_decoder(moge_engine* e, Plan* pl, const uint8_t* taps, const std::vector<long>& prow0, const float* cls,
                           float* mlp_scratch, const V2Bufs& v) {
    const moge_config_t& c = e->cfg;
    const int D = c.embed_dim;
    const int G = static_cast<int>(pl->groups.size());
    const int L = c.neck.num_levels;
    const StackBufs& nb = v.nb;
    const StackBufs& hb = v.hb;
    Plan* P = pl;
    auto gname = [&](const char* base, int gi) { return G == 1 ? std::string(base) : std::string(base) + ".g" + std::to_string(gi); };
    // ---- decoder, group by group
    for (int gi = 0; gi < G; ++gi) {
        const Group& g = pl->groups[gi];
        const int B = g.B, H = g.H, W = g.W, h = g.h, w = g.w, T = h * w;
        const float aspect = static_cast<float>(W) / H;
        const float su = aspect / sqrtf(1.f + aspect * aspect), sv = 1.f / sqrtf(1.f + aspect * aspect);
        const uint8_t* taps_g = taps + static_cast<size_t>(prow0[gi]) * c.num_taps * D * 2;
        std::vector<void*> neck_out(L, nullptr);
        // neck level 0: folded projection GEMM over the concatenated taps (+UV rank-2 term) -> padded NHWC
        {
            const Level g0 = level_geom(h, w, 0);
            const ConvW& f = e->fold0;
            if (f.Ktot % 64) return set_error("num_taps*embed_dim must be a multiple of 64");
            MG_TRY(add_linear(e, pl, taps_g, B * T, f.Ktot, f.w, f.N, EPI_DEC, nb.x_raw[0], f.bias, f.wu, f.N, gname("gemm.taps_proj", gi), nullptr,
                              &g0, c.neck.num_res_blocks[0] > 0 ? nb.x_relu[0] : nullptr, f.wv, su, sv));
        }
        void* neck_lowres[3] = {v.pts_lr[gi], v.nrm_lr[gi], v.msk_lr[gi]};
        const std::string sfx = G == 1 ? std::string() : ".g" + std::to_string(gi);
        MG_TRY(plan_stack(e, pl, ("neck" + sfx).c_str(), c.neck, e->neck, true, B, h, w, su, sv, nb, neck_out, nb.x_raw[0], nb.x_relu[0], nullptr, neck_lowres));
        for (int i = 0; i < 3; ++i) {
            const moge_stack_config_t& sc = *head_cfg(e, i);
            if (!sc.present) continue;
            const Level g0 = level_geom(h, w, 0);
            const StackW& sw = e->heads[i];
            MG_TRY(add_conv(e, pl, sw.in0, neck_out[0], nullptr, g0, B, EPI_DEC, hb.x_raw[0], sc.num_res_blocks[0] > 0 ? hb.x_relu[0] : nullptr,
                            nullptr, g0, sc.dim_res_blocks[0], false, false, 0, 0, std::string("conv1x1.") + head_name(i) + sfx + ".l0"));
            void* lowres = i == 0 ? static_cast<void*>(v.pts_lr[gi]) : i == 1 ? static_cast<void*>(v.nrm_lr[gi]) : static_cast<void*>(v.msk_lr[gi]);
            MG_TRY(plan_stack(e, pl, (std::string(head_name(i)) + sfx).c_str(), sc, sw, false, B, h, w, su, sv, hb, neck_out, hb.x_raw[0], hb.x_relu[0], lowres));
        }
    }
    // ---- phase 2 (caller-bound outputs): scale head, K17 fused resize + remap
    for (int gi = 0; gi < G; ++gi) {
        const Group& g = pl->groups[gi];
        const int B = g.B, H = g.H, W = g.W;
        const Level gl = level_geom(g.h, g.w, L - 1);
        if (c.scale_head_layers > 0) {
            std::vector<const float*> mw = e->mlp_w, mb = e->mlp_b;
            std::vector<int> dims(c.scale_head_dims, c.scale_head_dims + c.scale_head_layers + 1);
            const int nl = c.scale_head_layers;
            for (int d : dims) if (d > 4096) return set_error("scale head width %d > 4096", d);
            const float* cls_g = cls + static_cast<size_t>(g.img0) * D;
            float* scratch_g = mlp_scratch + static_cast<size_t>(2) * g.img0 * 4096;
            pl->ops.add([=](cudaStream_t st) {
                if (!P->groups[gi].scale) return 0;
                return launch_scale_head(cls_g, mw.data(), mb.data(), dims.data(), nl, B, P->groups[gi].scale, scratch_g, st);
            }, gname("scale_head", gi), 0, 0, 2);
        }
        const int remap = c.remap_output;
        float4* pl_ = v.pts_lr[gi]; float4* nl_ = v.nrm_lr[gi]; float* ml_ = v.msk_lr[gi];
        pl->ops.add([=](cudaStream_t st) {
            const Group& gg = P->groups[gi];
            return launch_head_output(gg.points ? pl_ : nullptr, gg.normal ? nl_ : nullptr, gg.mask ? ml_ : nullptr, B, gl.H, gl.W,
                                      H, W, remap, gg.points, gg.normal, gg.mask, st);
        }, gname("head_output", gi), 0, static_cast<double>(B) * H * W * 28 + static_cast<double>(B) * gl.H * gl.W * 36, 2);
    }
    return 0;
}

// Workspace layout + launch list of one call shape (a list of shape groups).  `dry`: only the byte count.
static int build_plan(moge_engine* e, Plan* pl, bool dry, size_t* bytes_out, cudaStream_t upload_stream = nullptr) {
    const moge_config_t& c = e->cfg;
    const int D = c.embed_dim;
    const bool bf16 = e->bf16;
    const int G = static_cast<int>(pl->groups.size());
    long M = 0, TT = 0;             // packed token rows (with cls) / patch tokens over all groups
    int imgs = 0;
    for (auto& g : pl->groups) {
        g.img0 = imgs; g.row0 = M;
        imgs += g.B;
        M += static_cast<long>(g.B) * (g.h * g.w + 1);
        TT += static_cast<long>(g.B) * g.h * g.w;
    }
    if (M > (1L << 30)) return set_error("too many tokens in one call (%ld)", M);
    WsAlloc ws(dry ? nullptr : pl->ws);
    // ---- encoder buffers (all groups packed back to back)
    uint8_t* patches = static_cast<uint8_t*>(ws.take(static_cast<size_t>(TT) * 592 * 2));
    float* x = static_cast<float*>(ws.take(static_cast<size_t>(M) * D * 4));
    uint8_t* ln = static_cast<uint8_t*>(ws.take(static_cast<size_t>(M) * D * 2));          // the rounded residual rows x16 (LayerNorm fold)
    float2* stats = static_cast<float2*>(ws.take(static_cast<size_t>(M) * kStatsLd * 8));
    float* rstd = static_cast<float*>(ws.take(static_cast<size_t>(M) * 4));
    void* qkv = ws.take(static_cast<size_t>(M) * 3 * D * 2);
    void* att = ws.take(static_cast<size_t>(M) * D * 2);
    void* hid = ws.take(static_cast<size_t>(M) * 4 * D * 2);
    uint8_t* taps = static_cast<uint8_t*>(ws.take(static_cast<size_t>(TT) * c.num_taps * D * 2));
    float* cls = static_cast<float*>(ws.take(static_cast<size_t>(imgs) * D * 4));
    float* mlp_scratch = static_cast<float*>(ws.take(static_cast<size_t>(2) * imgs * 4096 * 4));
    // ---- decoder buffers: MoGe-1 or MoGe-2 (the encoder above is shared)
    V1Bufs vb;
    V2Bufs v2b;
    if (e->v1) v1_alloc(e, pl->groups[0], ws, &vb);
    else alloc_v2_decoder(e, pl, ws, &v2b);
    if (bytes_out) *bytes_out = ws.off + 1024;
    if (dry) return 0;
    if (ws.off > pl->ws_bytes) return set_error("workspace too small: need %zu bytes, got %zu", ws.off, pl->ws_bytes);

    Plan* P = pl;
    const int sms = e->num_sms;
    auto gname = [&](const char* base, int gi) { return G == 1 ? std::string(base) : std::string(base) + ".g" + std::to_string(gi); };
    // ---- per group: K1 resize + normalise + patchify (phase 0: reads the caller's image), K2/K3 patch embed + pos embed, cls rows
    int parts_x = 0;              // column groups per row of the statistics the NEXT consumer reads
    long prow = 0;                // first patch row of the group in `patches` / `taps`
    std::vector<long> prow0(G);
    for (int gi = 0; gi < G; ++gi) {
        const Group& g = pl->groups[gi];
        const int B = g.B, H = g.H, W = g.W, h = g.h, w = g.w, T = h * w, N = T + 1;
        prow0[gi] = prow;
        uint8_t* patches_g = patches + static_cast<size_t>(prow) * 592 * 2;
        if (e->v1) {
            // MoGe-1 (v1.py:273-279): antialiased bicubic resize to (rh, rw), then the same normalise + aa-bilinear resize to
            // (14h, 14w) + patchify as MoGe-2 (normalising after the second resize instead of between the two commutes: both
            // resizes are convex combinations per channel and the normalisation is a per-channel affine map)
            const int rh = g.rh, rw = g.rw;
            float *tmp = vb.rs_tmp, *img = vb.rs_img;
            pl->ops.add([=](cudaStream_t st) { return launch_resize_bicubic_aa(P->groups[gi].image, P->groups[gi].image_dtype, B, 3, H, W, rh, rw, tmp, img, st); },
                        "resize_bicubic_aa", 0, static_cast<double>(B) * 3 * (static_cast<double>(H) * W * 4 + static_cast<double>(H) * rw * 8 + static_cast<double>(rh) * rw * 4), 0);
            pl->ops.add([=](cudaStream_t st) { return launch_preprocess(img, MOGE_F32, B, rh, rw, h, w, patches_g, 592, bf16, st); },
                        "preprocess", 0, static_cast<double>(B) * 3 * rh * rw * 4 + static_cast<double>(B) * T * 592 * 2, 0);
            prow += static_cast<long>(B) * T;
            continue;
        }
        pl->ops.add([=](cudaStream_t st) { return launch_preprocess(P->groups[gi].image, P->groups[gi].image_dtype, B, H, W, h, w, patches_g, 592, bf16, st); },
                    gname("preprocess", gi), 0, static_cast<double>(B) * 3 * H * W * 4 + static_cast<double>(B) * T * 592 * 2, 0);
        prow += static_cast<long>(B) * T;
    }
    for (int gi = 0; gi < G; ++gi) {
        const Group& g = pl->groups[gi];
        const int B = g.B, h = g.h, w = g.w, T = h * w, N = T + 1;
        uint8_t* patches_g = patches + static_cast<size_t>(prow0[gi]) * 592 * 2;
        float* x_g = x + static_cast<size_t>(g.row0) * D;
        uint8_t* ln_g = ln + static_cast<size_t>(g.row0) * D * 2;
        float2* stats_g = stats + static_cast<size_t>(g.row0) * kStatsLd;
        LnIO prod; prod.x16 = ln_g; prod.stats_out = stats_g; prod.parts_out = &parts_x;
        const Level grid = level_geom(h, w, 0);
        MG_TRY(add_linear(e, pl, patches_g, B * T, 592, e->w_patch, D, EPI_PATCH, x_g, nullptr, g.pos_table, D, gname("gemm.patch_embed", gi),
                          &prod, &grid));
        pl->ops.add([=](cudaStream_t st) { return launch_init_cls(x_g, P->cls_row, B, N, D, st); }, gname("init_cls", gi));
        const int parts0 = parts_x;
        pl->ops.add([=](cudaStream_t st) {
            return launch_ln_prepare(x_g, B, static_cast<long>(N) * D, D, ln_g, static_cast<long>(N) * D, stats_g, static_cast<long>(N) * kStatsLd, parts0, bf16, st);
        }, gname("ln_prepare.cls", gi));
    }
    const int Mi = static_cast<int>(M);
    LnIO prod; prod.x16 = ln; prod.stats_out = stats; prod.parts_out = &parts_x;
    auto add_rstd = [&](int parts) {      // per-row rstd of the rows the last producer wrote
        pl->ops.add([=](cudaStream_t st) { return launch_ln_rstd(stats, kStatsLd, parts, Mi, D, rstd, st); }, "ln_rstd", 0, static_cast<double>(M) * (parts * 8 + 4));
    };
    // ---- attention work list (image, head, query-tile pair) over the packed rows, cost-balanced over the SMs
    {
        std::vector<int> r0, nn;
        for (const auto& g : pl->groups)
            for (int b = 0; b < g.B; ++b) { r0.push_back(static_cast<int>(g.row0 + static_cast<long>(b) * (g.h * g.w + 1))); nn.push_back(g.h * g.w + 1); }
        attention_work_list(r0.data(), nn.data(), imgs, c.num_heads, sms, &pl->att_items, &pl->att_ranges);
    }
    AttnItem* items_dev = nullptr;
    int2* ranges_dev = nullptr;
    const int att_ctas = static_cast<int>(pl->att_ranges.size());
    {
        CUDA_TRY(cudaMalloc(reinterpret_cast<void**>(&items_dev), pl->att_items.size() * sizeof(AttnItem) + 16));
        pl->owned.push_back(items_dev);
        CUDA_TRY(cudaMalloc(reinterpret_cast<void**>(&ranges_dev), pl->att_ranges.size() * sizeof(int2) + 16));
        pl->owned.push_back(ranges_dev);
        CUDA_TRY(cudaMemcpyAsync(items_dev, pl->att_items.data(), pl->att_items.size() * sizeof(AttnItem), cudaMemcpyHostToDevice, upload_stream));
        CUDA_TRY(cudaMemcpyAsync(ranges_dev, pl->att_ranges.data(), pl->att_ranges.size() * sizeof(int2), cudaMemcpyHostToDevice, upload_stream));
    }
    double att_flops = 0;
    for (const auto& g : pl->groups) { const double N = g.h * g.w + 1; att_flops += 4.0 * g.B * N * N * D; }
    // ---- transformer blocks: ONE launch per linear / attention over the packed rows of every group
    int tap_idx = 0;
    for (int i = 0; i < c.depth; ++i) {
        const moge_engine::Blk& b = e->blk[i];
        if (i == 0) add_rstd(parts_x);
        LnIO cons; cons.ln_rstd = rstd;
        MG_TRY(add_linear(e, pl, ln, Mi, D, b.wqkv_ln, 3 * D, EPI_STORE16, qkv, b.b_qkv_ln, nullptr, 3 * D, "gemm.qkv", &cons));
        {
            CUtensorMap mq;
            MG_TRY(make_map_2d(&mq, qkv, 3 * static_cast<uint64_t>(D), M, 3 * static_cast<uint64_t>(D), 128));
            const int heads = c.num_heads;
            pl->ops.add([=](cudaStream_t st) { return launch_attention(mq, att, items_dev, ranges_dev, att_ctas, D, heads, bf16, st); }, "attention",
                        att_flops, static_cast<double>(M) * D * 8);
        }
        MG_TRY(add_linear(e, pl, att, Mi, D, b.wproj, D, EPI_RESID, x, b.bproj, b.g1, D, "gemm.proj", &prod));
        add_rstd(parts_x);
        MG_TRY(add_linear(e, pl, ln, Mi, D, b.wfc1_ln, 4 * D, EPI_GELU16, hid, b.b_fc1_ln, nullptr, 4 * D, "gemm.fc1", &cons));
        MG_TRY(add_linear(e, pl, hid, Mi, 4 * D, b.wfc2, D, EPI_RESID, x, b.bfc2, b.g2, D, "gemm.fc2", (i + 1 < c.depth) ? &prod : nullptr));
        if (i + 1 < c.depth) add_rstd(parts_x);
        if (tap_idx < c.num_taps && c.taps[tap_idx] == i) {
            const int j = tap_idx++;
            const bool lasttap = (j == c.num_taps - 1);
            const int ld = c.num_taps * D;
            const float* ng = e->norm_g; const float* nbv = e->norm_b;
            for (int gi = 0; gi < G; ++gi) {
                const Group& g = pl->groups[gi];
                const int N = g.h * g.w + 1, rows = g.B * N;
                const float* x_g = x + static_cast<size_t>(g.row0) * D;
                uint8_t* taps_g = taps + static_cast<size_t>(prow0[gi]) * ld * 2;
                float* cls_g = cls + static_cast<size_t>(g.img0) * D;
                pl->ops.add([=](cudaStream_t st) {
                    return launch_layernorm(x_g, ng, nbv, taps_g, rows, D, ld, j * D, 1, N, lasttap ? cls_g : nullptr, bf16, st);
                }, gname("layernorm.tap", gi), 0, static_cast<double>(rows) * D * 6);
            }
        }
    }
    if (tap_idx != c.num_taps) return set_error("intermediate_layers must be increasing block indices < depth");
    MG_TRY(e->v1 ? plan_v1_decoder(e, pl, taps, vb) : plan_v2_decoder(e, pl, taps, prow0, cls, mlp_scratch, v2b));
    // launch order: phase 0, 1, 2 (stable)
    std::stable_sort(pl->ops.begin(), pl->ops.end(), [](const Op& a, const Op& b) { return a.phase < b.phase; });
    return 0;
}

constexpr size_t kMaxPlans = 16;

// Plans are keyed on the call shape; the workspace pointer is part of what a plan bakes in (TMA descriptors), so a call with the
// same shape but another workspace REPLACES the plan instead of orphaning it.  A plan owns its device buffers (pos tables,
// attention work list) and frees them when it is replaced or evicted (LRU) -- after the device has drained, since launches
// that read them may still be queued on the caller's stream.
static int get_plan(moge_engine* e, const moge_group_t* groups, int n, void* ws, size_t ws_bytes, Plan** out, cudaStream_t st, int rh, int rw) {
    for (size_t i = 0; i < e->plans.size(); ++i) {
        if (!e->plans[i]->same_shape(groups, n, rh, rw)) continue;
        if (e->plans[i]->ws == ws && e->plans[i]->ws_bytes == ws_bytes) {
            std::rotate(e->plans.begin() + i, e->plans.begin() + i + 1, e->plans.end());      // most recently used last
            *out = e->plans.back().get();
            return 0;
        }
        CUDA_TRY(cudaDeviceSynchronize());
        if (e->last_plan == e->plans[i].get()) e->last_plan = nullptr;
        e->plans.erase(e->plans.begin() + i);
        break;
    }
    if (e->plans.size() >= kMaxPlans) {
        CUDA_TRY(cudaDeviceSynchronize());
        if (e->last_plan == e->plans.front().get()) e->last_plan = nullptr;
        e->plans.erase(e->plans.begin());
    }
    std::unique_ptr<Plan> pl(new Plan());
    pl->ws = ws; pl->ws_bytes = ws_bytes;
    const int D = e->cfg.embed_dim;
    void* p = nullptr;
    CUDA_TRY(cudaMalloc(&p, D * 4));
    pl->owned.push_back(p);
    pl->cls_row = static_cast<float*>(p);
    for (int i = 0; i < n; ++i) {
        Group g;
        g.B = groups[i].B; g.H = groups[i].H; g.W = groups[i].W; g.h = groups[i].h; g.w = groups[i].w;
        g.rh = rh; g.rw = rw;
        CUDA_TRY(cudaMalloc(&p, static_cast<size_t>(g.h) * g.w * D * 4));
        pl->owned.push_back(p);
        g.pos_table = static_cast<float*>(p);
        MG_TRY(launch_pos_table(e->pos_embed, e->cls_token, e->patch_bias, D, g.h, g.w, g.pos_table, pl->cls_row, st));
        pl->groups.push_back(g);
    }
    MG_TRY(build_plan(e, pl.get(), false, nullptr, st));
    *out = pl.get();
    e->plans.push_back(std::move(pl));
    return 0;
}

static int validate_cfg(const moge_config_t& c) {
    if (c.embed_dim <= 0 || c.embed_dim % 128 || c.embed_dim > 1024) return set_error("embed_dim=%d unsupported (multiple of 128, <= 1024)", c.embed_dim);
    if (c.num_heads * 64 != c.embed_dim) return set_error("head_dim must be 64 (embed_dim=%d, heads=%d)", c.embed_dim, c.num_heads);
    if (c.num_taps <= 0 || c.num_taps > MOGE_MAX_TAPS) return set_error("num_taps=%d out of range", c.num_taps);
    if (c.compute_dtype != MOGE_F16 && c.compute_dtype != MOGE_BF16) return set_error("compute_dtype must be MOGE_F16 or MOGE_BF16");
    if (c.neck.num_levels < 2 || c.neck.num_levels > MOGE_MAX_LEVELS) return set_error("neck.num_levels=%d out of range", c.neck.num_levels);
    const moge_stack_config_t* first = nullptr;
    for (const moge_stack_config_t* s : {&c.points_head, &c.normal_head, &c.mask_head}) {
        if (!s->present) continue;
        if (s->num_levels != c.neck.num_levels) return set_error("head and neck level counts differ");
        for (int l = 0; l < s->num_levels; ++l) {
            if (s->dim_res_blocks[l] != c.neck.dim_res_blocks[l]) return set_error("head widths must equal neck widths");
            if (first && (s->num_res_blocks[l] != first->num_res_blocks[l] || s->resamplers[l] != first->resamplers[l]))
                return set_error("all heads must share one residual-block / resampler layout");
        }
        if (!first) first = s;
    }
    // the neck's last level is folded through the heads' last-level input + output blocks (EPI_NECKOUT), which needs this shape
    const moge_stack_config_t& n = c.neck;
    const int L = n.num_levels;
    if (!first) return set_error("a model without points, normal and mask heads is unsupported (no released config has one)");
    if (n.resamplers[L - 2] != MOGE_RESAMPLE_BILINEAR)
        return set_error("neck: resampler %d before the last level unsupported (bilinear only; no released config uses another)", n.resamplers[L - 2]);
    if (n.num_res_blocks[L - 1] != 0)
        return set_error("neck: %d residual blocks at the last level unsupported (no released config uses them)", n.num_res_blocks[L - 1]);
    if (n.dim_res_blocks[L - 1] != 32) return set_error("neck: last-level width %d unsupported (32 only)", n.dim_res_blocks[L - 1]);
    return 0;
}

static int validate_v1(const moge_v1_config_t& c) {
    const int D = c.embed_dim;
    if (!((D == 384 && c.depth == 12 && c.num_heads == 6) || (D == 768 && c.depth == 12 && c.num_heads == 12) ||
          (D == 1024 && c.depth == 24 && c.num_heads == 16)))
        return set_error("v1: backbone (embed_dim=%d, depth=%d, heads=%d) unsupported: DINOv2 ViT-S/B/L only", D, c.depth, c.num_heads);
    if (c.num_taps <= 0 || c.num_taps > MOGE_MAX_TAPS) return set_error("v1: num_taps=%d out of range", c.num_taps);
    for (int i = 0; i < c.num_taps; ++i)
        if (c.taps[i] < 0 || c.taps[i] >= c.depth || (i > 0 && c.taps[i] <= c.taps[i - 1]))
            return set_error("v1: intermediate_layers must be increasing block indices < depth");
    if (c.compute_dtype != MOGE_F16 && c.compute_dtype != MOGE_BF16) return set_error("v1: compute_dtype must be MOGE_F16 or MOGE_BF16");
    if (c.remap_output < MOGE_REMAP_LINEAR || c.remap_output > MOGE_REMAP_SINH_EXP) return set_error("v1: remap_output=%d unsupported", c.remap_output);
    if (c.last_res_blocks != 0) return set_error("v1: last_res_blocks=%d unsupported (no released config uses it)", c.last_res_blocks);
    if (c.last_conv_size != 1) return set_error("v1: last_conv_size=%d unsupported (no released config uses it)", c.last_conv_size);
    if (c.last_conv_channels != 32) return set_error("v1: last_conv_channels=%d unsupported (32 only)", c.last_conv_channels);
    if (c.hidden_norm != MOGE_V1_GROUP_NORM && c.hidden_norm != MOGE_V1_LAYER_NORM) return set_error("v1: hidden_norm=%d unsupported", c.hidden_norm);
    if (c.num_res_blocks < 0 || c.hidden_mult < 1) return set_error("v1: num_res_blocks=%d / hidden_mult=%d out of range", c.num_res_blocks, c.hidden_mult);
    if (c.dim_proj <= 0 || c.dim_proj % 128 || c.dim_proj > 2048) return set_error("v1: dim_proj=%d unsupported (a multiple of 128, <= 2048)", c.dim_proj);
    if (c.num_levels < 1 || c.num_levels > MOGE_MAX_LEVELS) return set_error("v1: %d upsampling levels out of range", c.num_levels);
    for (int l = 0; l < c.num_levels; ++l) {
        const int C = c.dim_upsample[l], Hd = c.hidden_mult * C;
        if (C <= 0 || C % 64 || Hd > 2048) return set_error("v1: dim_upsample[%d]=%d (hidden %d) unsupported (multiples of 64, <= 2048)", l, C, Hd);
    }
    return 0;
}

}  // namespace mg

// ================================================================================================ C ABI
extern "C" {

const char* moge_last_error(void) { return mg::last_error(); }
const char* moge_version(void) { return "moge_b200 0.1.0 sm_90a"; }

static int create_engine(const moge_config_t* cfg, int device, moge_engine_t** out) {
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) return set_error("no CUDA device: moge_b200 has no CPU fallback");
    CUDA_TRY(cudaSetDevice(device));
    cudaDeviceProp prop;
    CUDA_TRY(cudaGetDeviceProperties(&prop, device));
    if (prop.major != 9 || prop.minor != 0) return set_error("device %d is sm_%d%d; libmoge_b200 contains sm_90a code only", device, prop.major, prop.minor);
    moge_engine* e = new moge_engine();
    e->cfg = *cfg; e->device = device; e->num_sms = prop.multiProcessorCount; e->bf16 = cfg->compute_dtype == MOGE_BF16;
    if (cudaStreamCreateWithFlags(&e->own_stream, cudaStreamNonBlocking) != cudaSuccess ||
        cudaEventCreateWithFlags(&e->ev_in, cudaEventDisableTiming) != cudaSuccess ||
        cudaEventCreateWithFlags(&e->ev_out, cudaEventDisableTiming) != cudaSuccess) {
        delete e;
        return set_error("stream/event creation failed");
    }
    *out = e;
    return 0;
}

int moge_engine_create(const moge_config_t* cfg, int device, moge_engine_t** out) {
    if (!cfg || !out) return set_error("null argument");
    MG_TRY(validate_cfg(*cfg));
    return create_engine(cfg, device, out);
}

int moge_engine_create_v1(const moge_v1_config_t* cfg, int device, moge_engine_t** out) {
    if (!cfg || !out) return set_error("null argument");
    MG_TRY(validate_v1(*cfg));
    moge_config_t enc{};         // the encoder part only: build_plan takes the MoGe-1 decoder path for this engine
    enc.embed_dim = cfg->embed_dim; enc.depth = cfg->depth; enc.num_heads = cfg->num_heads;
    enc.num_taps = cfg->num_taps;
    for (int i = 0; i < cfg->num_taps; ++i) enc.taps[i] = cfg->taps[i];
    enc.remap_output = cfg->remap_output;
    enc.compute_dtype = cfg->compute_dtype;
    MG_TRY(create_engine(&enc, device, out));
    (*out)->v1 = true;
    (*out)->v1cfg = *cfg;
    return 0;
}

void moge_engine_destroy(moge_engine_t* e) {
    if (!e) return;
    cudaSetDevice(e->device);
    cudaDeviceSynchronize();
    e->plans.clear();            // each plan frees its graph and buffers
    if (e->own_stream) cudaStreamDestroy(e->own_stream);
    if (e->ev_in) cudaEventDestroy(e->ev_in);
    if (e->ev_out) cudaEventDestroy(e->ev_out);
    for (void* p : e->owned) cudaFree(p);
    for (void* p : e->temps) cudaFree(p);
    for (auto& kv : e->raw) if (kv.second.p) cudaFree(kv.second.p);
    delete e;
}

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

static int check_groups(moge_engine_t* e, const moge_group_t* g, int n, bool need_ptrs) {
    if (!e || !g) return set_error("null argument");
    if (n <= 0 || n > 64) return set_error("number of shape groups %d out of range (1..64)", n);
    for (int i = 0; i < n; ++i) {
        if (g[i].B <= 0 || g[i].h <= 0 || g[i].w <= 0 || g[i].H <= 0 || g[i].W <= 0)
            return set_error("bad shape B=%d H=%d W=%d h=%d w=%d", g[i].B, g[i].H, g[i].W, g[i].h, g[i].w);
        if (!need_ptrs) continue;
        if (!g[i].image) return set_error("null argument");
        if (g[i].image_dtype != MOGE_F32 && g[i].image_dtype != MOGE_F16 && g[i].image_dtype != MOGE_BF16) return set_error("unsupported image dtype %d", g[i].image_dtype);
        if (e->v1) continue;                 // moge_v1_forward checks its outputs
        if (g[i].points && !e->cfg.points_head.present) return set_error("points requested but the model has no points head");
        if (g[i].normal && !e->cfg.normal_head.present) return set_error("normal requested but the model has no normal head");
        if (g[i].mask_prob && !e->cfg.mask_head.present) return set_error("mask requested but the model has no mask head");
        if (g[i].metric_scale && e->cfg.scale_head_layers == 0) return set_error("metric_scale requested but the model has no scale head");
    }
    return 0;
}

int moge_engine_workspace_bytes_groups(moge_engine_t* e, const moge_group_t* groups, int n, size_t* bytes) {
    if (!bytes) return set_error("null argument");
    MG_TRY(check_groups(e, groups, n, false));
    if (e->v1) return set_error("a MoGe-1 engine takes moge_v1_workspace_bytes");
    Plan pl;
    for (int i = 0; i < n; ++i) {
        Group g;
        g.B = groups[i].B; g.H = groups[i].H; g.W = groups[i].W; g.h = groups[i].h; g.w = groups[i].w;
        pl.groups.push_back(g);
    }
    return build_plan(e, &pl, true, bytes);
}

int moge_engine_workspace_bytes(moge_engine_t* e, int B, int H, int W, int h, int w, size_t* bytes) {
    moge_group_t g{};
    g.B = B; g.H = H; g.W = W; g.h = h; g.w = w;
    return moge_engine_workspace_bytes_groups(e, &g, 1, bytes);
}

// rh, rw: the resized image of a MoGe-1 call (0 for MoGe-2)
static int forward_impl(moge_engine_t* e, const moge_group_t* groups, int n, void* workspace, size_t workspace_bytes, void* stream, int rh, int rw) {
    if (!e || !workspace) return set_error("null argument");
    if (!e->finalized) return set_error("engine not finalized");
    MG_TRY(check_groups(e, groups, n, true));
    if (reinterpret_cast<uintptr_t>(workspace) & 1023) return set_error("workspace must be 1024-byte aligned");
    CUDA_TRY(cudaSetDevice(e->device));
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    Plan* pl;
    MG_TRY(get_plan(e, groups, n, workspace, workspace_bytes, &pl, st, rh, rw));
    long tokens = 0;
    for (int i = 0; i < n; ++i) {
        Group& g = pl->groups[i];
        g.image = groups[i].image; g.image_dtype = groups[i].image_dtype;
        g.points = groups[i].points; g.normal = groups[i].normal; g.mask = groups[i].mask_prob; g.scale = groups[i].metric_scale;
        tokens += static_cast<long>(g.B) * g.h * g.w;
    }
    e->last_plan = pl;
    // ---- graph replay of the workspace-only launches (small batches only: at large batch the GPU is the bottleneck and the CPU
    //      runs ahead anyway).  The first run of a plan is eager (sets kernel attributes, warms caches).
    const bool want_graph = tokens <= 4 * 3600;
    struct PdlScope {          // programmatic dependent launch for the small calls only (host_api.h)
        bool prev;
        explicit PdlScope(bool on) : prev(pdl_scope()) { pdl_scope() = on; }
        ~PdlScope() { pdl_scope() = prev; }
    } pdl(tokens <= 4 * 3600);
    if (!want_graph || pl->eager_runs == 0) {
        pl->eager_runs++;
        for (auto& op : pl->ops) MG_TRY(op.fn(st));
        return 0;
    }
    size_t i0 = 0, i1 = pl->ops.size();
    while (i0 < pl->ops.size() && pl->ops[i0].phase == 0) ++i0;
    while (i1 > i0 && pl->ops[i1 - 1].phase == 2) --i1;
    // stream capture is not allowed on the legacy default stream: run on the engine's own stream, fenced by events
    const bool legacy = (st == nullptr || st == cudaStreamLegacy || st == cudaStreamPerThread);
    cudaStream_t run = legacy ? e->own_stream : st;
    for (size_t i = 0; i < i0; ++i) MG_TRY(pl->ops[i].fn(st));
    if (legacy) {
        CUDA_TRY(cudaEventRecord(e->ev_in, st));
        CUDA_TRY(cudaStreamWaitEvent(e->own_stream, e->ev_in, 0));
    }
    if (!pl->exec) {
        cudaGraph_t graph = nullptr;
        CUDA_TRY(cudaStreamBeginCapture(run, cudaStreamCaptureModeThreadLocal));
        int rc = 0;
        for (size_t i = i0; i < i1; ++i) { rc = pl->ops[i].fn(run); if (rc) break; }
        cudaError_t ce = cudaStreamEndCapture(run, &graph);
        if (rc) { if (graph) cudaGraphDestroy(graph); return rc; }
        if (ce != cudaSuccess) return set_error("graph capture failed: %s", cudaGetErrorString(ce));
        ce = cudaGraphInstantiate(&pl->exec, graph, 0);
        cudaGraphDestroy(graph);
        if (ce != cudaSuccess) { pl->exec = nullptr; return set_error("cudaGraphInstantiate failed: %s", cudaGetErrorString(ce)); }
    }
    CUDA_TRY(cudaGraphLaunch(pl->exec, run));
    if (legacy) {
        CUDA_TRY(cudaEventRecord(e->ev_out, e->own_stream));
        CUDA_TRY(cudaStreamWaitEvent(st, e->ev_out, 0));
    }
    for (size_t i = i1; i < pl->ops.size(); ++i) MG_TRY(pl->ops[i].fn(st));
    return 0;
}

int moge_engine_forward_groups(moge_engine_t* e, const moge_group_t* groups, int n, void* workspace, size_t workspace_bytes, void* stream) {
    if (e && e->v1) return set_error("a MoGe-1 engine runs through moge_v1_forward");
    return forward_impl(e, groups, n, workspace, workspace_bytes, stream, 0, 0);
}

static int check_v1_shape(moge_engine_t* e, int B, int H, int W, int rh, int rw) {
    if (!e) return set_error("null argument");
    if (!e->v1) return set_error("not a MoGe-1 engine (moge_engine_create_v1)");
    if (B <= 0 || H <= 0 || W <= 0) return set_error("bad shape B=%d H=%d W=%d", B, H, W);
    if (rh < 14 || rw < 14) return set_error("resized image %dx%d is smaller than one 14-pixel patch", rh, rw);
    return 0;
}

int moge_v1_workspace_bytes(moge_engine_t* e, int B, int H, int W, int rh, int rw, size_t* bytes) {
    if (!bytes) return set_error("null argument");
    MG_TRY(check_v1_shape(e, B, H, W, rh, rw));
    Plan pl;
    Group g;
    g.B = B; g.H = H; g.W = W; g.h = rh / 14; g.w = rw / 14; g.rh = rh; g.rw = rw;
    pl.groups.push_back(g);
    return build_plan(e, &pl, true, bytes);
}

int moge_v1_forward(moge_engine_t* e, const void* image, int image_dtype, int B, int H, int W, int rh, int rw, void* workspace,
                    size_t workspace_bytes, float* points, float* mask, void* stream) {
    MG_TRY(check_v1_shape(e, B, H, W, rh, rw));
    if (!points || !mask) return set_error("null argument");
    moge_group_t g{};
    g.image = image; g.image_dtype = image_dtype; g.B = B; g.H = H; g.W = W; g.h = rh / 14; g.w = rw / 14;
    g.points = points; g.mask_prob = mask;
    return forward_impl(e, &g, 1, workspace, workspace_bytes, stream, rh, rw);
}

int moge_v1_postprocess(float* points, const float* mask, float mask_threshold, const float* focal_in, int B, int H, int W,
                        int force_projection, int apply_mask, float* depth, uint8_t* mask_out, float* intrinsics, float* focal,
                        float* shift, void* stream) {
    if (!points || !mask || !depth || !mask_out || !intrinsics || !focal || !shift) return set_error("null argument");
    if (B <= 0 || H <= 0 || W <= 0) return set_error("bad shape B=%d H=%d W=%d", B, H, W);
    return launch_v1_postprocess(points, mask, mask_threshold, focal_in, B, H, W, force_projection, apply_mask, depth, mask_out, intrinsics,
                                 focal, shift, static_cast<cudaStream_t>(stream));
}

int moge_engine_forward(moge_engine_t* e, const void* image, int image_dtype, int B, int H, int W, int h, int w, void* workspace,
                        size_t workspace_bytes, float* points, float* normal, float* mask_prob, float* metric_scale, void* stream) {
    moge_group_t g{};
    g.image = image; g.image_dtype = image_dtype; g.B = B; g.H = H; g.W = W; g.h = h; g.w = w;
    g.points = points; g.normal = normal; g.mask_prob = mask_prob; g.metric_scale = metric_scale;
    return moge_engine_forward_groups(e, &g, 1, workspace, workspace_bytes, stream);
}

int moge_engine_num_ops(moge_engine_t* e, int* n) {
    if (!e || !n) return set_error("null argument");
    if (!e->last_plan) return set_error("no forward has run yet");
    *n = static_cast<int>(e->last_plan->ops.size());
    return 0;
}

int moge_engine_op_info(moge_engine_t* e, int idx, char* name, int name_cap, double* flops, double* bytes) {
    if (!e || !e->last_plan) return set_error("no forward has run yet");
    if (idx < 0 || idx >= static_cast<int>(e->last_plan->ops.size())) return set_error("op index %d out of range", idx);
    const Op& op = e->last_plan->ops[idx];
    if (name && name_cap > 0) snprintf(name, name_cap, "%s", op.name.c_str());
    if (flops) *flops = op.flops;
    if (bytes) *bytes = op.bytes;
    return 0;
}

int moge_engine_profile(moge_engine_t* e, float* ms, int cap, void* stream) {
    if (!e || !e->last_plan || !ms) return set_error("profile: run moge_engine_forward once first");
    Plan* pl = e->last_plan;
    const int n = static_cast<int>(pl->ops.size());
    if (cap < n) return set_error("profile: need room for %d ops", n);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    CUDA_TRY(cudaSetDevice(e->device));
    std::vector<cudaEvent_t> ev(n + 1);
    for (auto& x : ev) CUDA_TRY(cudaEventCreate(&x));
    CUDA_TRY(cudaEventRecord(ev[0], st));
    for (int i = 0; i < n; ++i) {
        MG_TRY(pl->ops[i].fn(st));
        CUDA_TRY(cudaEventRecord(ev[i + 1], st));
    }
    CUDA_TRY(cudaStreamSynchronize(st));
    for (int i = 0; i < n; ++i) CUDA_TRY(cudaEventElapsedTime(&ms[i], ev[i], ev[i + 1]));
    for (auto& x : ev) cudaEventDestroy(x);
    return 0;
}

int moge_recover_focal_shift(const float* points, const float* mask_prob, const uint8_t* mask_u8, int B, int H, int W,
                             const float* focal_in, float* focal_out, float* shift_out, void* stream) {
    if (!points || !focal_out || !shift_out) return set_error("null argument");
    return launch_focal_shift(points, mask_prob, mask_u8, B, H, W, focal_in, focal_out, shift_out, static_cast<cudaStream_t>(stream));
}

int moge_postprocess(float* points, const float* normal_in, const float* mask_prob, const float* metric_scale, const float* focal,
                     const float* shift, int B, int H, int W, int force_projection, int apply_mask, float* depth, float* normal_out,
                     uint8_t* mask_out, float* intrinsics, void* stream) {
    if (!points || !focal || !shift || !depth || !intrinsics) return set_error("null argument");
    if (normal_in && !normal_out) return set_error("normal_out required when normal_in is given");
    return launch_postprocess(points, normal_in, mask_prob, metric_scale, focal, shift, B, H, W, force_projection, apply_mask, depth,
                              normal_out, mask_out, intrinsics, static_cast<cudaStream_t>(stream));
}

// ---------------------------------------------------------------------------------- operator-level entry points
static int dev_sms() {
    int dev = 0, sms = 132;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    return sms;
}

int moge_op_linear(const void* x, const void* w, const float* bias, const float* gamma, void* out, int M, int N, int K, int epi,
                   int dtype, void* stream) {
    if (K % 8) return set_error("op_linear: K must be a multiple of 8");
    if (epi < 0 || epi > 2) return set_error("op_linear: epi must be 0..2");
    GemmLaunch g;
    MG_TRY(gemm_linear(&g, dtype == MOGE_BF16, x, M, K, w, K, N, epi, out, N, bias, gamma));
    return launch_gemm(g, dev_sms(), static_cast<cudaStream_t>(stream));
}

int moge_op_attention(const void* qkv, void* out, int B, int N, int D, int heads, int dtype, void* stream) {
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    if (B <= 0 || N <= 0) return set_error("op_attention: bad shape B=%d N=%d", B, N);
    CUtensorMap mq;
    MG_TRY(make_map_2d(&mq, qkv, 3 * static_cast<uint64_t>(D), static_cast<uint64_t>(B) * N, 3 * static_cast<uint64_t>(D), 128));
    std::vector<int> row0(B), n(B, N);
    for (int b = 0; b < B; ++b) row0[b] = b * N;
    std::vector<AttnItem> items;
    std::vector<int2> ranges;
    attention_work_list(row0.data(), n.data(), B, heads, dev_sms(), &items, &ranges);
    AttnItem* items_dev = nullptr;
    int2* ranges_dev = nullptr;
    CUDA_TRY(cudaMalloc(reinterpret_cast<void**>(&items_dev), items.size() * sizeof(AttnItem) + 16));
    if (cudaMalloc(reinterpret_cast<void**>(&ranges_dev), ranges.size() * sizeof(int2) + 16) != cudaSuccess) { cudaFree(items_dev); return set_error("op_attention: cudaMalloc failed"); }
    int rc = 0;
    if (cudaMemcpyAsync(items_dev, items.data(), items.size() * sizeof(AttnItem), cudaMemcpyHostToDevice, st) != cudaSuccess ||
        cudaMemcpyAsync(ranges_dev, ranges.data(), ranges.size() * sizeof(int2), cudaMemcpyHostToDevice, st) != cudaSuccess)
        rc = set_error("op_attention: upload failed");
    if (rc == 0) rc = launch_attention(mq, out, items_dev, ranges_dev, static_cast<int>(ranges.size()), D, heads, dtype == MOGE_BF16, st);
    cudaStreamSynchronize(st);
    cudaFree(items_dev); cudaFree(ranges_dev);
    return rc;
}

int moge_attention_work_list(const int* n_tokens, int n_images, int heads, int n_ctas, int* items, int items_cap, int* ranges, int* n_items,
                             int* n_ranges) {
    // host only: the work list the engine uploads for the persistent attention kernel (plan time), for inspection and tests
    if (n_images < 0 || heads <= 0 || n_ctas <= 0 || !n_tokens) return set_error("attention_work_list: bad arguments");
    std::vector<int> row0(n_images);
    int r = 0;
    for (int i = 0; i < n_images; ++i) {
        if (n_tokens[i] <= 0) return set_error("attention_work_list: image %d has %d tokens", i, n_tokens[i]);
        row0[i] = r; r += n_tokens[i];
    }
    std::vector<AttnItem> it;
    std::vector<int2> rg;
    attention_work_list(row0.data(), n_tokens, n_images, heads, n_ctas, &it, &rg);
    if (n_items) *n_items = static_cast<int>(it.size());
    if (n_ranges) *n_ranges = static_cast<int>(rg.size());
    if (items) {
        if (items_cap < static_cast<int>(it.size())) return set_error("attention_work_list: items_cap %d < %zu", items_cap, it.size());
        for (size_t i = 0; i < it.size(); ++i) { items[4 * i] = it[i].row0; items[4 * i + 1] = it[i].n; items[4 * i + 2] = it[i].q0; items[4 * i + 3] = it[i].head; }
    }
    if (ranges) for (size_t i = 0; i < rg.size(); ++i) { ranges[2 * i] = rg[i].x; ranges[2 * i + 1] = rg[i].y; }
    return 0;
}

int moge_op_linear_ln(const float* x, const float* ln_gamma, const float* ln_beta, const float* w, const float* bias, void* out, int M,
                      int N, int K, int epi, int dtype, void* stream) {
    // out = epi(LayerNorm(x) W^T + bias) the way the engine computes it: rounded rows + row statistics, folded weights, one GEMM
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const bool bf16 = dtype == MOGE_BF16;
    if (K % 64) return set_error("op_linear_ln: K must be a multiple of 64");
    if (epi != EPI_STORE16 && epi != EPI_GELU16) return set_error("op_linear_ln: epi must be 0 (store) or 1 (GELU)");
    void *x16 = nullptr, *w16 = nullptr;
    float2* stats = nullptr;
    float *rstd = nullptr, *b2 = nullptr;
    int rc = 0;
    if (cudaMalloc(&x16, static_cast<size_t>(M) * K * 2) != cudaSuccess || cudaMalloc(&w16, static_cast<size_t>(N) * K * 2) != cudaSuccess ||
        cudaMalloc(&stats, static_cast<size_t>(M) * kStatsLd * 8) != cudaSuccess || cudaMalloc(&rstd, static_cast<size_t>(M) * 4) != cudaSuccess ||
        cudaMalloc(&b2, static_cast<size_t>(N) * 4) != cudaSuccess)
        rc = set_error("op_linear_ln: cudaMalloc failed");
    LnIO cons;
    cons.ln_rstd = rstd;
    GemmLaunch g;
    if (rc == 0) rc = gemm_linear(&g, bf16, x16, M, K, w16, K, N, epi, out, N, b2, nullptr, &cons);
    if (rc == 0) rc = launch_ln_prepare(x, M, K, K, x16, K, stats, kStatsLd, 1, bf16, st);
    if (rc == 0) rc = launch_ln_rstd(stats, kStatsLd, 1, M, K, rstd, st);
    if (rc == 0) rc = launch_ln_fold(w, ln_gamma, ln_beta, bias, N, K, K, w16, b2, bf16, st);
    if (rc == 0) rc = launch_gemm(g, dev_sms(), st);
    cudaStreamSynchronize(st);
    cudaFree(x16); cudaFree(w16); cudaFree(stats); cudaFree(rstd); cudaFree(b2);
    return rc;
}

int moge_op_layernorm(const float* x, const float* gamma, const float* beta, void* out, int rows, int D, int dtype, void* stream) {
    return launch_layernorm(x, gamma, beta, out, rows, D, D, 0, 0, 1, nullptr, dtype == MOGE_BF16, static_cast<cudaStream_t>(stream));
}

int moge_op_conv(const void* x, const float* w, const float* bias, const void* skip, void* out_raw, void* out_relu, int B, int H, int W,
                 int Cin, int Cout, int taps, int shuffle, int dtype, void* stream) {
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const bool bf16 = dtype == MOGE_BF16;
    if (Cin % 64) return set_error("op_conv: Cin must be a multiple of 64");
    if (taps != 1 && taps != 9) return set_error("op_conv: taps must be 1 or 9");
    if (shuffle && taps != 1) return set_error("op_conv: shuffle requires taps=1");
    const int N = shuffle ? 4 * Cout : Cout;
    const int Ktot = taps * Cin;
    void* wp = nullptr;
    CUDA_TRY(cudaMalloc(&wp, static_cast<size_t>(N) * Ktot * 2));
    int rc = shuffle ? launch_pack_convT(w, wp, bf16, Cin, Cout, st) : launch_pack_conv(w, wp, bf16, Cout, Cin, taps, Ktot, 0, st);
    if (rc == 0) {
        ConvW cw;
        cw.w = wp; cw.bias = const_cast<float*>(bias); cw.N = N; cw.Ktot = Ktot; cw.cin = Cin; cw.taps = taps;
        const Level gs = level_geom(H, W, 0), go = level_geom(H, W, shuffle ? 1 : 0);
        GemmLaunch g;
        rc = gemm_conv(&g, bf16, cw, x, nullptr, gs, B, EPI_DEC, out_raw, out_relu, skip, go, Cout, shuffle != 0, false, 0.f, 0.f);
        if (rc == 0) rc = launch_gemm(g, dev_sms(), st);
    }
    cudaStreamSynchronize(st);
    cudaFree(wp);
    return rc;
}

int moge_op_resize_bicubic_aa(const void* x, int dtype, int B, int C, int H, int W, int Ho, int Wo, float* out, void* stream) {
    if (!x || !out) return set_error("null argument");
    if (dtype != MOGE_F32 && dtype != MOGE_F16 && dtype != MOGE_BF16) return set_error("op_resize_bicubic_aa: unsupported dtype %d", dtype);
    if (B <= 0 || C <= 0 || H <= 0 || W <= 0 || Ho <= 0 || Wo <= 0) return set_error("op_resize_bicubic_aa: bad shape");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    float* tmp = nullptr;
    CUDA_TRY(cudaMalloc(reinterpret_cast<void**>(&tmp), static_cast<size_t>(B) * C * H * Wo * 4));
    const int rc = launch_resize_bicubic_aa(x, dtype, B, C, H, W, Ho, Wo, tmp, out, st);
    cudaStreamSynchronize(st);
    cudaFree(tmp);
    return rc;
}

int moge_op_groupnorm_relu(const void* x, void* out, const float* gamma, const float* beta, int B, int H, int W, int C, int G, int dtype,
                           void* stream) {
    if (!x || !out || !gamma || !beta) return set_error("null argument");
    if (B <= 0 || H <= 0 || W <= 0 || C <= 0 || C % 8) return set_error("op_groupnorm_relu: bad shape");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const bool bf16 = dtype == MOGE_BF16;
    const Level g = level_geom(H, W, 0);
    double2* part = nullptr;
    float2* stats = nullptr;
    int rc = 0;
    if (G <= 0 || cudaMalloc(reinterpret_cast<void**>(&part), static_cast<size_t>(B) * gn_tiles(H, W, C) * G * 16) != cudaSuccess ||
        cudaMalloc(reinterpret_cast<void**>(&stats), static_cast<size_t>(B) * G * 8) != cudaSuccess)
        rc = set_error("op_groupnorm_relu: G=%d / cudaMalloc failed", G);
    if (rc == 0) rc = launch_gn_stats(x, g, B, C, G, part, stats, bf16, st);
    if (rc == 0) rc = launch_gn_relu(x, out, g, B, C, G, stats, gamma, beta, bf16, st);
    cudaStreamSynchronize(st);
    cudaFree(part); cudaFree(stats);
    return rc;
}

int moge_op_conv_transpose_uv(const void* x, const float* w, const float* bias, void* out, int B, int H, int W, int Cin, int Cout, float su, float sv,
                     int dtype, void* stream) {
    // the engine's MoGe-1 upsampling ConvTranspose: the GEMM over the feature rows (pixel shuffle), then the input-grid UV term
    if (!x || !w || !bias || !out) return set_error("null argument");
    if (B <= 0 || H <= 0 || W <= 0) return set_error("op_conv_transpose_uv: bad shape");
    if (Cin % 64 || Cout <= 0 || Cout % 32) return set_error("op_conv_transpose_uv: Cin %% 64 and Cout %% 32 must be 0");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const bool bf16 = dtype == MOGE_BF16;
    void* wp = nullptr;
    float* wuv = nullptr;
    int rc = 0;
    if (cudaMalloc(&wp, static_cast<size_t>(4) * Cout * Cin * 2) != cudaSuccess ||
        cudaMalloc(reinterpret_cast<void**>(&wuv), static_cast<size_t>(8) * Cout * 4) != cudaSuccess)
        rc = set_error("op_conv_transpose_uv: cudaMalloc failed");
    if (rc == 0) rc = launch_pack_convT(w, wp, bf16, Cin, Cout, st);
    if (rc == 0) rc = launch_pack_convT_uv(w, Cin, Cout, wuv, st);
    if (rc == 0) {
        ConvW cw;
        cw.w = wp; cw.bias = const_cast<float*>(bias); cw.N = 4 * Cout; cw.Ktot = Cin; cw.cin = Cin; cw.taps = 1;
        const Level gs = level_geom(H, W, 0), go = level_geom(H, W, 1);
        GemmLaunch g;
        rc = gemm_conv(&g, bf16, cw, x, nullptr, gs, B, EPI_DEC, out, nullptr, nullptr, go, Cout, true, false, 0.f, 0.f);
        if (rc == 0) rc = launch_gemm(g, dev_sms(), st);
        if (rc == 0) rc = launch_uv_convT(out, go, B, Cout, wuv, su, sv, bf16, st);
    }
    cudaStreamSynchronize(st);
    cudaFree(wp); cudaFree(wuv);
    return rc;
}

int moge_bicubic_aa_weights(int in, int out, int i, int* lo, float* w, int cap) {
    if (!lo) return set_error("null argument");
    if (in <= 0 || out <= 0 || i < 0 || i >= out) return set_error("bicubic_aa_weights: bad arguments in=%d out=%d i=%d", in, out, i);
    return bicubic_aa_taps(in, out, i, lo, w, cap);
}

}  // extern "C"
