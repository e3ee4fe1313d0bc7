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
#include <stdlib.h>

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
    float* waux = nullptr;          // [ncomp, 32] = output block o last-level input block (applied to the neck's last-level map)
    int ncomp = 0;
    // neck only: its last level folded through the heads' waux (EPI_NECKOUT): N = 4 phases x 8 components
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
    bool same_shape(const moge_group_t* g, int n) const {
        if (static_cast<int>(groups.size()) != n) return false;
        for (int i = 0; i < n; ++i)
            if (groups[i].B != g[i].B || groups[i].H != g[i].H || groups[i].W != g[i].W || groups[i].h != g[i].h || groups[i].w != g[i].w) return false;
        return true;
    }
    ~Plan() {
        if (exec) cudaGraphExecDestroy(exec);
        for (void* p : owned) cudaFree(p);
    }
};

}  // namespace mg

using namespace mg;

struct moge_engine {
    moge_config_t cfg;
    int device = 0, num_sms = 132;
    bool bf16 = false, finalized = false;
    std::map<std::string, RawWeight> raw;
    std::vector<void*> owned;         // cudaMalloc'd, freed at destroy
    // packed encoder
    void* w_patch = nullptr;
    struct Blk {
        void *wqkv, *wproj, *wfc1, *wfc2;
        const float *bqkv, *bproj, *bfc1, *bfc2, *g1, *g2, *ln1g, *ln1b, *ln2g, *ln2b;
        // LayerNorm folded into the GEMM (default; MOGE_B200_LNFOLD=0 disables): centred W diag(gamma) in 16 bit, b + W beta
        void *wqkv_ln, *wfc1_ln;
        float *b_qkv_ln, *b_fc1_ln;
    };
    std::vector<Blk> blk;
    const float *norm_g = nullptr, *norm_b = nullptr, *pos_embed = nullptr, *cls_token = nullptr, *patch_bias = nullptr;
    ConvW fold0;                      // taps-concat GEMM: (output projections folded into neck.input_blocks.0)
    StackW neck, heads[3];            // heads: points, normal, mask
    std::vector<const float*> mlp_w, mlp_b;
    std::vector<std::unique_ptr<Plan>> plans;      // LRU order (most recently used last), at most kMaxPlans
    Plan* last_plan = nullptr;
    std::vector<void*> temps;         // load-time scratch (fp32 folds), freed at the end of finalize
    bool use_graphs = true;
    bool neck_fold = false;       // last neck level folded through the heads (EPI_NECKOUT); decided at finalize
    bool ln_fold = true;          // LayerNorm folded into qkv / fc1 (SURVEY K4/K7); MOGE_B200_LNFOLD=0: separate layernorm kernel
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

static int pack_stack(moge_engine* e, const std::string& name, const moge_stack_config_t& sc, bool is_neck, StackW* sw,
                      cudaStream_t st, const float* waux_all = nullptr) {
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
                if (waux_all != nullptr && l + 1 == L - 1) {
                    // Last neck level folded through the heads (EPI_NECKOUT).  The level-(L-1) neck map m = conv3x3(up2(x)) + b + Wuv uv
                    // is consumed ONLY by the heads' last-level input blocks and, with no nonlinearity in between, by their output
                    // blocks: head k-th component += waux_all[k, :] m.  Push waux_all through the (linear) conv: a 3x3 conv with
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
                        MG_TRY(launch_sgemm(waux_all, Cn, wexp + static_cast<size_t>(ph) * Cn * K9, K9, wfold + static_cast<size_t>(ph) * 8 * K9, K9, 8, K9, Cn, 0, st));
                    ConvW& no = sw->neckout;
                    no.N = 32; no.cin = conv_cin; no.taps = 9; no.Ktot = K9;
                    MG_TRY(e->alloc(&no.w, static_cast<size_t>(32) * K9 * 2));
                    MG_TRY(launch_pack_conv(wfold, no.w, e->bf16, 32, conv_cin, 9, K9, 0, st));
                    MG_TRY(sum_bias(e, bc, bi, Cn, &bsum, st));
                    MG_TRY(e->alloc(reinterpret_cast<void**>(&no.bias), 8 * 4));
                    MG_TRY(launch_sgemm(waux_all, Cn, bsum, 1, no.bias, 1, 8, 1, Cn, 0, st));
                    MG_TRY(e->alloc_temp(reinterpret_cast<void**>(&wuv), 2 * Cn * 4));
                    vec_combine_kernel<<<(Cn + 255) / 256, 256, 0, st>>>(wuv, wi->p, 2, nullptr, Cn);
                    vec_combine_kernel<<<(Cn + 255) / 256, 256, 0, st>>>(wuv + Cn, wi->p + 1, 2, nullptr, Cn);
                    CUDA_TRY(cudaGetLastError());
                    MG_TRY(e->alloc(reinterpret_cast<void**>(&no.wu), 8 * 4));
                    MG_TRY(e->alloc(reinterpret_cast<void**>(&no.wv), 8 * 4));
                    MG_TRY(launch_sgemm(waux_all, Cn, wuv, 1, no.wu, 1, 8, 1, Cn, 0, st));
                    MG_TRY(launch_sgemm(waux_all, Cn, wuv + Cn, 1, no.wv, 1, 8, 1, Cn, 0, st));
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
            MG_TRY(e->alloc(reinterpret_cast<void**>(&sw->waux), 3 * 32 * 4));
            CUDA_TRY(cudaMemsetAsync(sw->waux, 0, 3 * 32 * 4, st));
            MG_TRY(launch_sgemm(wo->p, Cl, w4->p, 32, sw->waux, 32, nc, 32, Cl, 0, st));       // [nc, 32]
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

static int finalize(moge_engine* e, cudaStream_t st) {
    const moge_config_t& c = e->cfg;
    const int D = c.embed_dim;
    const std::string bb = "encoder.backbone.";
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
        b.wqkv = nullptr; b.wfc1 = nullptr;
        if (!e->ln_fold) {       // (with the LayerNorm fold only the folded copies below are ever read)
            MG_TRY(pack_linear(e, p + "attn.qkv.weight", 3 * D, D, D, &b.wqkv, st));
            MG_TRY(pack_linear(e, p + "mlp.fc1.weight", 4 * D, D, D, &b.wfc1, st));
        }
        MG_TRY(pack_linear(e, p + "attn.proj.weight", D, D, D, &b.wproj, st));
        MG_TRY(pack_linear(e, p + "mlp.fc2.weight", D, 4 * D, 4 * D, &b.wfc2, st));
        MG_TRY(vec(e, p + "attn.qkv.bias", 3 * D, &b.bqkv));
        MG_TRY(vec(e, p + "attn.proj.bias", D, &b.bproj));
        MG_TRY(vec(e, p + "mlp.fc1.bias", 4 * D, &b.bfc1));
        MG_TRY(vec(e, p + "mlp.fc2.bias", D, &b.bfc2));
        MG_TRY(vec(e, p + "ls1.gamma", D, &b.g1));
        MG_TRY(vec(e, p + "ls2.gamma", D, &b.g2));
        MG_TRY(vec(e, p + "norm1.weight", D, &b.ln1g));
        MG_TRY(vec(e, p + "norm1.bias", D, &b.ln1b));
        MG_TRY(vec(e, p + "norm2.weight", D, &b.ln2g));
        MG_TRY(vec(e, p + "norm2.bias", D, &b.ln2b));
        if (e->ln_fold) {
            const RawWeight *wq, *wf;
            MG_TRY(get_raw(e, p + "attn.qkv.weight", &wq, {}));
            MG_TRY(get_raw(e, p + "mlp.fc1.weight", &wf, {}));
            MG_TRY(e->alloc(&b.wqkv_ln, static_cast<size_t>(3 * D) * D * 2));
            MG_TRY(e->alloc(&b.wfc1_ln, static_cast<size_t>(4 * D) * D * 2));
            MG_TRY(e->alloc(reinterpret_cast<void**>(&b.b_qkv_ln), static_cast<size_t>(3 * D) * 4));
            MG_TRY(e->alloc(reinterpret_cast<void**>(&b.b_fc1_ln), static_cast<size_t>(4 * D) * 4));
            MG_TRY(launch_ln_fold(wq->p, b.ln1g, b.ln1b, b.bqkv, 3 * D, D, D, b.wqkv_ln, b.b_qkv_ln, e->bf16, st));
            MG_TRY(launch_ln_fold(wf->p, b.ln2g, b.ln2b, b.bfc1, 4 * D, D, D, b.wfc1_ln, b.b_fc1_ln, e->bf16, st));
        }
    }
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
    for (int i = 0; i < 3; ++i)
        if (head_cfg(e, i)->present) MG_TRY(pack_stack(e, head_name(i), *head_cfg(e, i), false, &e->heads[i], st));
    // neck last: its final level can be folded through the heads' last-level input/output blocks (EPI_NECKOUT) when that level
    // is a bilinear resampler + conv with no residual blocks and 32 channels (every MoGe-2 config); MOGE_B200_NECKFOLD=0 keeps
    // the 32-channel map at the 16x grid and the per-head mat-vec instead
    {
        const int L = c.neck.num_levels;
        bool any_head = false;
        for (int i = 0; i < 3; ++i) any_head |= head_cfg(e, i)->present != 0;
        const char* env = getenv("MOGE_B200_NECKFOLD");
        e->neck_fold = !(env && env[0] == '0') && any_head && L >= 2 && c.neck.resamplers[L - 2] == MOGE_RESAMPLE_BILINEAR &&
                       c.neck.num_res_blocks[L - 1] == 0 && c.neck.dim_res_blocks[L - 1] == 32 && c.neck.dim_res_blocks[L - 2] % 64 == 0;
        float* waux_all = nullptr;
        if (e->neck_fold) {
            MG_TRY(e->alloc_temp(reinterpret_cast<void**>(&waux_all), 8 * 32 * 4));
            CUDA_TRY(cudaMemsetAsync(waux_all, 0, 8 * 32 * 4, st));
            const int row_of[3] = {0, 3, 6};          // points xyz | normal xyz | mask logit | pad
            for (int i = 0; i < 3; ++i)
                if (head_cfg(e, i)->present)
                    CUDA_TRY(cudaMemcpyAsync(waux_all + row_of[i] * 32, e->heads[i].waux, static_cast<size_t>(e->heads[i].ncomp) * 32 * 4,
                                             cudaMemcpyDeviceToDevice, st));
        }
        MG_TRY(pack_stack(e, "neck", c.neck, true, &e->neck, st, waux_all));
    }
    for (int l = 0; l < c.scale_head_layers; ++l) {
        const float *w, *b;
        MG_TRY(vec(e, "scale_head." + std::to_string(2 * l) + ".weight", c.scale_head_dims[l] * c.scale_head_dims[l + 1], &w));
        MG_TRY(vec(e, "scale_head." + std::to_string(2 * l) + ".bias", c.scale_head_dims[l + 1], &b));
        e->mlp_w.push_back(w);
        e->mlp_b.push_back(b);
    }
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
                    bool uv, float su, float sv, const std::string& name, int ncomp = 0, const float* waux = nullptr, void* out2 = nullptr,
                    int accum = 0) {
    GemmLaunch g;
    MG_TRY(gemm_conv(&g, e->bf16, cw, src, aux, gs, B, epi, out_raw, out_relu, skip, go, out_ch, shuffle, uv, su, sv, ncomp, waux, out2, accum));
    const double px = static_cast<double>(B) * gs.H * gs.W;
    const double flops = 2.0 * px * cw.N * cw.Ktot;
    double bytes = px * cw.cin * 2 + px * cw.caux * 2 + static_cast<double>(cw.N) * cw.Ktot * 2;
    if (epi == EPI_HEADOUT) bytes += 4 * px * (accum ? (ncomp == 1 ? 4 : 16) : 32 * 2) + 4 * px * (ncomp == 1 ? 4 : 16);     // 4 output pixels per low-res pixel
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
                      int w, float su, float sv, StackBufs& sb, const std::vector<void*>& neck_out, void* x0_raw, void* x0_relu,
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
                const bool acc = e->neck_fold;
                MG_TRY(add_conv(e, pl, sw.headout, x_raw, nullptr, g, B, EPI_HEADOUT, lowres_out, nullptr, acc ? nullptr : neck_out[l + 1], gn, 0, false,
                                false, 0, 0, nm("conv3x3up2.headout", l + 1), sw.ncomp, acc ? nullptr : sw.waux, nullptr, acc ? 1 : 0));
                break;
            }
            if (is_neck && e->neck_fold && l + 1 == L - 1) {
                // the neck's last level goes straight into the heads' output maps (folded through their last input/output blocks)
                MG_TRY(add_conv(e, pl, sw.neckout, x_raw, nullptr, g, B, EPI_NECKOUT, neck_lowres[0], neck_lowres[1], nullptr, gn, 0, false, true, su, sv,
                                nm("conv3x3up2.neckout", l + 1), 0, nullptr, neck_lowres[2]));
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
    uint8_t* ln = static_cast<uint8_t*>(ws.take(static_cast<size_t>(M) * D * 2));          // LN output, or (LN fold) the rounded residual rows x16
    float2* stats = static_cast<float2*>(ws.take(static_cast<size_t>(M) * kStatsLd * 8));
    float* rstd = static_cast<float*>(ws.take(static_cast<size_t>(M) * 4));
    void* qkv = ws.take(static_cast<size_t>(M) * 3 * D * 2);
    void* att = ws.take(static_cast<size_t>(M) * D * 2);
    void* hid = ws.take(static_cast<size_t>(M) * 4 * D * 2);
    uint8_t* taps = static_cast<uint8_t*>(ws.take(static_cast<size_t>(TT) * c.num_taps * D * 2));
    float* cls = static_cast<float*>(ws.take(static_cast<size_t>(imgs) * D * 4));
    float* mlp_scratch = static_cast<float*>(ws.take(static_cast<size_t>(2) * imgs * 4096 * 4));
    // ---- decoder buffers: the groups run one after the other through ONE set of maps sized for the largest group
    const int L = c.neck.num_levels;
    auto alloc_stack = [&](const moge_stack_config_t& sc, StackBufs& sb) {
        sb.x_raw.assign(L, nullptr); sb.x_relu.assign(L, nullptr); sb.y_relu.assign(L, nullptr); sb.t_up.assign(L, nullptr);
        for (int l = 0; l < L; ++l) {
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
            const bool folded_last = e->neck_fold && l == L - 1;      // with the neck fold no 16x-grid feature map exists at all
            if (folded_last) continue;
            sb.x_raw[l] = ws.take(sz);
            if (sc.num_res_blocks[l] > 0) {
                sb.x_relu[l] = ws.take(sz);
                sb.y_relu[l] = ws.take(sz);
            }
            sb.t_up[l] = ws.take(szt);
        }
    };
    StackBufs nb, hb;
    alloc_stack(c.neck, nb);
    // neck outputs must survive all heads: the neck's final x per level is whichever ping-pong map holds it (kept).
    bool any_head = false;
    for (int i = 0; i < 3; ++i) any_head |= head_cfg(e, i)->present != 0;
    if (any_head) alloc_stack(*head_cfg(e, c.points_head.present ? 0 : c.normal_head.present ? 1 : 2), hb);
    // low-resolution fp32 head outputs, PER GROUP (read by the phase-2 output kernels after every group's decoder has run)
    std::vector<float4*> pts_lr(G, nullptr), nrm_lr(G, nullptr);
    std::vector<float*> msk_lr(G, nullptr);
    for (int gi = 0; gi < G; ++gi) {
        const Group& g = pl->groups[gi];
        const Level gl = level_geom(g.h, g.w, L - 1);
        const size_t px = static_cast<size_t>(g.B) * gl.H * gl.W;
        if (c.points_head.present) pts_lr[gi] = static_cast<float4*>(ws.take(px * 16));
        if (c.normal_head.present) nrm_lr[gi] = static_cast<float4*>(ws.take(px * 16));
        if (c.mask_head.present) msk_lr[gi] = static_cast<float*>(ws.take(px * 4));
    }
    if (bytes_out) *bytes_out = ws.off + 1024;
    if (dry) return 0;
    if (ws.off > pl->ws_bytes) return set_error("workspace too small: need %zu bytes, got %zu", ws.off, pl->ws_bytes);

    Plan* P = pl;
    const bool fold = e->ln_fold;
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
                          fold ? &prod : nullptr, &grid));
        pl->ops.add([=](cudaStream_t st) { return launch_init_cls(x_g, P->cls_row, B, N, D, st); }, gname("init_cls", gi));
        if (fold) {
            const int parts0 = parts_x;
            pl->ops.add([=](cudaStream_t st) {
                return launch_ln_prepare(x_g, B, static_cast<long>(N) * D, D, ln_g, static_cast<long>(N) * D, stats_g, static_cast<long>(N) * kStatsLd, parts0, bf16, st);
            }, gname("ln_prepare.cls", gi));
        }
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
        const double ln_bytes = static_cast<double>(M) * D * 6;
        if (fold) {
            if (i == 0) add_rstd(parts_x);
            LnIO cons; cons.ln_rstd = rstd;
            MG_TRY(add_linear(e, pl, ln, Mi, D, b.wqkv_ln, 3 * D, EPI_STORE16, qkv, b.b_qkv_ln, nullptr, 3 * D, "gemm.qkv", &cons));
        } else {
            pl->ops.add([=](cudaStream_t st) { return launch_layernorm(x, b.ln1g, b.ln1b, ln, Mi, D, D, 0, 0, 1, nullptr, bf16, st); }, "layernorm", 0, ln_bytes);
            MG_TRY(add_linear(e, pl, ln, Mi, D, b.wqkv, 3 * D, EPI_STORE16, qkv, b.bqkv, nullptr, 3 * D, "gemm.qkv"));
        }
        {
            CUtensorMap mq;
            MG_TRY(make_map_2d(&mq, qkv, 3 * static_cast<uint64_t>(D), M, 3 * static_cast<uint64_t>(D), 128));
            const int heads = c.num_heads;
            pl->ops.add([=](cudaStream_t st) { return launch_attention(mq, att, items_dev, ranges_dev, att_ctas, D, heads, bf16, st); }, "attention",
                        att_flops, static_cast<double>(M) * D * 8);
        }
        if (fold) {
            MG_TRY(add_linear(e, pl, att, Mi, D, b.wproj, D, EPI_RESID, x, b.bproj, b.g1, D, "gemm.proj", &prod));
            add_rstd(parts_x);
            LnIO cons; cons.ln_rstd = rstd;
            MG_TRY(add_linear(e, pl, ln, Mi, D, b.wfc1_ln, 4 * D, EPI_GELU16, hid, b.b_fc1_ln, nullptr, 4 * D, "gemm.fc1", &cons));
            MG_TRY(add_linear(e, pl, hid, Mi, 4 * D, b.wfc2, D, EPI_RESID, x, b.bfc2, b.g2, D, "gemm.fc2", (i + 1 < c.depth) ? &prod : nullptr));
            if (i + 1 < c.depth) add_rstd(parts_x);
        } else {
            MG_TRY(add_linear(e, pl, att, Mi, D, b.wproj, D, EPI_RESID, x, b.bproj, b.g1, D, "gemm.proj"));
            pl->ops.add([=](cudaStream_t st) { return launch_layernorm(x, b.ln2g, b.ln2b, ln, Mi, D, D, 0, 0, 1, nullptr, bf16, st); }, "layernorm", 0, ln_bytes);
            MG_TRY(add_linear(e, pl, ln, Mi, D, b.wfc1, 4 * D, EPI_GELU16, hid, b.bfc1, nullptr, 4 * D, "gemm.fc1"));
            MG_TRY(add_linear(e, pl, hid, Mi, 4 * D, b.wfc2, D, EPI_RESID, x, b.bfc2, b.g2, D, "gemm.fc2"));
        }
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
    // ---- decoder, group by group
    for (int gi = 0; gi < G; ++gi) {
        const Group& g = pl->groups[gi];
        const int B = g.B, H = g.H, W = g.W, h = g.h, w = g.w, T = h * w;
        const float aspect = static_cast<float>(W) / H;
        const float su = aspect / sqrtf(1.f + aspect * aspect), sv = 1.f / sqrtf(1.f + aspect * aspect);
        uint8_t* taps_g = taps + static_cast<size_t>(prow0[gi]) * c.num_taps * D * 2;
        std::vector<void*> neck_out(L, nullptr);
        // neck level 0: folded projection GEMM over the concatenated taps (+UV rank-2 term) -> padded NHWC
        {
            const Level g0 = level_geom(h, w, 0);
            const ConvW& f = e->fold0;
            if (f.Ktot % 64) return set_error("num_taps*embed_dim must be a multiple of 64");
            MG_TRY(add_linear(e, pl, taps_g, B * T, f.Ktot, f.w, f.N, EPI_DEC, nb.x_raw[0], f.bias, f.wu, f.N, gname("gemm.taps_proj", gi), nullptr,
                              &g0, c.neck.num_res_blocks[0] > 0 ? nb.x_relu[0] : nullptr, f.wv, su, sv));
        }
        void* neck_lowres[3] = {pts_lr[gi], nrm_lr[gi], msk_lr[gi]};
        const std::string sfx = G == 1 ? std::string() : ".g" + std::to_string(gi);
        MG_TRY(plan_stack(e, pl, ("neck" + sfx).c_str(), c.neck, e->neck, true, B, h, w, su, sv, nb, neck_out, nb.x_raw[0], nb.x_relu[0], nullptr, neck_lowres));
        for (int i = 0; i < 3; ++i) {
            const moge_stack_config_t& sc = *head_cfg(e, i);
            if (!sc.present) continue;
            const Level g0 = level_geom(h, w, 0);
            const StackW& sw = e->heads[i];
            MG_TRY(add_conv(e, pl, sw.in0, neck_out[0], nullptr, g0, B, EPI_DEC, hb.x_raw[0], sc.num_res_blocks[0] > 0 ? hb.x_relu[0] : nullptr,
                            nullptr, g0, sc.dim_res_blocks[0], false, false, 0, 0, std::string("conv1x1.") + head_name(i) + sfx + ".l0"));
            void* lowres = i == 0 ? static_cast<void*>(pts_lr[gi]) : i == 1 ? static_cast<void*>(nrm_lr[gi]) : static_cast<void*>(msk_lr[gi]);
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
        float4* pl_ = pts_lr[gi]; float4* nl_ = nrm_lr[gi]; float* ml_ = msk_lr[gi];
        pl->ops.add([=](cudaStream_t st) {
            const Group& gg = P->groups[gi];
            return launch_head_output(gg.points ? pl_ : nullptr, gg.normal ? nl_ : nullptr, gg.mask ? ml_ : nullptr, B, gl.H, gl.W,
                                      H, W, remap, gg.points, gg.normal, gg.mask, st);
        }, gname("head_output", gi), 0, static_cast<double>(B) * H * W * 28 + static_cast<double>(B) * gl.H * gl.W * 36, 2);
    }
    // launch order: phase 0, 1, 2 (stable)
    std::stable_sort(pl->ops.begin(), pl->ops.end(), [](const Op& a, const Op& b) { return a.phase < b.phase; });
    return 0;
}

constexpr size_t kMaxPlans = 16;

// Plans are keyed on the call shape; the workspace pointer is part of what a plan bakes in (TMA descriptors), so a call with the
// same shape but another workspace REPLACES the plan instead of orphaning it.  A plan owns its device buffers (pos tables,
// attention work list) and frees them when it is replaced or evicted (LRU) -- after the device has drained, since launches
// that read them may still be queued on the caller's stream.
static int get_plan(moge_engine* e, const moge_group_t* groups, int n, void* ws, size_t ws_bytes, Plan** out, cudaStream_t st) {
    for (size_t i = 0; i < e->plans.size(); ++i) {
        if (!e->plans[i]->same_shape(groups, n)) continue;
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
    return 0;
}

}  // namespace mg

// ================================================================================================ C ABI
extern "C" {

const char* moge_last_error(void) { return mg::last_error(); }
const char* moge_version(void) { return "moge_b200 0.1.0 sm_90a"; }

int moge_engine_create(const moge_config_t* cfg, int device, moge_engine_t** out) {
    if (!cfg || !out) return set_error("null argument");
    MG_TRY(validate_cfg(*cfg));
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) return set_error("no CUDA device: moge_b200 has no CPU fallback");
    CUDA_TRY(cudaSetDevice(device));
    cudaDeviceProp prop;
    CUDA_TRY(cudaGetDeviceProperties(&prop, device));
    if (prop.major != 9 || prop.minor != 0) return set_error("device %d is sm_%d%d; libmoge_b200 contains sm_90a code only", device, prop.major, prop.minor);
    moge_engine* e = new moge_engine();
    e->cfg = *cfg; e->device = device; e->num_sms = prop.multiProcessorCount; e->bf16 = cfg->compute_dtype == MOGE_BF16;
    const char* env = getenv("MOGE_B200_GRAPHS");
    e->use_graphs = !(env && env[0] == '0');
    const char* env3 = getenv("MOGE_B200_LNFOLD");
    e->ln_fold = !(env3 != nullptr && env3[0] == '0');
    if (cudaStreamCreateWithFlags(&e->own_stream, cudaStreamNonBlocking) != cudaSuccess ||
        cudaEventCreateWithFlags(&e->ev_in, cudaEventDisableTiming) != cudaSuccess ||
        cudaEventCreateWithFlags(&e->ev_out, cudaEventDisableTiming) != cudaSuccess) {
        delete e;
        return set_error("stream/event creation failed");
    }
    *out = e;
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
    // squeeze leading singleton dims of parameter-like tensors so shape checks see the logical shape
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

int moge_engine_forward_groups(moge_engine_t* e, const moge_group_t* groups, int n, void* workspace, size_t workspace_bytes, void* stream) {
    if (!e || !workspace) return set_error("null argument");
    if (!e->finalized) return set_error("engine not finalized");
    MG_TRY(check_groups(e, groups, n, true));
    if (reinterpret_cast<uintptr_t>(workspace) & 1023) return set_error("workspace must be 1024-byte aligned");
    CUDA_TRY(cudaSetDevice(e->device));
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    Plan* pl;
    MG_TRY(get_plan(e, groups, n, workspace, workspace_bytes, &pl, st));
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
    const bool want_graph = e->use_graphs && tokens <= 4 * 3600;
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

}  // extern "C"
