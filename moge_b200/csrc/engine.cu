// Host runtime of libmoge_b200.so: per-shape execution plans (workspace layout, TMA descriptors, launch list), graph replay, and
// the extern "C" ABI declared in include/moge_b200.h except the weight loading (weights.cu).
#include "engine.h"
#include "gemm_kernel.cuh"

#include <algorithm>
#include <functional>
#include <memory>
#include <string>
#include <vector>
#include <math.h>

namespace mg {

const char* last_error();

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
    float* tokens = nullptr; float* cls_out = nullptr; float* prenorm = nullptr;     // DINOv2 backbone outputs (moge_dino_forward_groups)
};

// What a DINOv2 backbone plan exports besides its shape: the blocks whose rows it writes (increasing) and the MOGE_DINO_* flags
struct DinoKey {
    std::vector<int> layers;
    int flags = 0;
    bool operator==(const DinoKey& o) const { return layers == o.layers && flags == o.flags; }
};

// The group a public group struct describes, with its bindings
static Group make_group(const moge_group_t& m) {
    Group g;
    g.B = m.B; g.H = m.H; g.W = m.W; g.h = m.h; g.w = m.w;
    g.image = m.image; g.image_dtype = m.image_dtype; g.points = m.points; g.normal = m.normal; g.mask = m.mask_prob; g.scale = m.metric_scale;
    return g;
}

static Group make_group(const moge_v1_group_t& m) {     // MoGe-1: the token grid of the resized image, rh/14 x rw/14
    Group g;
    g.B = m.B; g.H = m.H; g.W = m.W; g.h = m.rh / 14; g.w = m.rw / 14; g.rh = m.rh; g.rw = m.rw;
    g.image = m.image; g.image_dtype = m.image_dtype; g.points = m.points; g.mask = m.mask;
    return g;
}

struct Plan {
    std::vector<Group> groups;
    DinoKey dino;                  // a DINOv2 backbone plan's exports (empty for the MoGe engines)
    void* ws = nullptr;
    size_t ws_bytes = 0;
    OpList ops;                    // in launch order: all phase-0 ops, then phase 1, then phase 2
    std::vector<void*> owned;      // device buffers that live and die with the plan (pos tables, cls row, attention work list)
    float* cls_row = nullptr;
    AttnWork att;
    // ONE CUDA graph of the phase-1 launches (they touch nothing but the workspace the plan is keyed on, so the graph never
    // goes stale when the caller passes fresh input / output tensors): the launch list of a single image is ~240 kernels of a
    // few microseconds each and replaying a graph removes the per-launch CPU cost.  Phase 0 / 2 launches run eagerly around it.
    cudaGraphExec_t exec = nullptr;
    int eager_runs = 0;
    bool same_shape(const std::vector<Group>& g) const {
        return std::equal(groups.begin(), groups.end(), g.begin(), g.end(), [](const Group& a, const Group& b) {
            return a.B == b.B && a.H == b.H && a.W == b.W && a.h == b.h && a.w == b.w && a.rh == b.rh && a.rw == b.rw;
        });
    }
    int alloc(void** p, size_t bytes) { CUDA_TRY(cudaMalloc(p, bytes)); owned.push_back(*p); return 0; }
    ~Plan() {
        if (exec) cudaGraphExecDestroy(exec);
        for (void* p : owned) cudaFree(p);
    }
};

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

static size_t map_bytes(const Level& g, int B, int C) { return static_cast<size_t>(B) * g.Hp * g.Wp * C * 2; }

// conv-type launch on padded NHWC maps. src/aux/skip/out buffers live in the workspace.
static int add_conv(moge_engine* e, Plan* pl, const ConvArgs& a, const std::string& name) {
    GemmLaunch g;
    MG_TRY(gemm_conv(&g, e->bf16, a));
    const ConvW& cw = a.cw;
    const double px = static_cast<double>(a.B) * a.gs.H * a.gs.W;
    const double flops = 2.0 * px * cw.N * cw.Ktot;
    double bytes = px * cw.cin * 2 + px * cw.caux * 2 + static_cast<double>(cw.N) * cw.Ktot * 2;
    // 4 output pixels per low-res pixel, each read (the neck's part) and written
    if (a.epi == EPI_HEADOUT) bytes += 2 * (4 * px * (a.ncomp == 1 ? 4 : 16));
    else if (a.epi == EPI_NECKOUT) bytes += 4 * px * ((a.out_raw ? 16 : 0) + (a.out_relu ? 16 : 0) + (a.out2 ? 4 : 0));
    else bytes += px * cw.N * 2 * ((a.out_raw ? 1 : 0) + (a.out_relu ? 1 : 0)) + (a.skip ? px * cw.N * 2 : 0);
    pl->ops.add([g, sms = e->num_sms](cudaStream_t st) { return launch_gemm(g, sms, st); }, name, flops, bytes);
    return 0;
}

// Linear over row-major A [M, K] with the engine's packed (dense [N, K]) weight W.
static int add_linear(moge_engine* e, Plan* pl, const LinearArgs& a, const std::string& name) {
    GemmLaunch g;
    MG_TRY(gemm_linear(&g, e->bf16, a));
    const double M = a.M, N = a.N, K = a.K;
    const double flops = 2.0 * M * N * K;
    double bytes = M * K * 2 + N * K * 2;
    bytes += (a.epi == EPI_RESID) ? M * N * 8 : (a.epi == EPI_PATCH) ? M * N * 4 + static_cast<double>(g.p.T) * N * 4 : M * N * 2;
    if (a.ln && a.ln->x16) bytes += M * N * 2;
    pl->ops.add([g, sms = e->num_sms](cudaStream_t st) { return launch_gemm(g, sms, st); }, name, flops, bytes);
    return 0;
}

struct StackBufs {     // per-level scratch maps of one ConvStack
    std::vector<void*> x_raw, x_relu, y_relu, t_up;
};

// What plan_stack reads: one ConvStack (the neck or a head) of one shape group.
struct StackIn {
    std::string name;
    const moge_stack_config_t* sc = nullptr;
    const StackW* sw = nullptr;
    int B = 0, h = 0, w = 0;                // batch and token grid
    float su = 0.f, sv = 0.f;               // UV half extents
    const StackBufs* sb = nullptr;          // scratch maps; level 0 holds the input (x_raw[0], its ReLU x_relu[0])
    void* const* neck_maps = nullptr;       // a head: the neck's per-level outputs, the sources of its input blocks
};

// The neck writes its per-level output maps to neck_out[l]; a head passes null.  `lowres`: the fp32 low-resolution output maps the
// last launch writes (a head: its own; the neck: points, normal and mask).
static int plan_stack(moge_engine* e, Plan* pl, const StackIn& in, void** neck_out, void* const* lowres) {
    const moge_stack_config_t& sc = *in.sc;
    const StackW& sw = *in.sw;
    const StackBufs& sb = *in.sb;
    const bool is_neck = neck_out != nullptr;
    const int L = sc.num_levels, B = in.B;
    const int* C = sc.dim_res_blocks;
    void* x_raw = sb.x_raw[0];
    void* x_relu = sb.x_relu[0];
    auto nm = [&](const char* kind, int l) { return std::string(kind) + "." + in.name + ".l" + std::to_string(l); };
    for (int l = 0; l < L; ++l) {
        const Level g = level_geom(in.h, in.w, l);
        const int nres = sc.num_res_blocks[l];
        ConvArgs res; res.B = B; res.gs = res.go = g; res.out_ch = C[l]; res.epi = EPI_DEC;        // the residual blocks' convs
        for (int r = 0; r < nres; ++r) {
            // y = conv3(relu(x)) -> only relu(y) is ever consumed
            ConvArgs ra = res; ra.cw = sw.res[l][2 * r]; ra.src = x_relu; ra.out_relu = sb.y_relu[l];
            MG_TRY(add_conv(e, pl, ra, nm("conv3x3.res_a", l)));
            // x = x + conv3(relu(y))
            void* nraw = (x_raw == sb.x_raw[l]) ? sb.t_up[l] : sb.x_raw[l];     // ping-pong between two raw maps
            ConvArgs rb = res; rb.cw = sw.res[l][2 * r + 1]; rb.src = sb.y_relu[l]; rb.skip = x_raw;
            rb.out_raw = nraw; rb.out_relu = (r + 1 < nres) ? x_relu : nullptr;
            MG_TRY(add_conv(e, pl, rb, nm("conv3x3.res_b", l)));
            x_raw = nraw;
        }
        if (is_neck) neck_out[l] = x_raw;
        if (l == L - 1) break;
        const Level gn = level_geom(in.h, in.w, l + 1);
        const bool tail = !is_neck && (l + 1 == L - 1);
        ConvArgs a; a.B = B; a.go = gn; a.epi = EPI_DEC;     // the level's 3x3 conv: after the convT, or with the bilinear x2 folded in
        const char* kind = "conv3x3.post";
        if (sc.resamplers[l] == MOGE_RESAMPLE_CONV_TRANSPOSE) {
            ConvArgs ct = a; ct.cw = sw.convT[l]; ct.src = x_raw; ct.gs = g; ct.out_ch = C[l + 1]; ct.out_raw = sb.t_up[l + 1]; ct.shuffle = true;
            MG_TRY(add_conv(e, pl, ct, nm("convT", l)));
            if (tail) return set_error("%s: the last resampler must be bilinear", in.name.c_str());
            a.src = sb.t_up[l + 1]; a.gs = gn;
            if (!is_neck) a.aux = in.neck_maps[l + 1];
        } else {
            // bilinear x2 + 3x3 conv run as ONE low-resolution conv with 4 output phases (weights expanded at load time)
            a.src = x_raw; a.gs = g;
            if (tail) {
                a.cw = sw.headout; a.epi = EPI_HEADOUT; a.out_raw = lowres[0]; a.ncomp = sw.ncomp;
                MG_TRY(add_conv(e, pl, a, nm("conv3x3up2.headout", l + 1)));
                break;
            }
            if (is_neck && l + 1 == L - 1) {
                // the neck's last level goes straight into the heads' output maps (folded through their last input/output blocks)
                a.cw = sw.neckout; a.epi = EPI_NECKOUT; a.out_raw = lowres[0]; a.out_relu = lowres[1]; a.out2 = lowres[2];
                a.uv = true; a.su = in.su; a.sv = in.sv;
                MG_TRY(add_conv(e, pl, a, nm("conv3x3up2.neckout", l + 1)));
                break;
            }
            a.shuffle = true;
            kind = "conv3x3up2.post";
        }
        a.cw = sw.post[l]; a.out_ch = C[l + 1]; a.uv = is_neck; a.su = in.su; a.sv = in.sv;
        a.out_raw = sb.x_raw[l + 1]; a.out_relu = sc.num_res_blocks[l + 1] > 0 ? sb.x_relu[l + 1] : nullptr;
        MG_TRY(add_conv(e, pl, a, nm(kind, l + 1)));
        x_raw = sb.x_raw[l + 1];
        x_relu = sb.x_relu[l + 1];
    }
    return 0;
}

// ---- MoGe-1 decoder: the groups run one after the other through ONE set of maps sized for the largest group
struct V1Bufs {
    float *rs_tmp = nullptr, *rs_img = nullptr;     // bicubic row pass (B,3,H,rw), resized image (B,3,rh,rw)
    void* x0 = nullptr;                             // projected taps, level 0
    struct Lv { void *m0, *m1, *relu, *hraw, *hrelu; };
    std::vector<Lv> lv;                             // per upsampling level (its output grid): ping-pong maps, ReLU maps
    double2* gn_part = nullptr;
    float2* gn_stats = nullptr;
    void *full = nullptr, *fout = nullptr;          // last map resized to (rh, rw); the output conv's 64 channels there
    std::vector<float4*> pts;                       // per group: (rh, rw) points before the resize to (H, W)
    std::vector<float*> msk;                        // per group: (rh, rw) mask logits
};

static Level full_geom(int rh, int rw) { return Level{rh, rw, std::max(rh + 2, TILE_PH), std::max(rw + 2, TILE_PW)}; }

static void v1_alloc(moge_engine* e, const Plan* pl, WsAlloc& ws, V1Bufs* vb) {
    const moge_v1_config_t& c = e->v1cfg;
    const int L = c.num_levels;
    // the largest size any group needs, of each map
    auto most = [&](const std::function<size_t(const Group&)>& f) {
        size_t m = 0;
        for (const Group& g : pl->groups) m = std::max(m, f(g));
        return m;
    };
    // one resize scratch for every group: the phase-0 resize -> preprocess pairs are issued group by group on one stream, so a
    // group's resize only overwrites the scratch after the previous group's preprocess has read it
    vb->rs_tmp = static_cast<float*>(ws.take(most([](const Group& g) { return static_cast<size_t>(g.B) * 3 * g.H * g.rw * 4; })));
    vb->rs_img = static_cast<float*>(ws.take(most([](const Group& g) { return static_cast<size_t>(g.B) * 3 * g.rh * g.rw * 4; })));
    vb->x0 = ws.take(most([&](const Group& g) { return map_bytes(level_geom(g.h, g.w, 0), g.B, c.dim_proj); }));
    vb->lv.resize(L);
    for (int l = 0; l < L; ++l) {
        const int Co = c.dim_upsample[l], Hd = c.hidden_mult * Co;
        auto bytes = [&](int C) { return most([&](const Group& g) { return map_bytes(level_geom(g.h, g.w, l + 1), g.B, C); }); };
        V1Bufs::Lv& m = vb->lv[l];
        m.m0 = ws.take(bytes(Co));
        m.m1 = ws.take(bytes(Co));
        m.relu = ws.take(bytes(Co));
        m.hraw = ws.take(bytes(Hd));
        m.hrelu = ws.take(bytes(Hd));
    }
    const size_t part = most([&](const Group& g) {
        size_t p = 0;
        for (int l = 0; l < L; ++l) {
            const Level go = level_geom(g.h, g.w, l + 1);
            const int Co = c.dim_upsample[l], Hd = c.hidden_mult * Co;
            const int G2 = c.hidden_norm == MOGE_V1_GROUP_NORM ? Hd / 32 : 1;
            p = std::max({p, static_cast<size_t>(g.B) * gn_tiles(go.H, go.W, Co), static_cast<size_t>(g.B) * gn_tiles(go.H, go.W, Hd) * G2});
        }
        return p;
    });
    const size_t stats = most([&](const Group& g) {
        size_t s = 0;
        for (int l = 0; l < L; ++l) {
            const int Hd = c.hidden_mult * c.dim_upsample[l];
            s = std::max(s, static_cast<size_t>(g.B) * (c.hidden_norm == MOGE_V1_GROUP_NORM ? Hd / 32 : 1));
        }
        return s;
    });
    vb->gn_part = static_cast<double2*>(ws.take(part * 16));
    vb->gn_stats = static_cast<float2*>(ws.take(stats * 8));
    vb->full = ws.take(most([&](const Group& g) { return map_bytes(full_geom(g.rh, g.rw), g.B, c.dim_upsample[L - 1]); }));
    vb->fout = ws.take(most([&](const Group& g) { return map_bytes(full_geom(g.rh, g.rw), g.B, 2 * c.last_conv_channels); }));
    // per group: the phase-2 output resizes read them after every group's decoder has run
    for (const Group& g : pl->groups) {
        vb->pts.push_back(static_cast<float4*>(ws.take(static_cast<size_t>(g.B) * g.rh * g.rw * 16)));
        vb->msk.push_back(static_cast<float*>(ws.take(static_cast<size_t>(g.B) * g.rh * g.rw * 4)));
    }
}

// MoGe-1 decoder launch list, group by group; group gi's encoder taps start at row prow0[gi] of `taps`.
static int plan_v1_decoder(moge_engine* e, Plan* pl, const uint8_t* taps, const std::vector<long>& prow0, const V1Bufs& vb) {
    const moge_v1_config_t& c = e->v1cfg;
    const V1W& v = e->v1w;
    const int G = static_cast<int>(pl->groups.size());
    const bool bf16 = e->bf16;
    Plan* P = pl;
    for (int gi = 0; gi < G; ++gi) {
        const Group& g = pl->groups[gi];
        const int B = g.B, H = g.H, W = g.W, h = g.h, w = g.w, rh = g.rh, rw = g.rw;
        const std::string sfx = G == 1 ? std::string() : ".g" + std::to_string(gi);
        // every UV plane of the head has the aspect of the resized image (v1.py:125, 133)
        const float aspect = static_cast<float>(rw) / rh;
        const float su = aspect / sqrtf(1.f + aspect * aspect), sv = 1.f / sqrtf(1.f + aspect * aspect);
        const Level g0 = level_geom(h, w, 0);
        LinearArgs proj; proj.A = taps + static_cast<size_t>(prow0[gi]) * e->cfg.num_taps * e->cfg.embed_dim * 2; proj.M = B * h * w; proj.K = v.proj.Ktot;
        proj.W = v.proj.w; proj.N = v.proj.N; proj.epi = EPI_DEC; proj.out = vb.x0; proj.bias = v.proj.bias; proj.grid = &g0;
        MG_TRY(add_linear(e, pl, proj, "gemm.projects" + sfx));
        const void* x = vb.x0;
        double2* part = vb.gn_part;
        float2* stats = vb.gn_stats;
        auto nm = [&](const char* kind, int l) { return std::string(kind) + sfx + ".l" + std::to_string(l); };
        auto add_gn = [&](const void* src, void* dst, const Level& gl, int C, int G2, const float* gamma, const float* beta, int l) {
            const double px = static_cast<double>(B) * gl.H * gl.W;
            pl->ops.add([=](cudaStream_t st) { return launch_gn_stats(src, gl, B, C, G2, part, stats, bf16, st); }, nm("groupnorm_stats", l), 0,
                        px * C * 2);
            pl->ops.add([=](cudaStream_t st) { return launch_gn_relu(src, dst, gl, B, C, G2, stats, gamma, beta, bf16, st); }, nm("groupnorm_relu", l), 0,
                        px * C * 4);
        };
        for (int l = 0; l < c.num_levels; ++l) {
            const V1Level& L = v.lv[l];
            const V1Bufs::Lv& m = vb.lv[l];
            const int Co = c.dim_upsample[l], Hd = c.hidden_mult * Co;
            const Level gin = level_geom(h, w, l), go = level_geom(h, w, l + 1);
            ConvArgs lv; lv.B = B; lv.gs = lv.go = go; lv.out_ch = Co; lv.epi = EPI_DEC;        // the level's convs on its output grid
            ConvArgs ct = lv; ct.cw = L.convT; ct.src = x; ct.gs = gin; ct.out_raw = m.m1; ct.shuffle = true;
            MG_TRY(add_conv(e, pl, ct, nm("convT", l)));
            const float* wuv = L.wuv;
            void* t = m.m1;
            pl->ops.add([=](cudaStream_t st) { return launch_uv_convT(t, go, B, Co, wuv, su, sv, bf16, st); }, nm("uv_convT", l), 0,
                        static_cast<double>(B) * go.H * go.W * Co * 4);
            ConvArgs cv = lv; cv.cw = L.conv; cv.src = m.m1; cv.out_raw = m.m0;
            MG_TRY(add_conv(e, pl, cv, nm("conv3x3", l)));
            void* xr = m.m0;
            void* other = m.m1;
            for (const V1Res& R : L.res) {
                add_gn(xr, m.relu, go, Co, 1, R.g1, R.b1, l);
                ConvArgs ra = lv; ra.cw = R.c1; ra.src = m.relu; ra.out_ch = Hd; ra.out_raw = m.hraw;
                MG_TRY(add_conv(e, pl, ra, nm("conv3x3.res_a", l)));
                add_gn(m.hraw, m.hrelu, go, Hd, R.G2, R.g2, R.b2, l);
                ConvArgs rb = lv; rb.cw = R.c2; rb.src = m.hrelu; rb.out_raw = other; rb.skip = xr;
                MG_TRY(add_conv(e, pl, rb, nm("conv3x3.res_b", l)));
                std::swap(xr, other);
            }
            x = xr;
        }
        // V7: bilinear resize to the resized-image grid, both output blocks' 3x3 conv, then their UV part, ReLU and 1x1 convs
        const int Cl = c.dim_upsample[c.num_levels - 1];
        const Level gl = level_geom(h, w, c.num_levels), gr = full_geom(rh, rw);
        const double pxr = static_cast<double>(B) * rh * rw;
        void* full = vb.full;
        pl->ops.add([=](cudaStream_t st) { return launch_resize_bilinear_nhwc(x, gl, full, gr, B, Cl, bf16, st); }, "resize_bilinear" + sfx, 0,
                    static_cast<double>(B) * gl.H * gl.W * Cl * 2 + pxr * Cl * 2);
        ConvArgs oc; oc.cw = v.out; oc.src = vb.full; oc.gs = oc.go = gr; oc.B = B; oc.out_ch = v.out.N; oc.epi = EPI_DEC; oc.out_raw = vb.fout;
        MG_TRY(add_conv(e, pl, oc, "conv3x3.output" + sfx));
        const void* fout = vb.fout;
        const float* wout = v.wout;
        float4* pts = vb.pts[gi];
        float* msk = vb.msk[gi];
        pl->ops.add([=](cudaStream_t st) { return launch_v1_output(fout, gr, B, wout, su, sv, pts, msk, bf16, st); }, "output_block" + sfx,
                    2.0 * pxr * 64 * 10, pxr * (64 * 2 + 20));
        // V8 (phase 2: the caller's outputs): bilinear resize to (H, W), remap; the mask stays a raw logit
        const int remap = c.remap_output;
        pl->ops.add([=](cudaStream_t st) {
            return launch_head_output(pts, nullptr, msk, B, rh, rw, H, W, remap, P->groups[gi].points, nullptr, P->groups[gi].mask, st, false);
        }, "head_output" + sfx, 0, static_cast<double>(B) * H * W * 16 + pxr * 20, 2);
    }
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
        // neck level 0: folded projection GEMM over the concatenated taps (+UV rank-2 term) -> padded NHWC
        const Level g0 = level_geom(h, w, 0);
        const ConvW& f = e->fold0;
        if (f.Ktot % 64) return set_error("num_taps*embed_dim must be a multiple of 64");
        LinearArgs tp; tp.A = taps_g; tp.M = B * T; tp.K = f.Ktot; tp.W = f.w; tp.N = f.N; tp.epi = EPI_DEC; tp.grid = &g0;
        tp.out = nb.x_raw[0]; tp.out_relu = c.neck.num_res_blocks[0] > 0 ? nb.x_relu[0] : nullptr;
        tp.bias = f.bias; tp.v1 = f.wu; tp.v2 = f.wv; tp.su = su; tp.sv = sv;
        MG_TRY(add_linear(e, pl, tp, gname("gemm.taps_proj", gi)));
        void* lowres[3] = {v.pts_lr[gi], v.nrm_lr[gi], v.msk_lr[gi]};
        const std::string sfx = G == 1 ? std::string() : ".g" + std::to_string(gi);
        std::vector<void*> neck_out(L, nullptr);
        StackIn in; in.B = B; in.h = h; in.w = w; in.su = su; in.sv = sv;
        in.name = "neck" + sfx; in.sc = &c.neck; in.sw = &e->neck; in.sb = &nb;
        MG_TRY(plan_stack(e, pl, in, neck_out.data(), lowres));
        in.sb = &hb; in.neck_maps = neck_out.data();
        for (int i = 0; i < 3; ++i) {
            const moge_stack_config_t& sc = *head_cfg(e, i);
            if (!sc.present) continue;
            in.name = head_name(i) + sfx; in.sc = &sc; in.sw = &e->heads[i];
            ConvArgs a; a.cw = e->heads[i].in0; a.src = neck_out[0]; a.gs = a.go = g0; a.B = B; a.out_ch = sc.dim_res_blocks[0]; a.epi = EPI_DEC;
            a.out_raw = hb.x_raw[0]; a.out_relu = sc.num_res_blocks[0] > 0 ? hb.x_relu[0] : nullptr;
            MG_TRY(add_conv(e, pl, a, "conv1x1." + in.name + ".l0"));
            MG_TRY(plan_stack(e, pl, in, nullptr, lowres + i));
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

// DINOv2 backbone outputs (phase 2: the caller's buffers, bound per call): each exported block's rows from the snapshot taken after
// it, or from the stream itself for the last block, through the final LayerNorm or raw, one launch over every group; then the
// pre-norm stream, one copy per group (a group's rows are contiguous, each image's class row first).
static int plan_dino_outputs(moge_engine* e, Plan* pl, const float* x, const std::vector<float*>& snaps) {
    const int D = e->cfg.embed_dim, depth = e->cfg.depth;
    const int G = static_cast<int>(pl->groups.size());
    const bool norm = pl->dino.flags & MOGE_DINO_NORM, chw = pl->dino.flags & MOGE_DINO_CHANNEL_MAJOR;
    const float* ng = norm ? e->norm_g : nullptr;
    const float* nb = norm ? e->norm_b : nullptr;
    Plan* P = pl;
    long M = 0;
    for (const Group& g : pl->groups) M += static_cast<long>(g.B) * (g.h * g.w + 1);
    size_t s = 0;
    for (size_t j = 0; j < pl->dino.layers.size(); ++j) {
        const float* src = pl->dino.layers[j] == depth - 1 ? x : snaps[s++];
        pl->ops.add([=](cudaStream_t st) {
            DinoExportOut outs[MOGE_DINO_MAX_GROUPS];
            for (int gi = 0; gi < G; ++gi) {
                const Group& g = P->groups[gi];
                const int T = g.h * g.w;
                outs[gi].B = g.B; outs[gi].N = T + 1;
                outs[gi].tokens = g.tokens ? g.tokens + j * static_cast<size_t>(g.B) * T * D : nullptr;
                outs[gi].cls = g.cls_out ? g.cls_out + j * static_cast<size_t>(g.B) * D : nullptr;
            }
            return launch_dino_export(src, outs, G, D, ng, nb, chw, st);
        }, chw ? "dino_export_chw" : "dino_export", 0, static_cast<double>(M) * D * 8, 2);
    }
    pl->ops.add([=](cudaStream_t st) {
        for (const Group& g : P->groups)
            if (g.prenorm)
                CUDA_TRY(cudaMemcpyAsync(g.prenorm, x + static_cast<size_t>(g.row0) * D, static_cast<size_t>(g.B) * (g.h * g.w + 1) * D * 4,
                                         cudaMemcpyDeviceToDevice, st));
        return 0;
    }, "dino_prenorm", 0, static_cast<double>(M) * D * 8, 2);
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
    std::vector<float*> snaps;      // DINOv2 backbone: the residual stream after each exported block but the last
    if (e->dino) {
        for (int l : pl->dino.layers)
            if (l != c.depth - 1) snaps.push_back(static_cast<float*>(ws.take(static_cast<size_t>(M) * D * 4)));
    } else if (e->v1) {
        v1_alloc(e, pl, ws, &vb);
    } else {
        alloc_v2_decoder(e, pl, ws, &v2b);
    }
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
        if (e->dino) {           // one front-end launch over every group, below
            prow += static_cast<long>(B) * T;
            continue;
        }
        if (e->v1) {
            // MoGe-1 (v1.py:273-279): antialiased bicubic resize to (rh, rw), then the same normalise + aa-bilinear resize to
            // (14h, 14w) + patchify as MoGe-2 (normalising after the second resize instead of between the two commutes: both
            // resizes are convex combinations per channel and the normalisation is a per-channel affine map)
            const int rh = g.rh, rw = g.rw;
            float *tmp = vb.rs_tmp, *img = vb.rs_img;
            pl->ops.add([=](cudaStream_t st) { return launch_resize_bicubic_aa(P->groups[gi].image, P->groups[gi].image_dtype, B, 3, H, W, rh, rw, tmp, img, st); },
                        gname("resize_bicubic_aa", gi), 0, static_cast<double>(B) * 3 * (static_cast<double>(H) * W * 4 + static_cast<double>(H) * rw * 8 + static_cast<double>(rh) * rw * 4), 0);
            pl->ops.add([=](cudaStream_t st) { return launch_preprocess(img, MOGE_F32, B, rh, rw, h, w, patches_g, 592, bf16, st); },
                        gname("preprocess", gi), 0, static_cast<double>(B) * 3 * rh * rw * 4 + static_cast<double>(B) * T * 592 * 2, 0);
            prow += static_cast<long>(B) * T;
            continue;
        }
        pl->ops.add([=](cudaStream_t st) { return launch_preprocess(P->groups[gi].image, P->groups[gi].image_dtype, B, H, W, h, w, patches_g, 592, bf16, st); },
                    gname("preprocess", gi), 0, static_cast<double>(B) * 3 * H * W * 4 + static_cast<double>(B) * T * 592 * 2, 0);
        prow += static_cast<long>(B) * T;
    }
    if (e->dino) {
        // the backbone's input is already normalised and a whole number of patches: no resize, no mean / std.  Each group's image
        // is read in its own dtype and shape into its patch rows.
        double bytes = 0;
        for (const Group& g : pl->groups) bytes += static_cast<double>(g.B) * 3 * g.H * g.W * 4 + static_cast<double>(g.B) * g.h * g.w * 592 * 2;
        pl->ops.add([=](cudaStream_t st) {
            DinoPatchIn in[MOGE_DINO_MAX_GROUPS];
            for (int gi = 0; gi < G; ++gi) {
                const Group& g = P->groups[gi];
                in[gi].image = g.image; in[gi].image_dtype = g.image_dtype; in[gi].B = g.B; in[gi].H = g.H; in[gi].W = g.W;
            }
            return launch_dino_patchify(in, G, patches, bf16, st);
        }, "dino_patchify", 0, bytes, 0);
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
        LinearArgs a; a.A = patches_g; a.M = B * T; a.K = 592; a.W = e->w_patch; a.N = D; a.epi = EPI_PATCH;
        a.out = x_g; a.v1 = g.pos_table; a.ln = &prod; a.grid = &grid;
        MG_TRY(add_linear(e, pl, a, gname("gemm.patch_embed", gi)));
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
        std::vector<int> n;
        for (const auto& g : pl->groups) n.insert(n.end(), g.B, g.h * g.w + 1);
        MG_TRY(upload_attention_work(n, c.num_heads, sms, [pl](void** p, size_t bytes) { return pl->alloc(p, bytes); }, upload_stream, &pl->att));
    }
    const AttnItem* items_dev = pl->att.items_dev; const int2* ranges_dev = pl->att.ranges_dev;
    const int att_ctas = static_cast<int>(pl->att.ranges.size());
    double att_flops = 0;
    for (const auto& g : pl->groups) { const double N = g.h * g.w + 1; att_flops += 4.0 * g.B * N * N * D; }
    // ---- transformer blocks: ONE launch per linear / attention over the packed rows of every group
    int tap_idx = 0;
    for (int i = 0; i < c.depth; ++i) {
        const moge_engine::Blk& b = e->blk[i];
        if (i == 0) add_rstd(parts_x);
        LnIO cons; cons.ln_rstd = rstd;
        LinearArgs a; a.A = ln; a.M = Mi; a.K = D; a.W = b.wqkv_ln; a.N = 3 * D; a.epi = EPI_STORE16; a.out = qkv; a.bias = b.b_qkv_ln; a.ln = &cons;
        MG_TRY(add_linear(e, pl, a, "gemm.qkv"));
        {
            CUtensorMap mq;
            MG_TRY(make_map_2d(&mq, qkv, 3 * static_cast<uint64_t>(D), M, 3 * static_cast<uint64_t>(D), 128));
            const int heads = c.num_heads;
            pl->ops.add([=](cudaStream_t st) { return launch_attention(mq, att, items_dev, ranges_dev, att_ctas, D, heads, bf16, st); }, "attention",
                        att_flops, static_cast<double>(M) * D * 8);
        }
        a = LinearArgs(); a.A = att; a.M = Mi; a.K = D; a.W = b.wproj; a.N = D; a.epi = EPI_RESID; a.out = x; a.bias = b.bproj; a.v1 = b.g1; a.ln = &prod;
        MG_TRY(add_linear(e, pl, a, "gemm.proj"));
        add_rstd(parts_x);
        a = LinearArgs(); a.A = ln; a.M = Mi; a.K = D; a.W = b.wfc1_ln; a.N = 4 * D; a.epi = EPI_GELU16; a.out = hid; a.bias = b.b_fc1_ln; a.ln = &cons;
        MG_TRY(add_linear(e, pl, a, "gemm.fc1"));
        a = LinearArgs(); a.A = hid; a.M = Mi; a.K = 4 * D; a.W = b.wfc2; a.N = D; a.epi = EPI_RESID; a.out = x; a.bias = b.bfc2; a.v1 = b.g2;
        a.ln = (i + 1 < c.depth) ? &prod : nullptr;
        MG_TRY(add_linear(e, pl, a, "gemm.fc2"));
        if (i + 1 < c.depth) add_rstd(parts_x);
        if (e->dino && i + 1 < c.depth && std::find(pl->dino.layers.begin(), pl->dino.layers.end(), i) != pl->dino.layers.end()) {
            // the rows the export reads after the last block are overwritten by the next one: keep a copy (phase 1, workspace only)
            float* dst = snaps[std::find(pl->dino.layers.begin(), pl->dino.layers.end(), i) - pl->dino.layers.begin()];
            const size_t bytes = static_cast<size_t>(M) * D * 4;
            pl->ops.add([=](cudaStream_t st) { CUDA_TRY(cudaMemcpyAsync(dst, x, bytes, cudaMemcpyDeviceToDevice, st)); return 0; },
                        "dino_snapshot", 0, 2.0 * bytes);
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
    if (e->dino) MG_TRY(plan_dino_outputs(e, pl, x, snaps));
    else MG_TRY(e->v1 ? plan_v1_decoder(e, pl, taps, prow0, vb) : plan_v2_decoder(e, pl, taps, prow0, cls, mlp_scratch, v2b));
    // launch order: phase 0, 1, 2 (stable)
    std::stable_sort(pl->ops.begin(), pl->ops.end(), [](const Op& a, const Op& b) { return a.phase < b.phase; });
    return 0;
}

constexpr size_t kMaxPlans = 16;

// Plans are keyed on the call shape; the workspace pointer is part of what a plan bakes in (TMA descriptors), so a call with the
// same shape but another workspace REPLACES the plan instead of orphaning it.  A plan owns its device buffers (pos tables,
// attention work list) and frees them when it is replaced or evicted (LRU) -- after the device has drained, since launches
// that read them may still be queued on the caller's stream.
static int get_plan(moge_engine* e, const std::vector<Group>& groups, const DinoKey& dino, void* ws, size_t ws_bytes, Plan** out,
                    cudaStream_t st) {
    for (size_t i = 0; i < e->plans.size(); ++i) {
        if (!e->plans[i]->same_shape(groups) || !(e->plans[i]->dino == dino)) continue;
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
    pl->ws = ws; pl->ws_bytes = ws_bytes; pl->dino = dino;
    const int D = e->cfg.embed_dim;
    MG_TRY(pl->alloc(reinterpret_cast<void**>(&pl->cls_row), D * 4));
    for (Group g : groups) {
        MG_TRY(pl->alloc(reinterpret_cast<void**>(&g.pos_table), static_cast<size_t>(g.h) * g.w * D * 4));
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

static int validate_dino(const moge_dino_config_t& c) {
    const int D = c.embed_dim;
    if (c.ffn_layer != MOGE_DINO_FFN_MLP)
        return set_error("dinov2: ffn_layer %s unsupported: the encoder kernels run the GELU MLP only (ViT-g uses SwiGLU)",
                         c.ffn_layer == MOGE_DINO_FFN_SWIGLU ? "swiglu" : c.ffn_layer == MOGE_DINO_FFN_IDENTITY ? "identity" : "(unknown)");
    if (D <= 0 || D % 128 || D > 1024)
        return set_error("dinov2: embed_dim=%d unsupported (a multiple of 128, <= 1024: ViT-S/B/L; ViT-g is not covered)", D);
    if (c.num_heads * 64 != D) return set_error("dinov2: head_dim must be 64 (embed_dim=%d, num_heads=%d)", D, c.num_heads);
    if (c.depth <= 0 || c.depth > 64) return set_error("dinov2: depth=%d out of range (1..64)", c.depth);
    if (c.patch_size != 14) return set_error("dinov2: patch_size=%d unsupported (14 only)", c.patch_size);
    if (c.num_register_tokens != 0)
        return set_error("dinov2: %d register tokens unsupported (the engine's rows are the class token and the patches only)",
                         c.num_register_tokens);
    if (c.interpolate_antialias) return set_error("dinov2: antialiased pos-embed interpolation unsupported");
    if (c.interpolate_offset != 0.1f) return set_error("dinov2: interpolate_offset=%g unsupported (0.1 only)", c.interpolate_offset);
    if (c.compute_dtype != MOGE_F16 && c.compute_dtype != MOGE_BF16) return set_error("dinov2: compute_dtype must be MOGE_F16 or MOGE_BF16");
    return 0;
}

}  // namespace mg

using namespace mg;

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

int moge_dino_create(const moge_dino_config_t* cfg, int device, moge_engine_t** out) {
    if (!cfg || !out) return set_error("null argument");
    MG_TRY(validate_dino(*cfg));
    moge_config_t enc{};         // the encoder part only: build_plan exports the backbone's rows instead of running a decoder
    enc.embed_dim = cfg->embed_dim; enc.depth = cfg->depth; enc.num_heads = cfg->num_heads;
    enc.compute_dtype = cfg->compute_dtype;
    MG_TRY(create_engine(&enc, device, out));
    (*out)->dino = true;
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
    for (auto& kv : e->raw) if (kv.second.p) cudaFree(kv.second.p);
    delete e;
}

// ---- a public group array as plan groups.  Every check fires in the order written here and in the entry points, so a bad call
//      reports the same first error however else it is wrong.

// The checks both public group structs share
static_assert(MOGE_DINO_MAX_GROUPS == 64, "the backbone's group tables (dinov2.cu) hold as many groups as any call carries");
static int check_group_count(int n) {
    if (n <= 0 || n > 64) return set_error("number of shape groups %d out of range (1..64)", n);
    return 0;
}

static int check_image(const void* image, int image_dtype) {
    if (!image) return set_error("null argument");
    if (image_dtype != MOGE_F32 && image_dtype != MOGE_F16 && image_dtype != MOGE_BF16) return set_error("unsupported image dtype %d", image_dtype);
    return 0;
}

// MoGe-2 groups, checked; `forward`: each group's image and requested outputs too
static int to_groups(moge_engine_t* e, const moge_group_t* g, int n, bool forward, std::vector<Group>* out) {
    if (!e || !g) return set_error("null argument");
    MG_TRY(check_group_count(n));
    for (int i = 0; i < n; ++i) {
        if (g[i].B <= 0 || g[i].h <= 0 || g[i].w <= 0 || g[i].H <= 0 || g[i].W <= 0)
            return set_error("bad shape B=%d H=%d W=%d h=%d w=%d", g[i].B, g[i].H, g[i].W, g[i].h, g[i].w);
        if (forward) {
            MG_TRY(check_image(g[i].image, g[i].image_dtype));
            if (g[i].points && !e->cfg.points_head.present) return set_error("points requested but the model has no points head");
            if (g[i].normal && !e->cfg.normal_head.present) return set_error("normal requested but the model has no normal head");
            if (g[i].mask_prob && !e->cfg.mask_head.present) return set_error("mask requested but the model has no mask head");
            if (g[i].metric_scale && e->cfg.scale_head_layers == 0) return set_error("metric_scale requested but the model has no scale head");
        }
        out->push_back(make_group(g[i]));
    }
    return 0;
}

// MoGe-1 groups, checked; `forward`: each group's outputs too (its image is checked after the call's own checks, check_forward)
static int v1_to_groups(moge_engine_t* e, const moge_v1_group_t* g, int n, bool forward, std::vector<Group>* out) {
    MG_TRY(check_group_count(n));
    if (!g || !e) return set_error("null argument");
    if (!e->v1) return set_error("not a MoGe-1 engine (moge_engine_create_v1)");
    for (int i = 0; i < n; ++i) {
        if (g[i].B <= 0 || g[i].H <= 0 || g[i].W <= 0) return set_error("bad shape B=%d H=%d W=%d", g[i].B, g[i].H, g[i].W);
        if (g[i].rh < 14 || g[i].rw < 14) return set_error("resized image %dx%d is smaller than one 14-pixel patch", g[i].rh, g[i].rw);
        if (forward && (!g[i].points || !g[i].mask)) return set_error("null argument");
        out->push_back(make_group(g[i]));
    }
    return 0;
}

// A DINOv2 backbone call as plan groups and its key, checked before anything runs: the group count, the engine, each group's shape,
// the layer list and flags; `forward`: each group's input too.  A group's error names its index when the call has several.
static int dino_groups(moge_engine_t* e, const moge_dino_group_t* groups, int n, const int* layers, int n_layers, int flags, bool forward,
                       std::vector<Group>* out, DinoKey* key) {
    MG_TRY(check_group_count(n));
    if (!e || !groups) return set_error("null argument");
    if (!e->dino) return set_error("not a DINOv2 backbone engine (moge_dino_create)");
    auto at = [n](int i) { return n > 1 ? "group " + std::to_string(i) + ": " : std::string(); };
    for (int i = 0; i < n; ++i) {
        const moge_dino_group_t& g = groups[i];
        if (g.B <= 0 || g.H <= 0 || g.W <= 0) return set_error("dinov2: %sbad shape B=%d H=%d W=%d", at(i).c_str(), g.B, g.H, g.W);
        if (g.H % 14 || g.W % 14)
            return set_error("dinov2: %sinput %d x %d is not a multiple of the patch size 14", at(i).c_str(), g.H, g.W);
    }
    if (n_layers < 0 || n_layers > e->cfg.depth) return set_error("dinov2: %d layers out of range (0..%d)", n_layers, e->cfg.depth);
    if (n_layers > 0 && !layers) return set_error("null argument");
    for (int j = 0; j < n_layers; ++j)
        if (layers[j] < 0 || layers[j] >= e->cfg.depth || (j > 0 && layers[j] <= layers[j - 1]))
            return set_error("dinov2: layers must be increasing block indices < depth (%d)", e->cfg.depth);
    if (flags & ~(MOGE_DINO_NORM | MOGE_DINO_CHANNEL_MAJOR)) return set_error("dinov2: unknown flags 0x%x", flags);
    for (int i = 0; i < n; ++i) {
        const moge_dino_group_t& m = groups[i];
        if (forward && !m.x) return set_error("%snull argument", at(i).c_str());
        if (forward && m.x_dtype != MOGE_F32 && m.x_dtype != MOGE_F16 && m.x_dtype != MOGE_BF16)
            return set_error("%sunsupported image dtype %d", at(i).c_str(), m.x_dtype);
        Group g;
        g.B = m.B; g.H = m.H; g.W = m.W; g.h = m.H / 14; g.w = m.W / 14;
        g.image = m.x; g.image_dtype = m.x_dtype;
        g.tokens = m.out_tokens; g.cls_out = m.out_cls; g.prenorm = m.out_prenorm;
        out->push_back(g);
    }
    key->layers.assign(layers, layers + n_layers);
    key->flags = flags;
    return 0;
}

int moge_engine_workspace_bytes_groups(moge_engine_t* e, const moge_group_t* groups, int n, size_t* bytes) {
    if (!bytes) return set_error("null argument");
    Plan pl;
    MG_TRY(to_groups(e, groups, n, false, &pl.groups));
    if (e->v1) return set_error("a MoGe-1 engine takes moge_v1_workspace_bytes_groups");
    if (e->dino) return set_error("a DINOv2 backbone engine takes moge_dino_workspace_bytes_groups");
    return build_plan(e, &pl, true, bytes);
}

// The checks of a forward call, before anything runs: the engine, its weights and the workspace pointer, then `groups` (the
// group checks that come after these), then the workspace alignment
static int check_forward(moge_engine_t* e, const void* workspace, const std::function<int()>& groups) {
    if (!e || !workspace) return set_error("null argument");
    if (!e->finalized) return set_error("engine not finalized");
    MG_TRY(groups());
    if (reinterpret_cast<uintptr_t>(workspace) & 1023) return set_error("workspace must be 1024-byte aligned");
    return 0;
}

// groups: checked, with their bindings
static int forward_impl(moge_engine_t* e, const std::vector<Group>& groups, void* workspace, size_t workspace_bytes, void* stream,
                        const DinoKey& dino = DinoKey()) {
    CUDA_TRY(cudaSetDevice(e->device));
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    Plan* pl;
    MG_TRY(get_plan(e, groups, dino, workspace, workspace_bytes, &pl, st));
    long tokens = 0;
    for (size_t i = 0; i < groups.size(); ++i) {
        Group& g = pl->groups[i];
        g.image = groups[i].image; g.image_dtype = groups[i].image_dtype;
        g.points = groups[i].points; g.normal = groups[i].normal; g.mask = groups[i].mask; g.scale = groups[i].scale;
        g.tokens = groups[i].tokens; g.cls_out = groups[i].cls_out; g.prenorm = groups[i].prenorm;
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
    if (e && e->v1) return set_error("a MoGe-1 engine runs through moge_v1_forward_groups");
    if (e && e->dino) return set_error("a DINOv2 backbone engine runs through moge_dino_forward_groups");
    std::vector<Group> gs;
    MG_TRY(check_forward(e, workspace, [&] { return to_groups(e, groups, n, true, &gs); }));
    return forward_impl(e, gs, workspace, workspace_bytes, stream);
}

int moge_v1_workspace_bytes_groups(moge_engine_t* e, const moge_v1_group_t* groups, int n, size_t* bytes) {
    if (!bytes) return set_error("null argument");
    Plan pl;
    MG_TRY(v1_to_groups(e, groups, n, false, &pl.groups));
    return build_plan(e, &pl, true, bytes);
}

int moge_v1_forward_groups(moge_engine_t* e, const moge_v1_group_t* groups, int n, void* workspace, size_t workspace_bytes, void* stream) {
    std::vector<Group> gs;
    MG_TRY(v1_to_groups(e, groups, n, true, &gs));
    MG_TRY(check_forward(e, workspace, [&] {
        for (const Group& g : gs) MG_TRY(check_image(g.image, g.image_dtype));
        return 0;
    }));
    return forward_impl(e, gs, workspace, workspace_bytes, stream);
}

int moge_v1_postprocess(float* points, const float* mask, float mask_threshold, const float* focal_in, int B, int H, int W,
                        int force_projection, int apply_mask, float* depth, uint8_t* mask_out, float* intrinsics, float* focal,
                        float* shift, void* stream) {
    if (!points || !mask || !depth || !mask_out || !intrinsics || !focal || !shift) return set_error("null argument");
    if (B <= 0 || H <= 0 || W <= 0) return set_error("bad shape B=%d H=%d W=%d", B, H, W);
    return launch_v1_postprocess(points, mask, mask_threshold, focal_in, B, H, W, force_projection, apply_mask, depth, mask_out, intrinsics,
                                 focal, shift, static_cast<cudaStream_t>(stream));
}

int moge_dino_workspace_bytes_groups(moge_engine_t* e, const moge_dino_group_t* groups, int n, const int* layers, int n_layers,
                                     int flags, size_t* bytes) {
    if (!bytes) return set_error("null argument");
    Plan pl;
    MG_TRY(dino_groups(e, groups, n, layers, n_layers, flags, false, &pl.groups, &pl.dino));
    return build_plan(e, &pl, true, bytes);
}

int moge_dino_forward_groups(moge_engine_t* e, const moge_dino_group_t* groups, int n, const int* layers, int n_layers, int flags,
                             void* workspace, size_t workspace_bytes, void* stream) {
    MG_TRY(check_group_count(n));
    std::vector<Group> gs;
    DinoKey key;
    MG_TRY(check_forward(e, workspace, [&] { return dino_groups(e, groups, n, layers, n_layers, flags, true, &gs, &key); }));
    return forward_impl(e, gs, workspace, workspace_bytes, stream, key);
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
    if (!e || !e->last_plan || !ms) return set_error("profile: run moge_engine_forward_groups once first");
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

}  // extern "C"
