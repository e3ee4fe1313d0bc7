// Internal declarations shared by the engine's two host units: the packed-weight structs and the engine object.  weights.cu fills
// them at load time (moge_engine_set_weight, moge_engine_finalize); engine.cu plans and runs forwards over them.
#pragma once
#include "moge_b200.h"
#include "host_api.h"

#include <map>
#include <memory>
#include <string>
#include <vector>

namespace mg {

struct RawWeight {          // fp32 staging copy of one checkpoint tensor
    float* p = nullptr;
    std::vector<int64_t> shape;
    size_t numel = 0;
    bool keep = false;      // read by a kernel at run time: survives finalize
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

struct Plan;                // engine.cu

}  // namespace mg

struct moge_engine {
    moge_config_t cfg;
    bool v1 = false;                  // created by moge_engine_create_v1: cfg holds the encoder only, v1cfg the rest
    moge_v1_config_t v1cfg{};
    bool dino = false;                // created by moge_dino_create: the backbone alone, its own weight keys, no decoder
    mg::V1W v1w;
    int device = 0, num_sms = 132;
    bool bf16 = false, finalized = false;
    std::map<std::string, mg::RawWeight> raw;
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
    mg::ConvW fold0;                  // taps-concat GEMM: (output projections folded into neck.input_blocks.0)
    mg::StackW neck, heads[3];        // heads: points, normal, mask
    std::vector<const float*> mlp_w, mlp_b;
    std::vector<std::unique_ptr<mg::Plan>> plans;      // LRU order (most recently used last), at most kMaxPlans
    mg::Plan* last_plan = nullptr;
    cudaStream_t own_stream = nullptr;
    cudaEvent_t ev_in = nullptr, ev_out = nullptr;

    int alloc(void** p, size_t bytes) {
        CUDA_TRY(cudaMalloc(p, bytes ? bytes : 16));
        owned.push_back(*p);
        return 0;
    }
};

namespace mg {

inline const moge_stack_config_t* head_cfg(const moge_engine* e, int i) {
    return i == 0 ? &e->cfg.points_head : i == 1 ? &e->cfg.normal_head : &e->cfg.mask_head;
}
inline const char* head_name(int i) { return i == 0 ? "points_head" : i == 1 ? "normal_head" : "mask_head"; }

}  // namespace mg
