// Internal host-side declarations shared by the .cu translation units of libmoge_b200.so.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stddef.h>
#include <atomic>
#include <vector>
#include <utility>

namespace mg {

// Thread-local error message behind moge_last_error(); returns -1 so callers can `return set_error(...)`.
int set_error(const char* fmt, ...);

#define CUDA_TRY(expr)                                                                                   \
    do {                                                                                                 \
        cudaError_t _e = (expr);                                                                         \
        if (_e != cudaSuccess)                                                                           \
            return ::mg::set_error("%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), __FILE__, __LINE__); \
    } while (0)
#define MG_TRY(expr)                \
    do {                            \
        int _r = (expr);            \
        if (_r != 0) return _r;     \
    } while (0)

// cudaFuncSetAttribute(MaxDynamicSharedMemorySize) is a PER-DEVICE property of a kernel: every launcher keeps one of these
// per kernel instantiation and sets the attribute on the first launch on each device (engines on several GPUs in one
// process; setting it twice from two threads is harmless, so relaxed atomics are enough).
struct DevOnce {
    std::atomic<bool> done[64];
    DevOnce() { for (auto& d : done) d.store(false, std::memory_order_relaxed); }
    // true when the current device has not been prepared yet (dev < 0: query failed -> always prepare)
    bool need(int* dev) {
        if (cudaGetDevice(dev) != cudaSuccess || *dev < 0 || *dev >= 64) { *dev = -1; return true; }
        return !done[*dev].load(std::memory_order_acquire);
    }
    void mark(int dev) { if (dev >= 0) done[dev].store(true, std::memory_order_release); }
};
#define MG_SET_SMEM_ONCE(kern, bytes)                                                                    \
    do {                                                                                                 \
        static ::mg::DevOnce _once;                                                                      \
        int _dev;                                                                                        \
        if (_once.need(&_dev)) {                                                                         \
            CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes));    \
            _once.mark(_dev);                                                                            \
        }                                                                                                \
    } while (0)

// Programmatic dependent launch (PDL): every kernel of the forward path starts with `pdl_prologue()` (common.cuh:
// griddepcontrol.launch_dependents, then griddepcontrol.wait) and is launched with programmatic stream serialization, so the NEXT
// kernel's launch, block scheduling and prologue overlap the tail of this one instead of waiting for the full drain of the grid;
// correctness is unchanged (the wait returns only when the predecessor grid has completed and flushed).  It matters at batch 1,
// where a forward is ~245 kernels of a few microseconds each (also inside the captured CUDA graph).  At large batches the kernels
// are long and early-resident dependents only get in the way, so the engine switches it on per call, for the small
// (graph-replayed) calls only: `pdl_scope` is thread-local state read by `launch_pdl`.
bool& pdl_scope();
template <typename... KArgs, typename... Args>
inline cudaError_t launch_pdl(void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, Args&&... args) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = st;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = pdl_scope() ? 1 : 0;
    cfg.attrs = attr; cfg.numAttrs = 1;
    return cudaLaunchKernelEx(&cfg, kern, std::forward<Args>(args)...);
}

// ---- TMA descriptors (driver entry point resolved at run time; no link-time libcuda dependency)
// 16-bit element maps with a 64-element (128-byte) inner box and SWIZZLE_128B.
int make_map_2d(CUtensorMap* m, const void* base, uint64_t cols, uint64_t rows, uint64_t row_pitch_elems, uint32_t box_rows);
// padded NHWC image [B, Hp, Wp, C]: box {64 ch, 16 px, 8 rows, 1}
int make_map_nhwc(CUtensorMap* m, const void* base, uint64_t C, uint64_t Wp, uint64_t Hp, uint64_t B, uint32_t box_rows = 8);

// ---- gemm_kernel launches (gemm.cu).  The builders choose the kernel variant (main-loop mode, tile width, epilogue) and fill its
// params and tensor maps; launch_gemm runs the result.  A builder fails (returns -1) on a shape no variant covers.
struct GemmLaunch;
struct Level { int H, W, Hp, Wp; };      // an image grid and its padded NHWC allocation (1-pixel replicated border)

struct ConvW {          // packed 3x3 / 1x1 / convT weights for one launch
    void* w = nullptr;  // [N, Ktot] 16-bit
    float* bias = nullptr;
    float* wu = nullptr;
    float* wv = nullptr;
    int N = 0, Ktot = 0, cin = 0, caux = 0, taps = 0;
};

constexpr int kStatsLd = 16;      // partial-sum slots per row of the LayerNorm statistics buffer
struct LnIO {                     // LayerNorm-fold plumbing of one linear (see elementwise.cu)
    void* x16 = nullptr;          // producer (EPI_RESID / EPI_PATCH): 16-bit copy of the rows it writes
    float2* stats_out = nullptr;  // producer: partial sums
    int* parts_out = nullptr;     // producer: number of column groups it writes per row
    const float* ln_rstd = nullptr;       // consumer (EPI_STORE16 / EPI_GELU16)
};

// Linear: A [M, K] (row pitch K) times the weight W [N, K] (row pitch ldw) -> epilogue `epi` into out (row pitch ldo elements),
// N a multiple of 128.  EPI_PATCH and EPI_DEC rows are the tokens of images on the token grid `grid`; EPI_DEC writes the padded
// NHWC map of that grid (raw: out, ReLU copy: out_relu, UV terms v1/v2 with half extents su/sv).
int gemm_linear(GemmLaunch* g, bool bf16, const void* A, int M, int K, const void* W, int ldw, int N, int epi, void* out, int ldo,
                const float* bias, const float* v1, const LnIO* ln = nullptr, const Level* grid = nullptr, void* out_relu = nullptr,
                const float* v2 = nullptr, float su = 0.f, float sv = 0.f);
// Conv on padded NHWC maps: source src (+ aux, the fused 1x1 input block) on grid gs, output on grid go with out_ch channels.
// Picks the main loop from the shape: CONV64 (3x3, C_in = 64), CONVH (3x3, C_in >= 128) or the per-tap GEMM.
int gemm_conv(GemmLaunch* g, bool bf16, const ConvW& cw, const void* src, const void* aux, const Level& gs, int B, int epi,
              void* out_raw, void* out_relu, const void* skip, const Level& go, int out_ch, bool shuffle, bool uv, float su, float sv,
              int ncomp = 0, void* out2 = nullptr);
int launch_gemm(const GemmLaunch& g, int num_sms, cudaStream_t st);

// Attention over PACKED token rows (ragged batches): qkv [rows, 3D] (map: box {64, 128}), one work item per (image, head, pair
// of 128-row query tiles); the persistent kernel's CTA c walks items [ranges[c].x, ranges[c].y).
struct AttnItem { int row0, n, q0, head; };      // image's first row, its token count, first query row (image-relative), head
void attention_work_list(const int* row0, const int* n, int nimg, int heads, int ncta, std::vector<AttnItem>* items,
                         std::vector<int2>* ranges);
int launch_attention(const CUtensorMap& mapQKV, void* out, const AttnItem* items_dev, const int2* ranges_dev, int ncta, int D, int heads,
                     bool bf16, cudaStream_t st);

// ---- small kernels (elementwise.cu)
// K1: antialiased bilinear resize to (14h,14w) + ImageNet normalise + patchify -> A[B*T, Kp] (16-bit, Kp = 592)
int launch_preprocess(const void* image, int image_dtype, int B, int H, int W, int h, int w, void* patches, int Kp,
                      bool bf16, cudaStream_t st);
// K3: table[t, d] = bicubic(pos_embed grid)[t, d] + patch bias[d]  (fp32), cls_row[d] = cls_token[d] + pos_embed[0, d]
int launch_pos_table(const float* pos_embed, const float* cls_token, const float* patch_bias, int D, int h, int w,
                     float* table, float* cls_row, cudaStream_t st);
int launch_init_cls(float* x, const float* cls_row, int B, int N, int D, cudaStream_t st);
// LayerNorm eps=1e-6 over D: fp32 in -> 16-bit out.  Row r of the input maps to out row r (ld_out elements per row).
// mode 0: plain (all rows).  mode 1 (taps): skip cls rows; patch token (b,t) -> out[(b*T+t)*ld_out + col_off + d];
// the cls row of each image is written (fp32) to cls_out[b, D] when cls_out != null.
int launch_layernorm(const float* x, const float* gamma, const float* beta, void* out, int rows, int D, int ld_out,
                     int col_off, int mode, int tokens_per_image, float* cls_out, bool bf16, cudaStream_t st);
// LayerNorm folded into the following GEMM (see elementwise.cu): rounded rows + per-row partial sums for rows no GEMM epilogue
// produces (cls rows; op-level tests), the per-row rstd reduction, and the load-time weight fold  w16 = T(rows of W diag(gamma), centred), b2 = b + W beta
int launch_ln_prepare(const float* x, int rows, long row_stride, int D, void* x16, long row_stride16, float2* stats, long stats_stride,
                      int parts, bool bf16, cudaStream_t st);
int launch_ln_fold(const float* W, const float* gamma, const float* beta, const float* bias, int N, int K, int ldw, void* w16,
                   float* b2, bool bf16, cudaStream_t st);
int launch_ln_rstd(const float2* stats, int ld, int parts, int rows, int D, float* rstd, cudaStream_t st);
// scale head: metric_scale[b] = exp(MLP(cls[b]))
int launch_scale_head(const float* cls, const float* const* w, const float* const* bias, const int* dims, int nlayers,
                      int B, float* out, float* scratch, cudaStream_t st);
// K17: bilinear resize of the low-res head maps to (H,W) + remap -> points (B,H,W,3), normal (B,H,W,3), mask prob (B,H,W)
// (mask_sigmoid = false: the resized mask logit as is, MoGe-1)
int launch_head_output(const float4* pts_lr, const float4* nrm_lr, const float* msk_lr, int B, int Hl, int Wl, int H, int W,
                       int remap_mode, float* points, float* normal, float* mask, cudaStream_t st, bool mask_sigmoid = true);
// K18
int launch_focal_shift(const float* points, const float* mask_prob, const uint8_t* mask_u8, int B, int H, int W,
                       const float* focal_in, float* focal_out, float* shift_out, cudaStream_t st);
// K19
int launch_postprocess(float* points, const float* normal_in, const float* mask_prob, const float* metric_scale,
                       const float* focal, const float* shift, int B, int H, int W, int force_projection, int apply_mask,
                       float* depth, float* normal_out, uint8_t* mask_out, float* intrinsics, cudaStream_t st);

// ---- MoGe-1 kernels (v1.cu); maps are padded NHWC 16-bit with C channels on grid g, border written
// antialiased bicubic (a = -0.5) resize (B,C,H,W) image -> fp32 (B,C,Ho,Wo) via the fp32 row pass tmp (B,C,H,Wo)
int launch_resize_bicubic_aa(const void* image, int dtype, int B, int C, int H, int W, int Ho, int Wo, float* tmp, float* out, cudaStream_t st);
// host side of the same filter: taps [*lo, *lo + n) of output index i and their normalised weights (w may be NULL); returns n
int bicubic_aa_taps(int in, int out, int i, int* lo, float* w, int cap);
// GroupNorm(G, C) statistics (mean, rstd) per (image, group); partials: B * gn_tiles(H, W, C) * G double2 of scratch
int gn_tiles(int H, int W, int C);
int launch_gn_stats(const void* map, const Level& g, int B, int C, int G, double2* partials, float2* stats, bool bf16, cudaStream_t st);
// dst = relu(gamma * (src - mean) * rstd + beta)
int launch_gn_relu(const void* src, void* dst, const Level& g, int B, int C, int G, const float2* stats, const float* gamma, const float* beta,
                   bool bf16, cudaStream_t st);
// in place: + the input-grid UV term of a k2s2 ConvTranspose, wuv [2][4 phases][C]; g is the OUTPUT grid
int launch_uv_convT(void* map, const Level& g, int B, int C, const float* wuv, float su, float sv, bool bf16, cudaStream_t st);
// wuv [2][4][Cout] from rows Cin, Cin + 1 of a ConvTranspose2d weight (Cin + 2, Cout, 2, 2) fp32 (load time)
int launch_pack_convT_uv(const float* w, int Cin, int Cout, float* wuv, cudaStream_t st);
// bilinear (align_corners=False) resize of a padded map from grid gs to grid gd
int launch_resize_bilinear_nhwc(const void* src, const Level& gs, void* dst, const Level& gd, int B, int C, bool bf16, cudaStream_t st);
// output-block tail over the 64-channel conv output: + folded UV, ReLU, block-diagonal 64 -> 4; pts (x,y,z,-), msk fp32 per pixel
int launch_v1_output(const void* map, const Level& g, int B, const float* wf, float su, float sv, float4* pts, float* msk, bool bf16, cudaStream_t st);
int launch_v1_postprocess(float* points, const float* mask, float mask_threshold, const float* focal_in, int B, int H, int W, int force_projection,
                          int apply_mask, float* depth, uint8_t* mask_out, float* intrinsics, float* focal, float* shift, cudaStream_t st);

// ---- weight packing (pack.cu): generic strided gather/cast and a small fp32 GEMM for load-time folds
int launch_cast_2d(const void* src, int src_dtype, void* dst, bool bf16, int rows, int cols, int src_ld, int dst_ld,
                   cudaStream_t st);
// dst16[n, k_off + tap*Cin + ci] = W[n, ci, tap]  for conv weight (Cout, Cin, kh, kw) fp32
int launch_pack_conv(const float* w, void* dst, bool bf16, int Cout, int Cin, int taps, int dst_ld, int k_off, cudaStream_t st);
// dst16[(q*Cout + co), ci] = W[ci, co, q]  for ConvTranspose2d weight (Cin, Cout, 2, 2)
int launch_pack_convT(const float* w, void* dst, bool bf16, int Cin, int Cout, cudaStream_t st);
// (Cout,Cin,3,3) -> (4*Cout,Cin,3,3): bilinear-x2-upsample folded into the following 3x3 conv (see pack.cu)
int launch_up2_expand(const float* w, float* dst, int Cout, int Cin, cudaStream_t st);
// C[M,N] (fp32, ldc) = A[M,K] (lda) * B[K,N] (ldb)  (+ C if accumulate)   -- load-time only, SIMT
int launch_sgemm(const float* A, int lda, const float* B, int ldb, float* C, int ldc, int M, int N, int K, int accumulate,
                 cudaStream_t st);

}  // namespace mg
