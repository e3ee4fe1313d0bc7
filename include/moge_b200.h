/* moge_b200 -- C ABI of the H100-native MoGe-2 (and MoGe-1) inference engine (libmoge_b200.so, sm_90a).
 *
 * The reference (microsoft/MoGe) has no FFI / plugin boundary on this path: the hot path is the Python nn.Module
 * `moge.model.v2.MoGeModel` (/root/reference/moge/model/v2.py).  This header is the boundary the replacement exports;
 * each entry point names the reference interface it replaces.  It is bound by moge_b200/capi.py (ctypes), which backs
 * the drop-in `moge.model.v2.MoGeModel` class (see INTEGRATION.md).
 *
 * Conventions
 *   - every function returns 0 on success, <0 on error; the message is in moge_last_error() (thread-local).
 *   - no C++ exceptions cross the ABI; no torch types; plain device pointers + sizes.
 *   - all work is enqueued on the `stream` argument (a cudaStream_t passed as void*); nothing synchronises the device.
 *   - the caller owns every input/output tensor and the workspace; the engine owns its packed weights.
 *   - calls on one engine must be serialised by the caller (stream order); engines on different devices (or several engines
 *     on one device) may live in one process and be driven from different threads.
 *   - there is NO CPU fallback: without a sm_90 (H100) device every compute entry point fails.
 */
#ifndef MOGE_B200_H
#define MOGE_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define MOGE_MAX_LEVELS 8
#define MOGE_MAX_TAPS 8
#define MOGE_MAX_MLP 8

/* element types of caller tensors */
enum { MOGE_F32 = 0, MOGE_F16 = 1, MOGE_BF16 = 2, MOGE_U8 = 3 };
/* v2.py:122-136 remap_output */
enum { MOGE_REMAP_LINEAR = 0, MOGE_REMAP_SINH = 1, MOGE_REMAP_EXP = 2, MOGE_REMAP_SINH_EXP = 3 };
/* modules.py:139-182 Resampler types used by MoGe-2 configs */
enum { MOGE_RESAMPLE_CONV_TRANSPOSE = 0, MOGE_RESAMPLE_BILINEAR = 1 };

/* One ConvStack (modules.py:195-254).  Norm-free residual blocks only (MoGe-2 configs). */
typedef struct moge_stack_config {
    int present;                          /* 0 = head absent (hasattr(model, head) is False, v2.py:50-57) */
    int num_levels;                       /* 5 */
    int dim_in[MOGE_MAX_LEVELS];          /* 0 = no input block at that level */
    int dim_res_blocks[MOGE_MAX_LEVELS];
    int num_res_blocks[MOGE_MAX_LEVELS];
    int dim_out[MOGE_MAX_LEVELS];         /* 0 = Identity output block */
    int resamplers[MOGE_MAX_LEVELS];      /* MOGE_RESAMPLE_* between level l and l+1 */
} moge_stack_config_t;

/* Mirrors the `model_config` dict stored in a MoGe-2 checkpoint (v2.py:30-57, configs/train/v2.json:237-285). */
typedef struct moge_config {
    int embed_dim, depth, num_heads;      /* DINOv2 backbone (vision_transformer.py:351-390); head_dim must be 64 */
    int num_taps;
    int taps[MOGE_MAX_TAPS];              /* encoder.intermediate_layers */
    int dim_out;                          /* encoder.dim_out */
    moge_stack_config_t neck, points_head, normal_head, mask_head;
    int scale_head_layers;                /* 0 = absent; number of Linear layers */
    int scale_head_dims[MOGE_MAX_MLP];    /* scale_head.dims */
    int remap_output;                     /* MOGE_REMAP_* */
    int compute_dtype;                    /* MOGE_F16 or MOGE_BF16: tensor-core operand type (fp32 accumulate) */
} moge_config_t;

typedef struct moge_engine moge_engine_t;

const char* moge_last_error(void);
/* library / build identification: "moge_b200 <version> sm_90a" */
const char* moge_version(void);

/* replaces MoGeModel.__init__ (v2.py:30-57) + .to(device) */
int moge_engine_create(const moge_config_t* cfg, int device, moge_engine_t** out);
void moge_engine_destroy(moge_engine_t* e);

/* replaces load_state_dict (v2.py:105): hand over one state-dict tensor by its PyTorch key, in its PyTorch layout
 * (contiguous, device memory, MOGE_F32 / MOGE_F16 / MOGE_BF16).  The engine copies it; the caller may free it. */
int moge_engine_set_weight(moge_engine_t* e, const char* key, const void* dev_ptr, const int64_t* shape, int ndim,
                           int dtype, void* stream);
/* repack all weights into the kernels' layouts (K-major 16-bit GEMM operands, folded linear maps); fails listing the
 * first missing key.  Must be called once after the last set_weight and before forward. */
int moge_engine_finalize(moge_engine_t* e, void* stream);

/* workspace (activations) size for a forward of B images of HxW pixels on an hxw token grid */
int moge_engine_workspace_bytes(moge_engine_t* e, int B, int H, int W, int h, int w, size_t* bytes);

/* replaces MoGeModel.forward (v2.py:138-192).  image: (B,3,H,W) in [0,1], dtype image_dtype.  h,w: token grid
 * (v2.py:142-147, computed by the caller).  Outputs are fp32, caller-allocated; pass NULL for absent heads:
 *   points (B,H,W,3)  normal (B,H,W,3)  mask_prob (B,H,W)  metric_scale (B,)                                     */
int moge_engine_forward(moge_engine_t* e, const void* image, int image_dtype, int B, int H, int W, int h, int w,
                        void* workspace, size_t workspace_bytes, float* points, float* normal, float* mask_prob,
                        float* metric_scale, void* stream);

/* Mixed-shape ("ragged") batches -- BASELINE.json configs[2]; the reference has no counterpart (a batch tensor has one shape and
 * its nested-tensor path, dinov2/layers/block.py:160-259, is dead code without xformers).  A call carries `n` shape groups; the
 * encoder (every linear, the attention) runs ONCE over the token rows of all groups packed back to back, the per-pixel stages
 * (resize/patchify, pos embed, decoder, output resize) run group by group.  moge_engine_forward is the n = 1 case. */
typedef struct moge_group {
    const void* image;          /* (B,3,H,W) in [0,1] */
    int image_dtype;            /* MOGE_F32 / MOGE_F16 / MOGE_BF16 */
    int B, H, W, h, w;          /* images, pixels, token grid of this group */
    float* points;              /* (B,H,W,3) or NULL */
    float* normal;              /* (B,H,W,3) or NULL */
    float* mask_prob;           /* (B,H,W) or NULL */
    float* metric_scale;        /* (B,) or NULL */
} moge_group_t;
int moge_engine_workspace_bytes_groups(moge_engine_t* e, const moge_group_t* groups, int n, size_t* bytes);
int moge_engine_forward_groups(moge_engine_t* e, const moge_group_t* groups, int n, void* workspace, size_t workspace_bytes,
                               void* stream);

/* ---- introspection of the launch list of the most recent forward (used by bench.py for the roofline numbers):
 * number of kernel launches, per-launch kernel class / algorithmic flops / algorithmic HBM bytes, and a profiling
 * replay that brackets every launch with CUDA events on `stream` (this one call synchronises the stream). */
int moge_engine_num_ops(moge_engine_t* e, int* n);
int moge_engine_op_info(moge_engine_t* e, int idx, char* name, int name_cap, double* flops, double* bytes);
int moge_engine_profile(moge_engine_t* e, float* ms_per_op, int cap, void* stream);

/* host only (no device work): the work list the engine builds at plan time for the persistent attention kernel.
 * n_tokens[n_images] = token rows per image (class token + patches).  One item = (first row of the image, its token
 * count, first query row, head) = one 256-query tile of one head; ranges[c] = [begin, end) of the items CTA c walks
 * (contiguous, cost-balanced, every CTA at least one item; n_ranges = min(n_ctas, n_items)).  items: 4 ints per item,
 * ranges: 2 ints per CTA (cap n_ctas); either may be NULL to query the counts only.                                     */
int moge_attention_work_list(const int* n_tokens, int n_images, int heads, int n_ctas, int* items, int items_cap, int* ranges,
                             int* n_items, int* n_ranges);

/* replaces recover_focal_shift (moge/utils/geometry_torch.py:115-170 + geometry_numpy.py:79-112; SciPy LM on the
 * host in the reference).  points (B,H,W,3) fp32.  Mask: mask_u8 (B,H,W) if non-NULL, else mask_prob > 0.5 if
 * non-NULL, else all valid.  focal_in: NULL (solve focal and shift) or (B,) known focal (solve shift only).      */
int moge_recover_focal_shift(const float* points, const float* mask_prob, const uint8_t* mask_u8, int B, int H, int W,
                             const float* focal_in, float* focal_out, float* shift_out, void* stream);

/* replaces the fp32 post-processing of MoGeModel.infer (v2.py:265-289): intrinsics, z += shift, mask &= z > 0,
 * re-projection (force_projection), metric scale, masking.  points is updated in place; normal_in/out, mask_prob,
 * metric_scale, mask_out may be NULL when the corresponding head is absent.                                     */
int moge_postprocess(float* points, const float* normal_in, const float* mask_prob, const float* metric_scale,
                     const float* focal, const float* shift, int B, int H, int W, int force_projection, int apply_mask,
                     float* depth, float* normal_out, uint8_t* mask_out, float* intrinsics, void* stream);

/* ---- output gather over NVLink peer memory (SURVEY.md 8e: "gather of outputs to rank 0"; BASELINE.json configs[3]).  No reference
 * counterpart (the reference is single-GPU).  Every rank exposes a staging buffer by CUDA IPC (moge_peer_alloc -> 64-byte handle,
 * exchanged by the caller, e.g. torch.distributed.all_gather_object), the gathering rank maps them (moge_peer_open) and pulls with
 * copy-engine DMAs (moge_peer_copy); steps are ordered by flags in peer memory: moge_peer_flag_set makes `*flag = value` visible
 * system-wide after everything earlier on `stream`; moge_peer_flag_wait blocks `stream` until `*flag >= value` (the flag may live on
 * another GPU).  No SM is used for the transfer.  Python: moge_b200.parallel.PeerGatherer. */
int moge_peer_alloc(size_t bytes, void** dev_ptr, unsigned char* handle64);
int moge_peer_free(void* dev_ptr);
int moge_peer_open(const unsigned char* handle64, void** dev_ptr);
int moge_peer_close(void* dev_ptr);
int moge_peer_copy(void* dst, const void* src, size_t bytes, void* stream);
int moge_peer_flag_set(int* flag, int value, void* stream);
int moge_peer_flag_wait(const int* flag, int value, void* stream);

/* ---- operator-level entry points (same kernels the engine launches; used by the parity tests and micro-benchmarks)
 * y = epilogue(x[M,K] @ w[N,K]^T): epi 0 = +bias -> 16-bit, 1 = +bias,GELU(erf) -> 16-bit,
 * 2 = out32[M,N] += gamma * (acc + bias).  x, w: 16-bit (dtype MOGE_F16/MOGE_BF16), K % 8 == 0, N % 128 == 0.       */
int moge_op_linear(const void* x, const void* w, const float* bias, const float* gamma, void* out, int M, int N, int K,
                   int epi, int dtype, void* stream);
/* y16[M,N] = epilogue(LayerNorm_eps1e-6(x32[M,K]; ln_gamma, ln_beta) @ w32[N,K]^T + bias), epi 0 or 1 as above, computed the way the
 * engine computes norm1->qkv and norm2->fc1 (dinov2/layers/block.py:84-92): the GEMM runs on the ROUNDED rows with the centred
 * weight W diag(gamma) (I - 11^T/K) (mean removal is linear), the epilogue scales by rstd[row] and adds b + W beta.
 * K % 64 == 0, N % 128 == 0.                                                                                                */
int moge_op_linear_ln(const float* x, const float* ln_gamma, const float* ln_beta, const float* w, const float* bias, void* out, int M,
                      int N, int K, int epi, int dtype, void* stream);
/* softmax(q k^T / 8) v per head on a fused qkv buffer (B,N,3*D) -> (B,N,D); D = heads*64 (attention.py:70-81) */
int moge_op_attention(const void* qkv, void* out, int B, int N, int D, int heads, int dtype, void* stream);
/* LayerNorm(eps=1e-6) of fp32 rows -> 16-bit */
int moge_op_layernorm(const float* x, const float* gamma, const float* beta, void* out, int rows, int D, int dtype,
                      void* stream);
/* 3x3 (taps=9) or 1x1 (taps=1) convolution on padded NHWC 16-bit maps (B,H+2,W+2,C) with replicated border:
 * out = conv(x, w) + bias (+ skip); writes raw (out_raw) and/or ReLU (out_relu) padded NHWC maps incl. border.
 * w: PyTorch Conv2d weight (Cout,Cin,k,k) fp32.  shuffle=1: w is a ConvTranspose2d k2s2 weight (Cin,Cout,2,2) and
 * the output map is (B,2H+2,2W+2,Cout).                                                                         */
int moge_op_conv(const void* x, const float* w, const float* bias, const void* skip, void* out_raw, void* out_relu,
                 int B, int H, int W, int Cin, int Cout, int taps, int shuffle, int dtype, void* stream);

/* ---- MoGe-1 (moge/model/v1.py; Python: moge_b200.model.v1, alias moge.model.v1).  The same DINOv2 encoder as above; the decoder
 * is v1's Head (v1.py:61-142): summed 1x1 projections of the taps, then per level a ConvTranspose2d(k2 s2) over cat(x, uv), a
 * replicate-padded 3x3 conv and GroupNorm residual blocks, then a bilinear resize to the resized-image grid and two output blocks
 * (points, mask).  moge_engine_create_v1 returns an engine that destroy / set_weight / finalize / num_ops / op_info / profile take
 * unchanged; its weight keys are the reference's v1 state-dict keys.  Configs the engine does not cover fail at create. */
enum { MOGE_V1_GROUP_NORM = 0, MOGE_V1_LAYER_NORM = 1 };
typedef struct moge_v1_config {
    int embed_dim, depth, num_heads;      /* DINOv2 ViT-S/B/L */
    int num_taps;
    int taps[MOGE_MAX_TAPS];              /* intermediate_layers as block indices (an int n means the last n blocks) */
    int dim_proj;                         /* multiple of 128 */
    int num_levels;                       /* len(dim_upsample) */
    int dim_upsample[MOGE_MAX_LEVELS];    /* multiples of 64 */
    int hidden_mult;                      /* dim_times_res_block_hidden */
    int num_res_blocks;
    int hidden_norm;                      /* MOGE_V1_GROUP_NORM: hidden/32 groups, MOGE_V1_LAYER_NORM: 1 group */
    int last_res_blocks;                  /* must be 0 */
    int last_conv_channels;               /* must be 32 */
    int last_conv_size;                   /* must be 1 */
    int remap_output;                     /* MOGE_REMAP_* */
    int compute_dtype;                    /* MOGE_F16 or MOGE_BF16 */
} moge_v1_config_t;
int moge_engine_create_v1(const moge_v1_config_t* cfg, int device, moge_engine_t** out);
/* workspace for B images of HxW pixels resized to (rh, rw) (v1.py:273-274: rh = int(H f), rw = int(W f)); token grid rh/14 x rw/14 */
int moge_v1_workspace_bytes(moge_engine_t* e, int B, int H, int W, int rh, int rw, size_t* bytes);
/* replaces MoGeModel.forward (v1.py:269-299): image (B,3,H,W) in [0,1]; points (B,H,W,3) remapped, mask (B,H,W) the raw mask
 * output (no sigmoid), both fp32 */
int moge_v1_forward(moge_engine_t* e, const void* image, int image_dtype, int B, int H, int W, int rh, int rw, void* workspace,
                    size_t workspace_bytes, float* points, float* mask, void* stream);
/* the fp32 part of MoGeModel.infer (v1.py:352-380): mask_out = mask > mask_threshold (u8), focal/shift recovery (focal_in NULL:
 * solve both), intrinsics (B,3,3), depth = z + shift, points re-projected (force_projection) or shifted in z, points and depth
 * +inf outside the mask (apply_mask).  points updated in place; focal, shift (B,) outputs. */
int moge_v1_postprocess(float* points, const float* mask, float mask_threshold, const float* focal_in, int B, int H, int W,
                        int force_projection, int apply_mask, float* depth, uint8_t* mask_out, float* intrinsics, float* focal,
                        float* shift, void* stream);
/* operator entry points of the v1 kernels.  resize: F.interpolate(bicubic, align_corners=False, antialias=True) of (B,C,H,W)
 * (dtype MOGE_F32/F16/BF16) to fp32 (B,C,Ho,Wo).  group norm: relu(GroupNorm(G, C, eps 1e-5)(x) * gamma + beta) of the interior
 * of a padded NHWC 16-bit map (B,Hp,Wp,C) (Hp = max(H+2, 8), Wp = max(W+2, 16)) into another such map, border replicated. */
int moge_op_resize_bicubic_aa(const void* x, int dtype, int B, int C, int H, int W, int Ho, int Wo, float* out, void* stream);
int moge_op_groupnorm_relu(const void* x, void* out, const float* gamma, const float* beta, int B, int H, int W, int C, int G,
                           int dtype, void* stream);
/* the MoGe-1 upsampling ConvTranspose2d(Cin + 2 -> Cout, k2 s2) over cat(x, uv): x a padded NHWC 16-bit map (B,Hp,Wp,Cin) on an
 * H x W grid, w the PyTorch weight (Cin + 2, Cout, 2, 2) fp32, bias (Cout) fp32; the UV planes (half extents su, sv) are taken on
 * the INPUT grid.  out: padded NHWC (B, max(2H+2, 8), max(2W+2, 16), Cout), border replicated.  Cin % 64 == 0, Cout % 32 == 0. */
int moge_op_conv_transpose_uv(const void* x, const float* w, const float* bias, void* out, int B, int H, int W, int Cin, int Cout, float su,
                     float sv, int dtype, void* stream);
/* host only: taps [*lo, *lo + n) and normalised weights (w may be NULL) of output index i of the antialiased bicubic filter
 * for a resize of `in` to `out` samples; returns n (< 0 on error) */
int moge_bicubic_aa_weights(int in, int out, int i, int* lo, float* w, int cap);

/* ---- truncated-L1 alignment solvers (moge/utils/alignment.py; Python: moge_b200.alignment, alias moge.utils.alignment).
 * A problem is n elements (x, y, w), w >= 0; it is solved as align() (alignment.py:52-146) solves it: after x, y *= sign(x), either
 * the lower weighted median of y / max(x, 1e-7) with weights w x (untruncated) or the least of sum_i min(t_i, w_i |a x_i - y_i|) over
 * its local minima at those candidates (truncated; element 0 when there is none).  Candidate keys are the reference's fp32 values;
 * prefix sums and objectives are fp64.  Inputs are contiguous fp32 device arrays.  Elements per problem are bounded: plain problems
 * at n <= 12288, anchored ones at n <= 4096 points (the 64x64 grid of the reference's callers); larger n fails before any launch.
 * The truncated solvers and the anchored ones need a workspace (256-byte aligned) of moge_align_workspace_bytes; it depends on the
 * current device's SM count.  Results are deterministic and do not depend on the other problems of the batch. */
enum { MOGE_ALIGN_PLAIN = 0, MOGE_ANCHOR_DEPTH = 1, MOGE_ANCHOR_POINTS_Z = 2, MOGE_ANCHOR_POINTS_XYZ = 3 };
int moge_align_workspace_bytes(int mode, int truncated, int64_t batch, int n, size_t* bytes);
/* align(): `batch` problems of n elements, rows x, y, w (batch, n).  trunc: NULL = untruncated, else a device pointer to one scalar
 * (trunc_per_elem = 0) or to (batch, n) values.  Outputs (batch,): a = y_i / max(x_i, 1e-7) at the chosen element (signs flipped),
 * loss = the objective there, index = the element.                                                                           */
int moge_align(const float* x, const float* y, const float* w, const float* trunc, int trunc_per_elem, int64_t batch, int n, float* a,
               float* loss, int64_t* index, void* workspace, size_t workspace_bytes, void* stream);
/* the anchored solvers (alignment.py:163-214 depth affine, 251-302 points scale + z shift, 305-355 points scale + xyz shift):
 * src, tgt (batch, n) for MOGE_ANCHOR_DEPTH, else (batch, n, 3); w (batch, n).  For every anchor p with w_p > 0 the problem
 * x = src - src_p, y = tgt - tgt_p (POINTS_Z: only z is anchored; points are flattened to 3n elements, w repeated) is solved;
 * trunc < 0 = untruncated.  Per image: the least (loss, anchor, index), ties to the smallest anchor then index; an image
 * without a positive weight gets loss = +inf, anchor = index = -1.                                                          */
int moge_align_anchored(const float* src, const float* tgt, const float* w, int mode, float trunc, int64_t batch, int n, float* loss,
                        int64_t* anchor, int64_t* index, void* workspace, size_t workspace_bytes, void* stream);
/* align_affine_lstsq (alignment.py:399-416): the least-squares solution of [sqrt(w) x, 1] (a, b)^T = sqrt(w) y per problem, as the
 * reference's torch.linalg.lstsq call poses it (the column of ones is not weighted); w NULL = 1.  fp64 accumulation, any n.  */
int moge_align_affine_lstsq(const float* x, const float* y, const float* w, int64_t batch, int64_t n, float* a, float* b, void* stream);

/* ---- evaluation metrics (moge/test/metrics.py; Python: moge_b200.metrics, alias moge.test.metrics).
 * Images are (batch, H, W) fp32 maps, (batch, H, W, 3) point maps and a (batch, H, W) uint8 mask, contiguous on the device.
 * Every floating-point reduction is fp64 over fixed tiles set by H x W, summed in a fixed order: results do not change from run
 * to run nor with the other images of the batch.  A variant is a prediction map plus per-image params (batch, 4) on the device:
 * depth kinds read (scale, shift, clamp, -), points kinds (scale, shift x, y, z).  The aligned value is formed in fp32 with one
 * rounding per operation: x s, x s + b, 1 / max(d s + b, clamp) with d = x or 1 / x, x + shift, x s + shift.          */
#define MOGE_METRICS_MAX_SEGMENTS 256     /* segment ids per image */
#define MOGE_METRICS_MAX_VARIANTS 8
#define MOGE_METRICS_F1_THRESHOLDS 10
#define MOGE_METRICS_F1_COUNTS 90         /* per image: (radius 1..3, threshold, {TP, GT, pred}) */
#define MOGE_METRICS_OUT_SEGMENTS 17      /* moge_metrics_eval output: first per-segment entry */
enum { MOGE_MV_DEPTH = 0, MOGE_MV_DEPTH_SCALE = 1, MOGE_MV_DEPTH_AFFINE = 2, MOGE_MV_DISPARITY = 3, MOGE_MV_DISPARITY_FROM_DEPTH = 4,
       MOGE_MV_POINTS_SHIFT = 5, MOGE_MV_POINTS_SCALE = 6, MOGE_MV_POINTS_AFFINE = 7 };
typedef struct { int kind; const float* src; const float* params; } moge_metric_variant_t;
/* workspace (256-byte aligned) of moge_metrics_stats / moge_metrics_eval for S segment slots per image (0 <= S <= 256) */
int moge_metrics_workspace_bytes(int64_t batch, int H, int W, int S, size_t* bytes);
/* masked nearest resize to th x tw (utils3d.pt.masked_nearest_resize): lr_mask, lr_index (flat source pixel) (batch, th, tw); the
 * valid targets in row-major order as list (batch, th*tw) with list_w = 1, padded by the first entry at list_w = 0; count (batch). */
int moge_metrics_resize(const uint8_t* mask, int64_t batch, int H, int W, int th, int tw, uint8_t* lr_mask, int64_t* lr_index,
                        int64_t* list, float* list_w, int32_t* count, void* stream);
/* statistics: disp_params (batch, 4) = the least-squares (scale, shift) of disparity (disp_src, or 1 / disp_src when
 * disp_from_depth; NULL: NaN) against 1 / gt_depth over the mask, fp32(1 / (double) max masked GT), max masked GT.  With a
 * segmentation map seg (batch, H, W) int32, seg_ids (batch, S) sorted unique per image and seg_count (batch) ids in use:
 * diameter (batch, S) = max over xyz of the extent of the GT points over (seg == id) & mask (NaN when empty).            */
int moge_metrics_stats(const float* gt_depth, const float* gt_points, const uint8_t* mask, const float* disp_src, int disp_from_depth,
                       const int32_t* seg, const int32_t* seg_ids, const int32_t* seg_count, int S, int64_t batch, int H, int W,
                       float* disp_params, float* diameter, void* workspace, size_t workspace_bytes, void* stream);
/* metric pass: out (batch, out_stride) doubles: [2v] = sum of rel, [2v + 1] = delta1 count of variant v, [16] = mask count; with
 * segments, [17 + 3s + {0, 1, 2}] = (sum of |p - g| / diameter, count of |p - g| < 0.25 diameter, pixels) of slot s, where p is
 * local_src aligned by seg_params (batch, S, 4) (scale, shift xyz).                                                        */
int moge_metrics_eval(const float* gt_depth, const float* gt_points, const uint8_t* mask, const moge_metric_variant_t* variants,
                      int num_variants, const float* local_src, const int32_t* seg, const int32_t* seg_ids, const int32_t* seg_count, int S,
                      const float* seg_params, const float* seg_diameter, int64_t batch, int H, int W, double* out, int64_t out_stride,
                      void* workspace, size_t workspace_bytes, void* stream);
/* boundary F1 counts of a depth variant against gt_depth for radii 1, 2, 3 and the 10 sorted thresholds (host array): ADDED to
 * counts (batch, counts_stride) int64 at [(r - 1) * 30 + t * 3 + {TP, GT, pred}]; the caller zeroes them.                    */
int moge_metrics_boundary(const float* gt_depth, const uint8_t* mask, const moge_metric_variant_t* aligned, const float* thresholds,
                          int64_t batch, int H, int W, int64_t* counts, int64_t counts_stride, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* MOGE_B200_H */
