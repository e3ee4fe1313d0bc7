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

/* replaces MoGeModel.forward (v2.py:138-192).  A call carries `n` shape groups; one image shape is a call with one group.
 * Per group: image (B,3,H,W) in [0,1], dtype image_dtype; h,w its token grid (v2.py:142-147, computed by the caller).  Outputs
 * are fp32, caller-allocated; pass NULL for absent heads.
 * Mixed-shape ("ragged") batches -- BASELINE.json configs[2]; the reference has no counterpart (a batch tensor has one shape and
 * its nested-tensor path, dinov2/layers/block.py:160-259, is dead code without xformers).  The encoder (every linear, the
 * attention) runs ONCE over the token rows of all groups packed back to back, the per-pixel stages (resize/patchify, pos embed,
 * decoder, output resize) run group by group. */
typedef struct moge_group {
    const void* image;          /* (B,3,H,W) in [0,1] */
    int image_dtype;            /* MOGE_F32 / MOGE_F16 / MOGE_BF16 */
    int B, H, W, h, w;          /* images, pixels, token grid of this group (computed by the caller) */
    float* points;              /* (B,H,W,3) or NULL */
    float* normal;              /* (B,H,W,3) or NULL */
    float* mask_prob;           /* (B,H,W) or NULL */
    float* metric_scale;        /* (B,) or NULL */
} moge_group_t;
/* workspace (activations) size for a forward of these groups */
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

/* ---- operator-level entry points of the encoder's row plumbing, each running the engine's kernels with its arguments and in its
 * order.  T = h*w patch tokens per image, N = T + 1 rows per image (the cls row first).  LayerNorm statistics `stats` are float2
 * (sum, sum of squares) per row and column group, MOGE_STATS_LD slots per row; `parts` is the number of groups a producer wrote. */
#define MOGE_STATS_LD 16
/* K1 (build_plan "preprocess"): antialiased bilinear resize of image (B,3,H,W) (dtype MOGE_F32/F16/BF16) to (14h, 14w), ImageNet
 * normalisation, im2col -> patches (B*T, 592) 16-bit, column (c, py, px) = c*196 + py*14 + px, columns 588..591 zero. */
int moge_op_preprocess(const void* image, int image_dtype, int B, int H, int W, int h, int w, void* patches, int dtype, void* stream);
/* K3 (plan time, "pos table"): table (T, D) fp32 = bicubic resampling of the 37 x 37 grid of pos_embed (1 + 37*37, D) at scale
 * ((h+0.1)/37, (w+0.1)/37), + patch_bias (D); cls_row (D) = cls_token + pos_embed[0]. */
int moge_op_pos_table(const float* pos_embed, const float* cls_token, const float* patch_bias, int D, int h, int w, float* table,
                      float* cls_row, void* stream);
/* The encoder's front end for one group ("preprocess", "gemm.patch_embed", "init_cls", "ln_prepare.cls"): pos table, preprocess,
 * the (D,3,14,14) weight w_patch packed to (D, 592), then x (B*N, D) fp32 with row b*N+1+t = patches[b*T+t] w^T + table[t] and
 * row b*N = cls_row; x16 (B*N, D) its 16-bit copy, stats (B*N, MOGE_STATS_LD) the producer's partial sums (cls rows: slot 0, the
 * other `*parts` slots zero). */
int moge_op_patch_embed(const void* image, int image_dtype, int B, int H, int W, int h, int w, const float* w_patch, const float* b_patch,
                        const float* pos_embed, const float* cls_token, int D, float* x, void* x16, float* stats, int* parts, int dtype,
                        void* stream);
/* "gemm.proj" / "gemm.fc2": x (M,N) fp32 += gamma * (a (M,K) w (N,K)^T + bias), a and w 16-bit, with the LayerNorm producer side:
 * x16 (M,N) the rounded new rows, stats (M, MOGE_STATS_LD) their partial sums, *parts the groups per row.  Fails, launching
 * nothing, when N needs more groups than MOGE_STATS_LD.  K % 8 == 0, N % 128 == 0. */
int moge_op_linear_resid_ln(const void* a, const void* w, const float* bias, const float* gamma, float* x, void* x16, float* stats,
                            int* parts, int M, int N, int K, int dtype, void* stream);
/* "ln_rstd": rstd[r] = 1 / sqrt(E[x^2] - E[x]^2 + 1e-6) over D columns from slots [0, parts) of stats row r. */
int moge_op_ln_rstd(const float* stats, int parts, int rows, int D, float* rstd, void* stream);
/* "gemm.qkv" / "gemm.fc1" on given rows: out (M,N) 16-bit = epi(LayerNorm(x) w^T + bias) from the rounded rows x16 (M,K) and
 * their rstd (M), with the folded weight of moge_op_linear_ln.  epi 0 = store, 1 = GELU.  K % 64 == 0, N % 128 == 0. */
int moge_op_linear_ln_rows(const void* x16, const float* rstd, const float* ln_gamma, const float* ln_beta, const float* w, const float* bias,
                           void* out, int M, int N, int K, int epi, int dtype, void* stream);
/* "layernorm.tap": LayerNorm(eps=1e-6) of x (B*N, D) fp32; patch row (b, t) -> out[(b*(N-1) + t) * ld_out + col_off + d] 16-bit,
 * the cls row of image b -> cls_out[b*D + d] fp32 (skipped when cls_out is NULL). */
int moge_op_layernorm_taps(const float* x, const float* gamma, const float* beta, void* out, float* cls_out, int B, int N, int D,
                           int ld_out, int col_off, int dtype, void* stream);

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
/* replaces MoGeModel.forward (v1.py:269-299), as moge_engine_forward_groups for MoGe-2: a call carries `n` (1..64) shape groups;
 * one image shape is a call with one group.  The encoder runs ONCE over the token rows of all groups packed back to back, the
 * resize, decoder and output resize run group by group through one set of decoder maps sized for the largest group.  Every group
 * is checked before anything runs.  Outputs are fp32.  Python: MoGeModel.forward / infer / infer_many (moge.model.v1). */
typedef struct moge_v1_group {
    const void* image;          /* (B,3,H,W) in [0,1] */
    int image_dtype;            /* MOGE_F32 / MOGE_F16 / MOGE_BF16 */
    int B, H, W;                /* images and pixels of this group */
    int rh, rw;                 /* its resized image (>= 14 each; v1.py:273-274: rh = int(H f), rw = int(W f)); token grid
                                   rh/14 x rw/14 */
    float* points;              /* (B,H,W,3), remapped */
    float* mask;                /* (B,H,W), the raw mask output (no sigmoid) */
} moge_v1_group_t;
/* workspace for a forward of these groups */
int moge_v1_workspace_bytes_groups(moge_engine_t* e, const moge_v1_group_t* groups, int n, size_t* bytes);
int moge_v1_forward_groups(moge_engine_t* e, const moge_v1_group_t* groups, int n, void* workspace, size_t workspace_bytes,
                           void* stream);
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

/* ---- the DINOv2 backbone on its own (moge/model/dinov2: models/vision_transformer.py DinoVisionTransformer, hub/backbones.py;
 * Python: moge_b200.dinov2, aliases under moge.model.dinov2).  The same encoder kernels as the MoGe engines; the input is an image
 * that is already normalised (no resize, no mean / std), its H and W multiples of 14.  moge_dino_create returns an engine that
 * destroy / set_weight / finalize / num_ops / op_info / profile take unchanged; its weight keys are the backbone's own state-dict
 * keys (patch_embed.proj.weight, blocks.{i}.attn.qkv.weight, norm.weight, pos_embed, ...; mask_token is not read).  Configs the
 * encoder kernels do not cover fail at create: registers, SwiGLU / identity FFNs (ViT-g), other patch sizes, antialiased or
 * offset-free pos-embed interpolation, head_dim != 64, embed_dim not a multiple of 128 or above 1024. */
enum { MOGE_DINO_FFN_MLP = 0, MOGE_DINO_FFN_SWIGLU = 1, MOGE_DINO_FFN_IDENTITY = 2 };
typedef struct moge_dino_config {
    int embed_dim, depth, num_heads;
    int patch_size;                       /* 14 only */
    int num_register_tokens;              /* 0 only */
    float interpolate_offset;             /* 0.1 only */
    int interpolate_antialias;            /* 0 only */
    int ffn_layer;                        /* MOGE_DINO_FFN_MLP only */
    int compute_dtype;                    /* MOGE_F16 or MOGE_BF16 */
} moge_dino_config_t;
int moge_dino_create(const moge_dino_config_t* cfg, int device, moge_engine_t** out);
/* forward flags: MOGE_DINO_NORM applies the final LayerNorm (`norm`) to the exported rows; MOGE_DINO_CHANNEL_MAJOR writes the
 * patch tokens as (B, D, h, w) instead of (B, T, D) */
#define MOGE_DINO_NORM 1
#define MOGE_DINO_CHANNEL_MAJOR 2
/* A call carries `n` (1..MOGE_DINO_MAX_GROUPS) shape groups; one image shape is a call with one group.  `layers` and `flags` apply
 * to every group.  Per group: x (B,3,H,W), dtype x_dtype (MOGE_F32/F16/BF16), normalised; h = H/14, w = W/14, T = h*w.  layers:
 * n_layers (0..depth) strictly increasing block indices; after block layers[j] the residual stream (or its final LayerNorm,
 * MOGE_DINO_NORM) is written, fp32:
 *   out_tokens  layer j at out_tokens + j*B*T*D, as (B,T,D) or, with MOGE_DINO_CHANNEL_MAJOR, (B,D,h,w)
 *   out_cls     layer j's class-token rows at out_cls + j*B*D, (B,D)
 *   out_prenorm the residual stream after the last block, (B,T+1,D), the class token first
 * Any output may be NULL.  Rows are normalised with fixed-order statistics and no atomics: the outputs of an image are bitwise the
 * same run to run.  The encoder runs once over the token rows of all groups packed back to back; the front end and each exported
 * block's export are one launch each over all groups.  An image's outputs are bitwise those it gets in a call of its own. */
#define MOGE_DINO_MAX_GROUPS 64
typedef struct moge_dino_group {
    const void* x; int x_dtype;
    int B, H, W;
    float* out_tokens; float* out_cls; float* out_prenorm;     /* any may be NULL */
} moge_dino_group_t;
int moge_dino_workspace_bytes_groups(moge_engine_t* e, const moge_dino_group_t* groups, int n, const int* layers, int n_layers,
                                     int flags, size_t* bytes);
int moge_dino_forward_groups(moge_engine_t* e, const moge_dino_group_t* groups, int n, const int* layers, int n_layers, int flags,
                             void* workspace, size_t workspace_bytes, void* stream);

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

/* ---- mesh export (moge/scripts/infer.py:124-150: utils3d's depth_map_edge and build_mesh_from_map; Python: moge_b200.mesh).
 * Maps are (batch, H, W[, C]) contiguous on the device, masks uint8 (nonzero = in), at most 2^30 pixels per image.  Results are
 * bitwise those of the numpy restatement in oracle/utils3d_mesh.py and do not depend on the other images of the batch.        */
#define MOGE_MESH_MAX_MAPS 8
#define MOGE_MESH_MAX_CHANNELS 4
/* map kinds: fp32 copied; uint8 / 255 in fp32; the pixel-centre UV ((j + 0.5) / W, (i + 0.5) / H) generated (src unused, 2 ch) */
enum { MOGE_MESH_F32 = 0, MOGE_MESH_U8_UNIT = 1, MOGE_MESH_UV = 2 };
enum { MOGE_MESH_HWC = 0, MOGE_MESH_CHW = 1 };
/* one attribute map: a source (batch, H, W, C) or (batch, C, H, W); each value x is written as x * sign[c], then + offset[c] when
 * offset[c] != 0, each one fp32 rounding; the rows of kept vertices go to dst (total vertices, C) at the image's first row.   */
typedef struct {
    const void* src; int kind; int channels; int layout;
    float sign[MOGE_MESH_MAX_CHANNELS]; float offset[MOGE_MESH_MAX_CHANNELS];
    float* dst;
} moge_mesh_map_t;
/* workspace (256-byte aligned) of moge_mesh_count / moge_mesh_build; one workspace carries the counts from one to the other */
int moge_mesh_workspace_bytes(int64_t batch, int H, int W, size_t* bytes);
/* depth_map_edge: diff = max(d) + max(-d) over the kernel_size x kernel_size window (3, 5 or 7; -inf outside the image and,
 * with mask, off it; NaN propagates), edge = diff > *atol | diff / d > *rtol (a NULL tolerance is not tested).  out (batch, H, W)
 * uint8 = edge, or keep & !edge when keep is given (the cleaned mask).                                                       */
int moge_depth_edge(const float* depth, const uint8_t* mask, const uint8_t* keep, int64_t batch, int H, int W, int kernel_size,
                    const float* atol, const float* rtol, uint8_t* out, void* stream);
/* point_map_to_normal_map (oracle/utils3d_normals.py, bitwise): points (batch, H, W, 3) fp32 -> normal (batch, H, W, 3), the
 * normalised sum of the four normalised neighbour cross products whose neighbours and centre are in mask (zero points off the
 * image; NULL mask: every product, including those against the zero padding).  With a mask, normals are 0 where no product is
 * valid.  normal_mask (batch, H, W) uint8 (may be NULL) = some product valid.                                               */
int moge_normal_map(const float* points, const uint8_t* mask, int64_t batch, int H, int W, float* normal, uint8_t* normal_mask, void* stream);
/* normal_map_edge: the largest arccos of the dot product of a pixel's normal with those of its kernel_size window (3, 5 or 7,
 * edge-padded; with mask, 0 where the window pixel is off it), max-pooled over the same window (NaN propagates), is compared
 * as fp64: edge = angle > tol (radians).  With and_edge (batch, H, W) uint8, edge &= and_edge; out (batch, H, W) uint8 = edge, or
 * keep & !edge when keep is given.  angle (may be NULL) receives the pooled fp32 angle map.  At most 65535 * 32 rows.      */
int moge_normal_edge(const float* normals, const uint8_t* mask, const uint8_t* and_edge, const uint8_t* keep, int64_t batch, int H, int W,
                     int kernel_size, double tol, uint8_t* out, float* angle, void* stream);
/* count pass: a quad (top-left pixel (i, j)) is kept when its four corners are in the mask (NULL: every quad), a vertex when a
 * kept quad uses it.  totals (batch, 4) int64 on the device = (vertices, quads, first vertex row, first quad) of each image in
 * the batch-wide outputs.                                                                                                   */
int moge_mesh_count(const uint8_t* mask, int64_t batch, int H, int W, int64_t* totals, void* workspace, size_t workspace_bytes, void* stream);
/* emit pass, after moge_mesh_count on the same mask, totals and workspace: the maps' rows at the kept vertices (row-major order)
 * and the faces as vertex indices local to each image, int32: quads [(i,j), (i+1,j), (i+1,j+1), (i,j+1)] in row-major order, or
 * with tri two triangles [a, b, c], [a, c, d] per quad (faces then holds 6 ints per quad).                                   */
int moge_mesh_build(const uint8_t* mask, int64_t batch, int H, int W, int tri, const moge_mesh_map_t* maps, int num_maps,
                    const int64_t* totals, int32_t* faces, void* workspace, size_t workspace_bytes, void* stream);

/* ---- panorama inference (moge/utils/panorama.py and moge/scripts/infer_panorama.py:83-122; Python: moge_b200.panorama).
 * A camera is the reference's fp32 extrinsics [R | t] (R row-major) and its normalised pinhole intrinsics in fp64.  Panorama
 * maps are equirectangular, h x w, at least 2 x 2 and at most 2^28 pixels.                                                  */
#define MOGE_PANORAMA_MAX_VIEWS 20
typedef struct { float R[9]; float t[3]; double fx, fy, cx, cy; } moge_panorama_camera_t;
/* Every call takes `n` (1..MOGE_PANORAMA_MAX_BATCH) entries, one per panorama, each with its own sizes and pointers, and one set of
 * cameras; a single panorama is a call with one entry.  Each kernel is one launch over all entries, and each panorama's result is
 * bitwise what it gets in a call of its own.  An entry's error names its index.  The entry count is checked first, and every
 * argument before the device is touched.                                                                                     */
#define MOGE_PANORAMA_MAX_BATCH 64
/* split_panorama_image: views_f32 (views total, 3, res, res) = value / 255 of cv2.remap(image, INTER_LINEAR, BORDER_CONSTANT 0) at
 * the panorama pixel of each view pixel's ray; grid (res) is the fp32 pixel-centre coordinate of uv_map; views_u8 (views total,
 * res, res, 3) the uint8 values (may be NULL).  Panorama k's image is (H, W, 3) uint8 RGB; its `views` views go to views_f32 /
 * views_u8 from view view0 on.                                                                                               */
typedef struct {
    const uint8_t* image;
    int H, W;
    int view0;
} moge_panorama_split_t;
int moge_panorama_split_groups(const moge_panorama_split_t* panos, int n, const moge_panorama_camera_t* cams, int views,
                               const float* grid, int res, float* views_f32, uint8_t* views_u8, void* stream);
/* One merge level of one panorama, h x w.  Each call reads the fields it names.
 * rhs: the level's right-hand side.  src (views total, vh, vw, channels) fp32 is the distance (channels 1) or the point map whose
 * norm is the distance (channels 3), mask (views total, vh, vw) uint8; the entry's views are view0 .. view0 + views - 1 of them.
 * directions (h, w, 3) fp32 are the panorama rays.  b fp64 and row_mask uint8 hold 2hw + (h-1)(w+1) rows in the reference's
 * order: x-gradient h*w, y-gradient (h-1) x (w+1) (column w repeats column 0, as the reference's x-wrapped grid does), Laplacian
 * h*w; b = 0 where masked out.  pano_mask (h, w) uint8 = any view's mask.
 * lsmr: SciPy's lsmr(A, b, atol = btol = 1e-5, x0 = log(init)) on the rows of row_mask (init NULL: x0 = None), depth (h, w) fp32
 * = exp(x); stats (2) int32 on the device = (iterations, istop).  The systems of one call share one cooperative launch, which ends
 * when every system has stopped; no host synchronisation.  A system's reductions depend on its own size only, so it gets bitwise
 * its single-call result.
 * workspace_bytes: the workspace (256-byte aligned) of rhs and lsmr.  The workspace of a call fits any call whose entries are
 * each no larger (so the finest levels' workspace serves every coarser level).                                               */
typedef struct {
    int h, w;
    int view0;
    const float* directions;
    double* b;
    uint8_t* row_mask;
    uint8_t* pano_mask;
    const float* init;
    float* depth;
    int32_t* stats;
} moge_panorama_level_t;
int moge_panorama_workspace_bytes_groups(const moge_panorama_level_t* levels, int n, int views, size_t* bytes);
int moge_panorama_rhs_groups(const float* src, int channels, const uint8_t* mask, int views, int vh, int vw,
                             const moge_panorama_camera_t* cams, const moge_panorama_level_t* levels, int n, void* workspace,
                             size_t workspace_bytes, void* stream);
int moge_panorama_lsmr_groups(const moge_panorama_level_t* levels, int n, void* workspace, size_t workspace_bytes, void* stream);
/* cv2.resize(src, (W, H), INTER_LINEAR) of fp32 maps, src (h, w) -> dst (H, W): the pyramid's upsampling */
typedef struct {
    const float* src;
    int h, w, H, W;
    float* dst;
} moge_panorama_resize_t;
int moge_panorama_resize_groups(const moge_panorama_resize_t* maps, int n, void* stream);
/* infer_panorama.py:120-122: from depth (h, w) and mask (h, w), depth_out (H, W) the resized depth, mask_out (H, W) uint8 the
 * bilinear resize of the 0/1 mask > 0, points (H, W, 3) = depth_out * spherical_uv_to_directions(uv_map(H, W)).              */
typedef struct {
    const float* depth;
    const uint8_t* mask;
    int h, w, H, W;
    float* depth_out;
    uint8_t* mask_out;
    float* points;
} moge_panorama_finish_t;
int moge_panorama_finish_groups(const moge_panorama_finish_t* maps, int n, void* stream);

/* ---- training losses of moge/train/losses.py (Python: moge_b200.losses, moge_b200.local_loss; alias moge.train.losses).
 * Maps are (batch, H, W) fp32 and point maps (batch, H, W, 3) fp32, contiguous on the device.  Each call either reduces
 * (coef NULL): sums (batch, MOGE_LOSS_SUMS) doubles, fp64 over fixed tiles set by H x W and added in tile order, so results do
 * not change from run to run nor with the other images of the batch; or computes a gradient (coef given): grad = coef[image]
 * times the derivative of the per-pixel term, each pixel written by one thread, no atomics.  A GT point is valid when its three
 * coordinates are finite; an invalid one reads as (1, 1, 1), as in the reference.                                          */
#define MOGE_LOSS_SUMS 4                  /* doubles per image in every sums output */
enum { MOGE_LOSS_MASK_L2 = 0, MOGE_LOSS_MASK_BCE = 1, MOGE_LOSS_EDGE = 2, MOGE_LOSS_NORMAL = 3 };
/* workspace (256-byte aligned) of every loss call on (batch, H, W) */
int moge_loss_workspace_bytes(int64_t batch, int H, int W, size_t* bytes);
/* per-pixel mask losses of pred (batch, H, W) with per-pixel factors a, b:
 *   MOGE_LOSS_MASK_L2:  a = gt_mask_neg, b = gt_mask_pos, term a x^2 + b (1 - x)^2;
 *   MOGE_LOSS_MASK_BCE: a = gt_mask_pos | gt_mask_neg, b = gt_mask_pos, term a (-(b max(log x, -100) + (1 - b) max(log(1 - x), -100)))
 *     with torch's gradient (x - b) / max(x (1 - x), 1e-12).
 * sums[0] = sum of the terms; coef (batch) fp32. */
int moge_loss_mask(int kind, const float* pred, const float* a, const float* b, int64_t batch, int H, int W, const float* coef,
                   float* grad, double* sums, void* workspace, size_t workspace_bytes, void* stream);
/* stencil losses of points against gt (raw, invalid points allowed), the term smooth(clamp(atan2(|v x u| + 1e-12, v . u), lo, hi))
 * of a predicted vector v and its GT vector u, counted where the GT points it is built from are valid:
 *   MOGE_LOSS_EDGE:   v = p[i, j] - p[i+1, j] (sums[0], coef[2 image]) and p[i, j] - p[i, j+1] (sums[1], coef[2 image + 1]),
 *                     lo = 0.1 deg;
 *   MOGE_LOSS_NORMAL: the four triangle normals of each quad (sums[0], coef[2 image]), lo = 1 deg.
 * hi = 90 deg, smooth(e) = e < beta ? e^2 / (2 beta) : e - beta / 2 with beta = 3 deg.  The gradient follows torch autograd:
 * clamp passes it at its bounds, |0| has gradient 0.  coef (batch, 2) fp32. */
int moge_loss_stencil(int kind, const float* points, const float* gt, int64_t batch, int H, int W, const float* coef, float* grad,
                      double* sums, void* workspace, size_t workspace_bytes, void* stream);
/* normal map loss of pred (batch, H, W, 3) against gt (raw, invalid normals allowed): the term mask theta^2 per pixel, with theta
 * = angle_between(p, g) = 2 atan2(|p^ - g^|, |p^ + g^|), v^ = v / |v| (utils3d's half-angle form); mask multiplies, so a NaN
 * theta at an invalid pixel (a zero or non-finite prediction) still gives NaN.  sums[0] = sum of the terms; coef (batch) fp32.
 * The gradient is 0 where theta is exactly 0 or pi, as in torch autograd, and NaN where theta is. */
int moge_loss_normal_map(const float* pred, const float* gt, int64_t batch, int H, int W, const float* coef, float* grad,
                         double* sums, void* workspace, size_t workspace_bytes, void* stream);
/* affine-invariant global loss of pred (batch, H, W, 3) against gt, params (batch, 8) fp32 per image = (scale, shift x, y, z,
 * valid (0 / 1), cap, coef, -), with w = valid & mask / max(gt z, 1e-5) and the aligned point q = scale p + shift:
 *   pass 0: sums = (sum of w, mask count);
 *   pass 1: sums = (sum over coordinates of smooth(|q - g| min(w, cap)), sum over the mask of min(|q - g| / gt z, 1), count of
 *           |q - g| / gt z < 1 over the mask), smooth as above with `beta` (0: identity);
 *   pass 2: grad = d(pass 1's first sum)/dp times coef, sums = (dL/dscale, dL/dshift x, y, z).  */
int moge_loss_global(const float* pred, const float* gt, const float* params, float beta, int pass, int64_t batch, int H, int W,
                     float* grad, double* sums, void* workspace, size_t workspace_bytes, void* stream);
/* sampled local loss.  compute_anchor_sampling_weight's per-pixel pass: pixel (b, i, j) with mask (batch, H, W) u8 counts the
 * num_test offsets di, dj (H, W, num_test) int64 (shared by the images) whose target (i + di, j + dj) is inside the map, valid
 * and within radius[b, i, j] of points[b, i, j] (fp32 |d| = sqrt((dx^2 + dy^2) + dz^2)); weight (batch, H, W) fp32 =
 * mask ? 1 / max(count, 1) : 0.  No workspace. */
int moge_loss_anchor_weight(const float* points, const uint8_t* mask, const int64_t* di, const int64_t* dj, const float* radius,
                            int64_t batch, int H, int W, int num_test, float* weight, void* stream);
/* the P <= 65535 patches of side S = 2 r + 1 around anchor (P, 3) int64 (image, i, j): radius (P) = (1 / focal[image]) *
 * half_level * gt z at the anchor; patch_mask (P, S, S) u8 marks the positions whose pixel is inside the map, valid in mask and
 * within radius of the anchor's GT point; count (P) int32 = the marked positions.  gt (batch, H, W, 3) raw. */
int moge_loss_patch_mask(const float* gt, const uint8_t* mask, const int64_t* anchor, const float* focal, float half_level,
                         int64_t batch, int H, int W, int64_t P, int r, uint8_t* patch_mask, int* count, float* radius, void* stream);
/* the local loss's passes.  params (P, MOGE_LOSS_LOCAL_PARAMS) fp32 per patch = (scale, shift x, y, z, valid (0 / 1), cap,
 * radius, coef); at a marked position of a valid patch, q = scale p + shift and w = 1 / max(gt z, cap):
 *   pass 0: sums (batch, 4) = (sum over valid GT of 1 / (z + 1e-7), valid count), per image (pred, anchor, params unused);
 *   pass 1: sums (P, 4) = (sum over xyz of smooth(|q - g| w), position count, sum of min(err, 1), count of err < 1) with
 *           err = |q - g| / radius, smooth as for moge_loss_global;
 *   pass 2: sums (P, 4) = (dL/dscale, dL/dshift x, y, z) of pass 1's first sum times coef; with grad (batch, H, W, 3), also
 *           dL/dpred, each pixel gathering its patches' terms in patch order.
 * Workspace: moge_loss_workspace_bytes(batch, H, W) for pass 0, (P, S, S) for passes 1 and 2. */
#define MOGE_LOSS_LOCAL_PARAMS 8
int moge_loss_local(const float* pred, const float* gt, const int64_t* anchor, const float* params, const uint8_t* patch_mask,
                    float beta, int pass, int64_t batch, int H, int W, int64_t P, int r, float* grad, double* sums, void* workspace,
                    size_t workspace_bytes, void* stream);

/* ---- map colourisation (moge/utils/vis.py: colorize_depth, colorize_depth_affine, colorize_disparity, colorize_normal;
 * Python: moge_b200.vis).  Maps are (batch, H, W) fp32 contiguous on the device, masks uint8 (nonzero = in), at most 2^30 pixels
 * per image.  Results are bitwise those of oracle/vis_port.py and do not depend on the other images of the batch.  Value kinds:
 * MOGE_VIS_DEPTH colours 1 / depth where depth > 0 (+inf depth is disparity 0), MOGE_VIS_VALUE the value itself; NaN values and
 * pixels off the mask are excluded.                                                                                        */
#define MOGE_VIS_MAX_QUANTILES 4
enum { MOGE_VIS_DEPTH = 0, MOGE_VIS_VALUE = 1 };
/* workspace (256-byte aligned) of moge_vis_quantiles */
int moge_vis_workspace_bytes(int64_t batch, int H, int W, size_t* bytes);
/* np.nanquantile(values, q[i]) of each image's valid values, linear method in fp32 (q is a host array of nq values in [0, 1]):
 * out (batch, nq) fp32 on the device, NaN for an image without a valid value.  Same bits on every run; no host wait.        */
int moge_vis_quantiles(const float* src, int kind, const uint8_t* mask, int64_t batch, int H, int W, const float* q, int nq, float* out,
                       void* workspace, size_t workspace_bytes, void* stream);
/* out (batch, H, W, 3) uint8 = the 256-entry RGB table lut (device, 768 bytes) at x * 256 with matplotlib's Colormap rules
 * (256 -> 255, below 0 -> entry 0, 256 or more -> entry 255, NaN -> black), x the value normalised by range (batch, 2) = (lo,
 * hi) on the device as (v - lo) / (hi - lo) (NULL: not normalised), then 1 - x when invert.  bgr swaps the channels.      */
int moge_vis_colorize(const float* src, int kind, int invert, const uint8_t* mask, int64_t batch, int H, int W, const float* range,
                      const uint8_t* lut, int bgr, uint8_t* out, void* stream);
/* colorize_normal: out (batch, H, W, 3) uint8 = trunc(clip(n * (0.5, -0.5, -0.5) + 0.5, 0, 1) * 255) in fp64 of normal (batch, H,
 * W, 3) fp32, n = 0 off the mask (may be NULL); bgr swaps the channels.                                                     */
int moge_vis_normal(const float* normal, const uint8_t* mask, int64_t batch, int H, int W, int bgr, uint8_t* out, void* stream);

/* ---- geometry utilities (moge/utils/geometry_torch.py: refine_depth_with_normal, dilate_with_mask, theshold_depth_change,
 * gaussian_blur_2d; Python: moge_b200.geometry).  Maps are (batch, H, W) fp32 contiguous on the device, masks uint8 (nonzero =
 * in), at most 2^30 pixels per map.  No atomics: the same inputs give the same bits on every run.  Kernel sizes are odd.     */
#define MOGE_GEOMETRY_MAX_REFINE_KERNEL 9
#define MOGE_GEOMETRY_MAX_POOL_KERNEL 15
#define MOGE_GEOMETRY_MAX_BLUR_KERNEL 31
enum { MOGE_DILATE_MEAN = 0, MOGE_DILATE_MIN = 1, MOGE_DILATE_MAX = 2, MOGE_DILATE_MEDIAN = 3 };
/* workspace (256-byte aligned) of moge_refine_depth_with_normal */
int moge_geometry_workspace_bytes(int64_t batch, int H, int W, size_t* bytes);
/* refine_depth_with_normal: depth is clamped to at least eps IN PLACE (NaN stays NaN); normal (batch, H, W, 3), intrinsics
 * (batch, 3, 3) fp32; out (batch, H, W) = exp of the log-depth after `iterations` Jacobi sweeps of the kernel_size (3 to
 * MOGE_GEOMETRY_MAX_REFINE_KERNEL) bilateral stencil at the pixels kernel_size / 2 or more from the border, the input
 * log-depth elsewhere. */
int moge_refine_depth_with_normal(float* depth, const float* normal, const float* intrinsics, int64_t batch, int H, int W,
                                  int iterations, float damp, float eps, int kernel_size, float* out, void* workspace,
                                  size_t workspace_bytes, void* stream);
/* one dilate_with_mask step over the 3 x 3 cross (outside the map: invalid): out = input where mask, else the filter
 * (MOGE_DILATE_*) of the valid neighbours; mask_out = mask or any valid neighbour.  out and mask_out must not alias the inputs. */
int moge_dilate_with_mask(const float* input, const uint8_t* mask, int64_t batch, int H, int W, int filter, float* out,
                          uint8_t* mask_out, void* stream);
/* theshold_depth_change: pool_max ? (masked window max > depth * factor) : (masked window min < depth * factor), out uint8 0 / 1;
 * the window is kernel_size (1 to MOGE_GEOMETRY_MAX_POOL_KERNEL) square, NaN propagating, factor = 1 +- rtol in fp32. */
int moge_threshold_depth_change(const float* depth, const uint8_t* mask, int64_t batch, int H, int W, int pool_max, float factor,
                                int kernel_size, uint8_t* out, void* stream);
/* gaussian_blur_2d of `planes` (H, W) maps with replicate padding: the kernel_size (1 to MOGE_GEOMETRY_MAX_BLUR_KERNEL) square
 * kernel is the outer product of the host array kernel1d (kernel_size fp32 values), each product rounded once in fp32. */
int moge_gaussian_blur_2d(const float* input, int64_t planes, int H, int W, const float* kernel1d, int kernel_size, float* out,
                          void* stream);

#ifdef __cplusplus
}
#endif
#endif /* MOGE_B200_H */
