// The one tensor-core kernel of the engine: a persistent, warp-specialised wgmma GEMM whose A operand is either
// a row-major matrix (encoder linears) or an 8x16-pixel window of a padded NHWC image shifted by a filter tap
// (decoder implicit-GEMM convolutions).  TMA -> 128B-swizzled smem ring -> wgmma (fp32 accumulators in registers)
// -> accumulator tile staged in shared memory -> fused epilogue.
//
// Roles (warpgroup-uniform): warpgroup 0 = TMA producer (one elected lane of warp 0), warpgroups 1 and 2 = consumers:
// each issues the wgmma of its 64 rows of the 128-row tile, then all eight consumer warps run the epilogue (warp ew owns
// rows 32 (ew & 3) .. +31; with 8 epilogue warps the two warps of a row quarter split the columns).
//
// Three main loops share the kernel (MODE):
//   MODE_GEMM   one stage = one 64-wide K block of A (row tile, or one filter tap's pixel window) and of B.
//   MODE_CONV64 3x3 convs with C_in = 64: the packed weights of the CTA's output-channel tile (9 taps [+ the fused 1x1 input
//               block]) are loaded ONCE and stay resident; a stage is one halo box (16 px x 10 rows, one per horizontal tap
//               offset) whose three 2 KB-aligned row windows are the A operands of the three vertical taps.
//   MODE_CONVH  3x3 convs with C_in >= 128: the same halo boxes per 64-channel block, the three vertical-tap weight blocks
//               streamed in the same stage.
//
// Reference ops covered (SURVEY.md 2c): K2 patch-embed, K4 qkv, K6 proj+LayerScale+residual, K7 fc1+GELU,
// K8 fc2+LayerScale+residual, K9 tap projection sum, K10/K11 1x1 + UV, K12 ConvTranspose2d k2s2, K13/K14 3x3
// replicate-padded conv with ReLU/residual, K17 head output projection.
#pragma once
#include "common.cuh"
#include <type_traits>

namespace mg {

enum : int { AMODE_ROWS = 0, AMODE_TILES = 1 };
enum : int {
    EPI_STORE16 = 0,   // out16[row, col] = T(acc + bias[col])
    EPI_GELU16 = 1,    // out16[row, col] = T(gelu(acc + bias[col]))
    EPI_RESID = 2,     // x32[row, col] += gamma[col] * (acc + bias[col])            (fp32 residual stream, in place)
    EPI_PATCH = 3,     // x32[b*(T+1)+1+t, col] = acc + table[t, col]                (patch embed + pos embed)
    EPI_DEC = 4,       // padded-NHWC decoder store: acc + bias (+ UV rank-2) (+ skip) -> raw and/or ReLU copies
    EPI_HEADOUT = 5,   // BN=16: (bilinear x2 + 3x3 conv + output 1x1) folded into one low-res 3x3 conv with 4 output phases,
                       //        + folded 1x1 of the high-res neck map -> fp32 maps at the high resolution
    EPI_NECKOUT = 6,   // BN=32: the neck's last level (bilinear x2 + 3x3 conv + UV 1x1) folded THROUGH the heads' last-level
                       //        input + output blocks: 4 phases x 8 components (points xyz, normal xyz, mask logit, pad) written
                       //        straight into the heads' fp32 output maps; the heads' EPI_HEADOUT launches then accumulate
};

enum : int { MODE_GEMM = 0, MODE_CONV64 = 1, MODE_CONVH = 2 };
constexpr int TILE_M = 128;
constexpr int TILE_K = 64;     // 64 x 16-bit = one 128-byte swizzle row
constexpr int TILE_PW = 16;    // pixel tile = 8 rows x 16 columns
constexpr int TILE_PH = 8;

struct GemmParams {
    // GEMM shape
    int M;                 // AMODE_ROWS: number of valid rows
    int N;                 // total output columns (multiple of BN)
    int ntaps;             // 1 (centre) or 9 (3x3)
    int kb_main;           // 64-wide K blocks per tap from the main source
    int kb_aux;            // 64-wide K blocks from the aux source (centre tap), appended after the taps
    int num_m_tiles, num_n_tiles;
    // pixel geometry (AMODE_TILES: of the A source; EPI_DEC/HEADOUT: output pixel grid derives from it)
    int B, H, W;           // A-source unpadded size (AMODE_ROWS + EPI_DEC: the h x w token grid)
    int tiles_x, tiles_y;
    // epilogue operands
    void* out0;            // EPI_STORE16/GELU16: T* ; EPI_RESID/PATCH: float* ; EPI_DEC: raw T* (or null) ; HEADOUT: float*
    void* out1;            // EPI_DEC: ReLU copy T* (or null); NECKOUT: normal map float4* (or null)
    void* out2;            // NECKOUT: mask-logit map float* (or null)
    int accum;             // HEADOUT: 1 = add to the values already in out0 (written by the NECKOUT launch)
    const float* bias;     // [N] (EPI_DEC shuffle: [C_out]); HEADOUT: [16]
    const float* vec1;     // EPI_RESID: gamma[N]; EPI_PATCH: table[T, N]; EPI_DEC: wu[C] (or null); HEADOUT: waux[ncomp,32] (or null)
    const float* vec2;     // EPI_DEC: wv[C]
    const void* skip;      // EPI_DEC: residual input, same geometry as out ; HEADOUT: neck level-4 map (T*, 32 ch, padded)
    int ldo;               // row pitch of out (elements): ROWS epilogues: N total; DEC: channels of the out buffer
    int T;                 // EPI_PATCH / ROWS+EPI_DEC: tokens per image
    int Ho, Wo, Hop, Wop;  // EPI_DEC/HEADOUT: output pixel grid and its padded allocation
    int shuffle;           // EPI_DEC: 1 = ConvTranspose2d k2s2 pixel shuffle (Ho = 2H, Wo = 2W), N = 4*C_out
    int ncomp;             // HEADOUT: 3 (float4 per pixel) or 1 (float per pixel)
    float su, sv;          // UV half extents
    // LayerNorm folded into the consuming GEMM (ROWS epilogues; see elementwise.cu "LayerNorm folded into the next GEMM")
    void* x16;                 // producers (EPI_RESID / EPI_PATCH): 16-bit copy of the rows written to out0 (pitch ldo), or null
    float2* stats_out;         // producers: [row, stats_ld] partial (sum, sum of squares) of the ROUNDED row, one per column group
    const float* ln_rstd;      // consumers (EPI_STORE16 / EPI_GELU16): 1/sqrt(var + eps) of the A rows; null = plain bias epilogue
    int stats_ld;              // partial sums per row in stats_out
};

// DF < 0: the EPI_DEC variant (raw / ReLU copies, skip, UV, pixel shuffle) is decided at run time from the params;
// DF >= 0: compile-time bit mask (DF_RAW | DF_RELU | DF_SKIP | DF_UV | DF_SHUFFLE) -- a much smaller hot loop.
enum : int { DF_RAW = 1, DF_RELU = 2, DF_SKIP = 4, DF_UV = 8, DF_SHUFFLE = 16 };
inline int dec_flags(const GemmParams& p) {
    return (p.out0 ? DF_RAW : 0) | (p.out1 ? DF_RELU : 0) | (p.skip ? DF_SKIP : 0) | (p.vec1 ? DF_UV : 0) | (p.shuffle ? DF_SHUFFLE : 0);
}

// One launch of gemm_kernel as gemm_linear / gemm_conv (gemm.cu) choose it: the kernel variant, its tensor maps and params.
struct GemmLaunch {
    int bn, mode, amode, epi;
    int df;                    // EPI_DEC: the compile-time DF mask of the variant, or -1 (run-time flags)
    bool bf16;
    CUtensorMap a, aux, b;     // A operand, aux A operand (fused 1x1 input block), weights
    GemmParams p;
};

template <int BN, int MODE = MODE_GEMM> struct GemmCfg {
    static constexpr int kHaloBytes = 160 * 128;                 // box {64 ch, 16 px, 10 rows}
    static constexpr int kABytes = (MODE == MODE_GEMM) ? TILE_M * 128 : kHaloBytes;
    static constexpr int kBBytes = (MODE == MODE_GEMM) ? BN * 128 : (MODE == MODE_CONVH) ? 3 * BN * 128 : 0;
    static constexpr int kStageBytes = kABytes + kBBytes;
    static constexpr int kResidentBytes = (MODE == MODE_CONV64) ? 10 * BN * 128 : 0;     // 9 taps + 1 aux block, each [BN][64]
    // accumulator tile staged for the epilogue: 32 x 32 fp32 blocks, [row quarter][column chunk]; float4 (r, q) of a block at
    // r * 8 + (q ^ (r & 7)) -- a lane reads its row conflict-free, 8 lanes x float4 read one row of the block conflict-free
    static constexpr int kChunks = (BN < 32) ? 1 : BN / 32;
    static constexpr int kAccBytes = TILE_M * kChunks * 32 * 4;
    static constexpr int kFixedBytes = kAccBytes + kResidentBytes + 1024 /*align slack*/ + 256 /*barriers*/;
    static constexpr int kFit = (kMaxDynSmem - kFixedBytes) / kStageBytes;
    static constexpr int kStages = kFit > 8 ? 8 : kFit;
    static constexpr int kEpiWarps = (BN >= 64) ? 8 : 4;
    static constexpr int kThreads = 384;
    static constexpr int kSmemBytes = kStages * kStageBytes + kFixedBytes;
    static constexpr int kColsPerWarp = (kEpiWarps == 8) ? BN / 2 : BN;
    static_assert(kStages >= 2, "gemm_kernel: fewer than two ring stages fit beside the accumulator tile");
    static_assert(kSmemBytes <= kMaxDynSmem, "gemm_kernel: stage ring + accumulator tile exceed the shared memory of one CTA");
    static_assert((2 * kStages + 1) * 8 <= 256, "gemm_kernel: barrier block overflows its 256 bytes");
};

// Block of the staged accumulator tile holding rows 32 quarter .. +31, columns col .. col + 31 (col a multiple of 32).
template <int BN>
__device__ __forceinline__ const float4* acc_block(const float4* stg, int quarter, int col) {
    return stg + (quarter * GemmCfg<BN>::kChunks + (col >> 5)) * 256;
}
// Consumer warpgroup g (rows 64 g .. +63) writes its m64nBN accumulator fragment into the staged tile.
template <int BN>
__device__ __forceinline__ void acc_stage(float4* stg, const float* d, int g, int wl, int lane) {
    float* s = reinterpret_cast<float*>(stg);
#pragma unroll
    for (int i = 0; i < BN / 2; i += 2) {
        const int row = 64 * g + 16 * wl + (lane >> 2) + 8 * ((i >> 1) & 1);
        const int col = 8 * (i >> 2) + 2 * (lane & 3);
        const int rl = row & 31, q = (col & 31) >> 2;
        float* blk = s + ((row >> 5) * GemmCfg<BN>::kChunks + (col >> 5)) * 1024;
        *reinterpret_cast<float2*>(blk + (rl * 8 + (q ^ (rl & 7))) * 4 + (col & 3)) = make_float2(d[i], d[i + 1]);
    }
}
// This lane's row (lane of the block) over the block's first 4 NQ columns.
template <int NQ>
__device__ __forceinline__ void acc_row(const float4* blk, int lane, float* v) {
#pragma unroll
    for (int q = 0; q < NQ; ++q) {
        const float4 t = blk[lane * 8 + (q ^ (lane & 7))];
        v[4 * q] = t.x; v[4 * q + 1] = t.y; v[4 * q + 2] = t.z; v[4 * q + 3] = t.w;
    }
}

// First image pixel (image b, row y0, column x0) of pixel tile mt (AMODE_TILES).
struct TileOrigin { int b, y0, x0; };
__device__ __forceinline__ TileOrigin tile_origin(const GemmParams& p, int mt) {
    const int per_img = p.tiles_x * p.tiles_y;
    TileOrigin o;
    o.b = mt / per_img;
    const int r = mt % per_img;
    o.y0 = (r / p.tiles_x) * TILE_PH;
    o.x0 = (r % p.tiles_x) * TILE_PW;
    return o;
}

// Exact-erf GELU (nn.GELU() default, vision_transformer.py:61) of two lanes: gelu(x) = relu(x) - 0.5 |x| erfc(|x|/sqrt2), with
// erfc(|x|/sqrt2) = 2^q(|x|), q a degree-5 fit of log2(erfc) on [0,6] (weighted for the GELU error; max |gelu error|
// 7e-7 in fp32, far below the 16-bit output rounding).  5 FMA + 1 MUFU.EX2 + 4 other instructions per lane instead of libdevice
// erff's ~25: the fc1 epilogue is bound by instruction issue.
// (No clamp of |x|: the polynomial keeps decreasing beyond the fitted range -- q(6) = -29.2, q(8) = -51.8, q(20) = -1019 -- so
// |x| * 2^q just underflows to 0 for large |x|; the clamp cost one instruction per element in an epilogue that is bound by
// instruction issue.)
__device__ __forceinline__ float2 gelu_erf2(float2 x) {
    const float2 ab = make_float2(fabsf(x.x), fabsf(x.y));
    const float2 ax = ab;
    float2 q = ffma2(make_float2(-4.804994387e-04f, -4.804994387e-04f), ax, make_float2(7.133518346e-03f, 7.133518346e-03f));
    q = ffma2(q, ax, make_float2(-5.194617063e-02f, -5.194617063e-02f));
    q = ffma2(q, ax, make_float2(-4.598676562e-01f, -4.598676562e-01f));
    q = ffma2(q, ax, make_float2(-1.150842190e+00f, -1.150842190e+00f));
    q = ffma2(q, ax, make_float2(-3.041332639e-05f, -3.041332639e-05f));
    const float2 t = fmul2(ab, make_float2(ex2_approx(q.x), ex2_approx(q.y)));
    return ffma2(make_float2(-0.5f, -0.5f), t, make_float2(fmaxf(x.x, 0.0f), fmaxf(x.y, 0.0f)));
}

// LayerNorm fold, consumer side: rstd of the 8 rows a lane serves after the transpose (row 4*i + sub of the warp's 32).  The
// loads of tile i+1 are issued while tile i is drained and consumed one iteration later (no latency on the critical path).
struct LnRows { float rs[8]; };
__device__ __forceinline__ void ln_load(const GemmParams& p, int mt, int quarter, int lane, LnRows& r) {
    const int sub = lane >> 3;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        const long grow = static_cast<long>(mt) * TILE_M + quarter * 32 + 4 * i + sub;
        r.rs[i] = (grow < p.M) ? p.ln_rstd[grow] : 1.f;
    }
}

// 16-byte store of 8 x 16-bit channels of one pixel into the 1-pixel border of a padded NHWC buffer, replicating the edge pixel
// (so that 3x3 taps of the consumer never need clamping).  Cold path: edge pixels only.
static __device__ __noinline__ void store_px_border16(uint8_t* base, int b, int Y, int X, int Ho, int Wo, int Hop, int Wop,
                                                      int ld, int c0, uint4 q) {
    uint8_t* centre = base + (((static_cast<size_t>(b) * Hop + Y + 1) * Wop + X + 1) * ld + c0) * 2;
    const int dy0 = (Y == 0) ? -1 : 0, dy1 = (Y == Ho - 1) ? 1 : 0;
    const int dx0 = (X == 0) ? -1 : 0, dx1 = (X == Wo - 1) ? 1 : 0;
    const ptrdiff_t rowp = static_cast<ptrdiff_t>(Wop) * ld * 2, colp = static_cast<ptrdiff_t>(ld) * 2;
    for (int dy = dy0; dy <= dy1; ++dy)
        for (int dx = dx0; dx <= dx1; ++dx)
            if (dy != 0 || dx != 0) *reinterpret_cast<uint4*>(centre + dy * rowp + dx * colp) = q;
}

// EPI_DEC epilogue (decoder maps, padded NHWC): after the 32x32 transpose every lane owns EIGHT channels of one pixel
// (4 lanes per pixel row, 8 pixels per warp instruction, 4 passes per chunk) and moves 16 bytes per load/store.
template <int BN, int COLS, int AMODE, bool BF16, int DF>
__device__ __forceinline__ void epilogue_dec16(const GemmParams& p, int mt, int nt, const float4* stg, int quarter, int lane,
                                               int col_begin) {
    using H = H16<BF16>;
    const bool has_raw = (DF < 0) ? (p.out0 != nullptr) : ((DF & DF_RAW) != 0);
    const bool has_relu = (DF < 0) ? (p.out1 != nullptr) : ((DF & DF_RELU) != 0);
    const bool has_skip = (DF < 0) ? (p.skip != nullptr) : ((DF & DF_SKIP) != 0);
    const bool has_uv = (DF < 0) ? (p.vec1 != nullptr) : ((DF & DF_UV) != 0);
    const bool shuffle = (DF < 0) ? (p.shuffle != 0) : ((DF & DF_SHUFFLE) != 0);
    const int sub = lane >> 2;        // which of the 8 rows of a pass this lane serves
    const int q8 = lane & 3;          // which group of 8 channels of the 32-column chunk
    int tile_b = 0, tile_y0 = 0, tile_x0 = 0;
    if (AMODE == AMODE_TILES) {
        const TileOrigin org = tile_origin(p, mt);
        tile_b = org.b; tile_y0 = org.y0; tile_x0 = org.x0;
    }
    bool ok[4];
    int rb[4], ry[4], rx[4], eflags[4];
    size_t roff[4];                   // byte offset of the centre output pixel (channel 0)
    const int sh = shuffle ? 2 : 1;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int rl = quarter * 32 + 8 * i + sub;
        if (AMODE == AMODE_ROWS) {
            const long grow = static_cast<long>(mt) * TILE_M + rl;
            ok[i] = grow < p.M;
            rb[i] = static_cast<int>(grow / p.T);
            const int t = static_cast<int>(grow % p.T);
            ry[i] = t / p.W; rx[i] = t % p.W;
        } else {
            rb[i] = tile_b;
            ry[i] = tile_y0 + rl / TILE_PW;
            rx[i] = tile_x0 + rl % TILE_PW;
            ok[i] = (ry[i] < p.H) && (rx[i] < p.W);
        }
        roff[i] = ((static_cast<size_t>(rb[i]) * p.Hop + sh * ry[i] + 1) * p.Wop + sh * rx[i] + 1) * p.ldo * 2;
        eflags[i] = (ry[i] == 0 ? 1 : 0) | (ry[i] == p.H - 1 ? 2 : 0) | (rx[i] == 0 ? 4 : 0) | (rx[i] == p.W - 1 ? 8 : 0);
    }
    const float inv_wo = 1.0f / static_cast<float>(p.Wo), inv_ho = 1.0f / static_cast<float>(p.Ho);
    // Interior tiles (every pixel inside the image and none on its border: most tiles of a large map) take a straight-line
    // path: no per-row validity predicates, no border-replication bookkeeping, which otherwise outweigh the useful work of this
    // epilogue.  The phase of a pixel-shuffle chunk comes from a shift when C_out is a power of two (every MoGe config) instead
    // of an integer division per chunk.
    bool interior;
    if (AMODE == AMODE_TILES) interior = tile_y0 > 0 && tile_x0 > 0 && tile_y0 + TILE_PH < p.H && tile_x0 + TILE_PW < p.W;
    else interior = false;
    const int ldo_shift = ((p.ldo & (p.ldo - 1)) == 0) ? (31 - __clz(p.ldo)) : -1;
    auto chunk = [&](int c, auto fast_tag) {
        constexpr bool FAST = decltype(fast_tag)::value;
        const float4* scr = acc_block<BN>(stg, quarter, col_begin + c);
        const int col = nt * BN + col_begin + c;
        int co = col + 8 * q8, qd = 0, qmask = 15;
        size_t qoff = 0;
        if (shuffle) {
            qd = (ldo_shift >= 0) ? (col >> ldo_shift) : (col / p.ldo);      // ldo == C_out; a 32-column chunk never straddles a phase
            co -= qd * p.ldo;
            qoff = (static_cast<size_t>(qd >> 1) * p.Wop + (qd & 1)) * p.ldo * 2;
            qmask = ((qd >> 1) ? 2 : 1) | ((qd & 1) ? 8 : 4);
        }
        qoff += static_cast<size_t>(co) * 2;
        const float4 b0 = *reinterpret_cast<const float4*>(p.bias + co), b1 = *reinterpret_cast<const float4*>(p.bias + co + 4);
        float4 g0 = make_float4(0.f, 0.f, 0.f, 0.f), g1 = g0, h0 = g0, h1 = g0;
        if (has_uv) {
            g0 = *reinterpret_cast<const float4*>(p.vec1 + co); g1 = *reinterpret_cast<const float4*>(p.vec1 + co + 4);
            h0 = *reinterpret_cast<const float4*>(p.vec2 + co); h1 = *reinterpret_cast<const float4*>(p.vec2 + co + 4);
        }
        // phase 1: all global reads of the chunk back to back
        uint4 sk[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            sk[i] = make_uint4(0u, 0u, 0u, 0u);
            if (has_skip && (FAST || ok[i])) sk[i] = *reinterpret_cast<const uint4*>(static_cast<const uint8_t*>(p.skip) + roff[i] + qoff);
        }
        // phase 2: math + 16-byte stores
        uint4 pk_raw[4], pk_relu[4];
        unsigned edge_rows = 0;
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const int rl = 8 * i + sub;
            float4 a0 = scr[rl * 8 + ((2 * q8) ^ (rl & 7))];
            float4 a1 = scr[rl * 8 + ((2 * q8 + 1) ^ (rl & 7))];
            if (!FAST && !ok[i]) continue;
            a0.x += b0.x; a0.y += b0.y; a0.z += b0.z; a0.w += b0.w;
            a1.x += b1.x; a1.y += b1.y; a1.z += b1.z; a1.w += b1.w;
            if (has_skip) {
                const float2 s0 = H::unpack(sk[i].x), s1 = H::unpack(sk[i].y), s2 = H::unpack(sk[i].z), s3 = H::unpack(sk[i].w);
                a0.x += s0.x; a0.y += s0.y; a0.z += s1.x; a0.w += s1.y;
                a1.x += s2.x; a1.y += s2.y; a1.z += s3.x; a1.w += s3.y;
            }
            if (has_uv) {
                const int X = sh * rx[i] + (qd & 1), Y = sh * ry[i] + (qd >> 1);
                const float uu = p.su * ((2 * X + 1) * inv_wo - 1.0f);
                const float vv = p.sv * ((2 * Y + 1) * inv_ho - 1.0f);
                a0.x += g0.x * uu + h0.x * vv; a0.y += g0.y * uu + h0.y * vv; a0.z += g0.z * uu + h0.z * vv; a0.w += g0.w * uu + h0.w * vv;
                a1.x += g1.x * uu + h1.x * vv; a1.y += g1.y * uu + h1.y * vv; a1.z += g1.z * uu + h1.z * vv; a1.w += g1.w * uu + h1.w * vv;
            }
            if (!FAST && (eflags[i] & qmask) != 0) edge_rows |= 1u << i;
            if (has_raw) {
                pk_raw[i] = make_uint4(H::pack(a0.x, a0.y), H::pack(a0.z, a0.w), H::pack(a1.x, a1.y), H::pack(a1.z, a1.w));
                *reinterpret_cast<uint4*>(static_cast<uint8_t*>(p.out0) + roff[i] + qoff) = pk_raw[i];
            }
            if (has_relu) {
                pk_relu[i] = make_uint4(H::pack(fmaxf(a0.x, 0.f), fmaxf(a0.y, 0.f)), H::pack(fmaxf(a0.z, 0.f), fmaxf(a0.w, 0.f)),
                                        H::pack(fmaxf(a1.x, 0.f), fmaxf(a1.y, 0.f)), H::pack(fmaxf(a1.z, 0.f), fmaxf(a1.w, 0.f)));
                *reinterpret_cast<uint4*>(static_cast<uint8_t*>(p.out1) + roff[i] + qoff) = pk_relu[i];
            }
        }
        if (!FAST && edge_rows != 0) {
#pragma unroll
            for (int i = 0; i < 4; ++i)
                if (edge_rows >> i & 1) {
                    const int X = sh * rx[i] + (qd & 1), Y = sh * ry[i] + (qd >> 1);
                    if (has_raw) store_px_border16(static_cast<uint8_t*>(p.out0), rb[i], Y, X, p.Ho, p.Wo, p.Hop, p.Wop, p.ldo, co, pk_raw[i]);
                    if (has_relu) store_px_border16(static_cast<uint8_t*>(p.out1), rb[i], Y, X, p.Ho, p.Wo, p.Hop, p.Wop, p.ldo, co, pk_relu[i]);
                }
        }
    };
    if (interior) {
#pragma unroll 1
        for (int c = 0; c < COLS; c += 32) chunk(c, std::true_type{});
    } else {
#pragma unroll 1
        for (int c = 0; c < COLS; c += 32) chunk(c, std::false_type{});
    }
}


// EPI_HEADOUT epilogue: lane = low-resolution pixel, 16 B (or 4 B) per lane, consecutive lanes = consecutive pixels of a tile row.
template <int BN, bool BF16>
__device__ __forceinline__ void epilogue_headout(const GemmParams& p, int mt, const float4* stg, int quarter, int lane) {
    using H = H16<BF16>;
    const int row = quarter * 32 + lane;
    const TileOrigin org = tile_origin(p, mt);
    const int b = org.b;
    const int py = org.y0 + row / TILE_PW;
    const int px = org.x0 + row % TILE_PW;
    const bool valid = (py < p.H) && (px < p.W);
    float v[16];
    acc_row<4>(acc_block<BN>(stg, quarter, 0), lane, v);
    if (valid) {
        // accumulator columns: (phase, component); phase (qy,qx) -> output pixel (2*py+qy, 2*px+qx)
#pragma unroll
        for (int ph = 0; ph < 4; ++ph) {
            const int Y = 2 * py + (ph >> 1), X = 2 * px + (ph & 1);
            float o[3];
#pragma unroll
            for (int k = 0; k < 3; ++k) o[k] = (k < p.ncomp) ? v[ph * p.ncomp + k] + p.bias[k] : 0.f;
            if (p.vec1 != nullptr) {
                const uint4* src = reinterpret_cast<const uint4*>(
                    static_cast<const uint8_t*>(p.skip) + ((static_cast<size_t>(b) * p.Hop + Y + 1) * p.Wop + X + 1) * 64);
#pragma unroll
                for (int q = 0; q < 4; ++q) {
                    const uint4 u = src[q];
                    const uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
                    for (int e = 0; e < 4; ++e) {
                        const float2 f = H::unpack(w[e]);
                        const int c = q * 8 + e * 2;
#pragma unroll
                        for (int k = 0; k < 3; ++k)
                            if (k < p.ncomp) o[k] += p.vec1[k * 32 + c] * f.x + p.vec1[k * 32 + c + 1] * f.y;
                    }
                }
            }
            const size_t pix = (static_cast<size_t>(b) * p.Ho + Y) * p.Wo + X;
            if (p.accum) {       // the neck's folded contribution is already there (EPI_NECKOUT)
                if (p.ncomp == 1) o[0] += static_cast<const float*>(p.out0)[pix];
                else { const float4 t = static_cast<const float4*>(p.out0)[pix]; o[0] += t.x; o[1] += t.y; o[2] += t.z; }
            }
            if (p.ncomp == 1) static_cast<float*>(p.out0)[pix] = o[0];
            else static_cast<float4*>(p.out0)[pix] = make_float4(o[0], o[1], o[2], 0.f);
        }
    }
    __syncwarp();
}

// EPI_NECKOUT epilogue: lane = low-resolution pixel; 32 accumulator columns = (phase, component).
template <int BN>
__device__ __forceinline__ void epilogue_neckout(const GemmParams& p, int mt, const float4* stg, int quarter, int lane) {
    const int row = quarter * 32 + lane;
    const TileOrigin org = tile_origin(p, mt);
    const int b = org.b;
    const int py = org.y0 + row / TILE_PW;
    const int px = org.x0 + row % TILE_PW;
    const bool valid = (py < p.H) && (px < p.W);
    float v[32];
    acc_row<8>(acc_block<BN>(stg, quarter, 0), lane, v);
    if (valid) {
        float b8[8], gu[8], gv[8];
#pragma unroll
        for (int k = 0; k < 8; ++k) { b8[k] = p.bias[k]; gu[k] = p.vec1[k]; gv[k] = p.vec2[k]; }
        const float inv_wo = 1.0f / static_cast<float>(p.Wo), inv_ho = 1.0f / static_cast<float>(p.Ho);
#pragma unroll
        for (int ph = 0; ph < 4; ++ph) {
            const int Y = 2 * py + (ph >> 1), X = 2 * px + (ph & 1);
            const float uu = p.su * ((2 * X + 1) * inv_wo - 1.0f);
            const float vv = p.sv * ((2 * Y + 1) * inv_ho - 1.0f);
            float o[8];
#pragma unroll
            for (int k = 0; k < 8; ++k) o[k] = v[ph * 8 + k] + b8[k] + gu[k] * uu + gv[k] * vv;
            const size_t pix = (static_cast<size_t>(b) * p.Ho + Y) * p.Wo + X;
            if (p.out0) static_cast<float4*>(p.out0)[pix] = make_float4(o[0], o[1], o[2], 0.f);
            if (p.out1) static_cast<float4*>(p.out1)[pix] = make_float4(o[3], o[4], o[5], 0.f);
            if (p.out2) static_cast<float*>(p.out2)[pix] = o[6];
        }
    }
    __syncwarp();
}

// Row-major epilogues (EPI_STORE16 / GELU16 / RESID / PATCH) of one epilogue warp (rows 32 quarter .. +31, columns
// [col_begin, col_begin+COLS)) from the staged tile `stg`: 8 lanes x float4 cover the 32 columns of one row of a block and each
// warp instruction touches 4 rows (4 x 128 B), fully coalesced.
template <int BN, int COLS, int EPI, bool BF16>
__device__ __forceinline__ void epilogue_rows(const GemmParams& p, int mt, int nt, const float4* stg, int quarter, int lane,
                                              int col_begin, bool ln_rows_on, LnRows lnr) {
    using H = H16<BF16>;
    const int sub = lane >> 3;        // which of the 4 rows of a pass this lane serves
    const int q4 = lane & 7;          // which float4 (4 columns) of the 32-column chunk
    // ---- the 8 rows this lane serves after the transpose (row = 4*i + sub of the warp's 32)
    bool ok[8];
    int rb[8], ry[8], rx[8];     // EPI_PATCH: image, token row and token column of the row
    size_t roff[8];      // element offset of the row in out0 / x16
    int xrow[8];         // row index in the output / statistics arrays
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        const int rl = quarter * 32 + 4 * i + sub;
        rb[i] = 0; ry[i] = 0; rx[i] = 0; roff[i] = 0; xrow[i] = 0;
        const long grow = static_cast<long>(mt) * TILE_M + rl;
        ok[i] = grow < p.M;
        xrow[i] = static_cast<int>(grow);
        roff[i] = static_cast<size_t>(grow) * p.ldo;
        if (EPI == EPI_PATCH) {
            rb[i] = static_cast<int>(grow / p.T);
            const int t = static_cast<int>(grow % p.T);
            ry[i] = t / p.W; rx[i] = t % p.W;
            xrow[i] = rb[i] * (p.T + 1) + 1 + t;
            roff[i] = static_cast<size_t>(xrow[i]) * p.ldo;
        }
    }
    // LayerNorm fold, consumer side: rstd and -rstd*mean of this lane's 8 rows from the producers' partial sums (the 8
    // lanes that share a row split the partials, fixed order -> deterministic)
    constexpr bool LN_CONS = EPI == EPI_STORE16 || EPI == EPI_GELU16;
    constexpr bool LN_PROD = EPI == EPI_RESID || EPI == EPI_PATCH;
    const bool ln_on = LN_CONS && ln_rows_on;
    const bool x16_on = LN_PROD && p.x16 != nullptr;
    float ln_rs[8], st1[8], st2[8];        // st1/st2 (producers): partial sums of x and x^2 of this lane's 8 rows
#pragma unroll
    for (int i = 0; i < 8; ++i) { ln_rs[i] = ln_on ? lnr.rs[i] : 1.f; st1[i] = 0.f; st2[i] = 0.f; }
    // Full row tiles (all but the last of a GEMM) take a path without the per-row validity predicates.
    const bool full_tile = (static_cast<long>(mt) + 1) * TILE_M <= static_cast<long>(p.M);
    auto chunk = [&](int c, auto full_tag) {
        constexpr bool FULL = decltype(full_tag)::value;
        const int col = nt * BN + col_begin + c;       // first global output column of this chunk
        const int co = col + 4 * q4;                   // this lane's 4 columns
        float4 pre[8];
        const float4* scr = acc_block<BN>(stg, quarter, col_begin + c);
        float4 bias4 = make_float4(0.f, 0.f, 0.f, 0.f), g4 = bias4;
        if (EPI != EPI_PATCH) bias4 = *reinterpret_cast<const float4*>(p.bias + co);
        if (EPI == EPI_RESID) g4 = *reinterpret_cast<const float4*>(p.vec1 + co);
        // ---- phase 1: issue every global READ of this chunk (residual / pos table) back to back, so their L2 latencies
        //      overlap instead of serialising behind the stores of the previous row
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            pre[i] = make_float4(0.f, 0.f, 0.f, 0.f);
            if (!FULL && !ok[i]) continue;
            if (EPI == EPI_RESID) {
                pre[i] = *reinterpret_cast<const float4*>(static_cast<const float*>(p.out0) + roff[i] + co);
            } else if (EPI == EPI_PATCH) {
                const int t = ry[i] * p.W + rx[i];
                pre[i] = *reinterpret_cast<const float4*>(p.vec1 + static_cast<size_t>(t) * p.ldo + co);
            }
        }
        // ---- phase 2: math + stores
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            const int rl = 4 * i + sub;
            float4 a = scr[rl * 8 + (q4 ^ (rl & 7))];
            if (!FULL && !ok[i]) continue;
            if (EPI == EPI_STORE16 || EPI == EPI_GELU16) {
                float2 a01, a23;
                if (ln_on) {      // LN(x) W^T + b = rstd * (x16 W''^T) + b'   (mean removal lives in the centred weight W'')
                    a01 = make_float2(fmaf(ln_rs[i], a.x, bias4.x), fmaf(ln_rs[i], a.y, bias4.y));
                    a23 = make_float2(fmaf(ln_rs[i], a.z, bias4.z), fmaf(ln_rs[i], a.w, bias4.w));
                } else {
                    a01 = make_float2(a.x + bias4.x, a.y + bias4.y);
                    a23 = make_float2(a.z + bias4.z, a.w + bias4.w);
                }
                if (EPI == EPI_GELU16) { a01 = gelu_erf2(a01); a23 = gelu_erf2(a23); }
                uint2 pk;
                pk.x = H::pack(a01.x, a01.y); pk.y = H::pack(a23.x, a23.y);
                *reinterpret_cast<uint2*>(static_cast<typename H::T*>(p.out0) + roff[i] + co) = pk;
            } else {          // EPI_RESID / EPI_PATCH: fp32 rows (+ the LayerNorm producer side: 16-bit copy and partial sums)
                float4 x;
                if (EPI == EPI_RESID) {
                    x = pre[i];
                    x.x += g4.x * (a.x + bias4.x); x.y += g4.y * (a.y + bias4.y);
                    x.z += g4.z * (a.z + bias4.z); x.w += g4.w * (a.w + bias4.w);
                } else {
                    x = make_float4(a.x + pre[i].x, a.y + pre[i].y, a.z + pre[i].z, a.w + pre[i].w);
                }
                *reinterpret_cast<float4*>(static_cast<float*>(p.out0) + roff[i] + co) = x;
                if (x16_on) {
                    uint2 pk;
                    pk.x = H::pack(x.x, x.y); pk.y = H::pack(x.z, x.w);
                    *reinterpret_cast<uint2*>(static_cast<typename H::T*>(p.x16) + roff[i] + co) = pk;
                    const float2 f0 = H::unpack(pk.x), f1 = H::unpack(pk.y);
                    const float2 s1 = fadd2(f0, f1), s2 = ffma2(f0, f0, fmul2(f1, f1));
                    st1[i] += s1.x + s1.y;
                    st2[i] += s2.x + s2.y;
                }
            }
        }
        __syncwarp();
    };
    if (full_tile) {
#pragma unroll 1
        for (int c = 0; c < COLS; c += 32) chunk(c, std::true_type{});
    } else {
#pragma unroll 1
        for (int c = 0; c < COLS; c += 32) chunk(c, std::false_type{});
    }
    // LayerNorm fold, producer side: partial (sum, sum of squares) of this warp's column group for each of its rows
    if (x16_on) {
        const int part = (nt * BN + col_begin) / COLS;
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            float a = st1[i], b = st2[i];
#pragma unroll
            for (int o = 1; o < 8; o <<= 1) { a += __shfl_xor_sync(0xffffffffu, a, o); b += __shfl_xor_sync(0xffffffffu, b, o); }
            if (q4 == 0 && ok[i]) p.stats_out[static_cast<size_t>(xrow[i]) * p.stats_ld + part] = make_float2(a, b);
        }
    }
}

template <int BN, int MODE, int AMODE, int EPI, bool BF16, int DF = -1>
__global__ void __launch_bounds__(384, 1)
gemm_kernel(const __grid_constant__ CUtensorMap mapA, const __grid_constant__ CUtensorMap mapAux,
            const __grid_constant__ CUtensorMap mapB, const GemmParams p) {
    static_assert(AMODE == AMODE_ROWS || EPI == EPI_DEC || EPI == EPI_HEADOUT || EPI == EPI_NECKOUT,
                  "gemm_kernel: a pixel-tile A operand pairs only with the decoder epilogues (DEC, HEADOUT, NECKOUT)");
    pdl_launch_dependents();      // (the wait sits after the barrier set-up below: that prologue overlaps the previous kernel's tail)
    using Cfg = GemmCfg<BN, MODE>;
    constexpr int S = Cfg::kStages;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
    float4* stg = reinterpret_cast<float4*>(smem + S * Cfg::kStageBytes);
    uint8_t* sW = smem + S * Cfg::kStageBytes + Cfg::kAccBytes;         // MODE_CONV64: resident weights
    uint64_t* full = reinterpret_cast<uint64_t*>(sW + Cfg::kResidentBytes);
    uint64_t* empty = full + S;
    uint64_t* wfull = empty + S;

    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;
    const int total_tiles = p.num_m_tiles * p.num_n_tiles;
    // stages per tile
    const int kb_taps = p.ntaps * p.kb_main;
    const int nstage = (MODE == MODE_GEMM) ? kb_taps + p.kb_aux : (MODE == MODE_CONV64) ? 3 + p.kb_aux : 3 * p.kb_main + p.kb_aux;

    if (threadIdx.x == 0) {
        tma_prefetch_desc(&mapA);
        tma_prefetch_desc(&mapB);
        if (p.kb_aux) tma_prefetch_desc(&mapAux);
        // empty: one arrival per consumer warp once its warpgroup's MMAs that read the stage have completed
        for (int s = 0; s < S; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], 8); }
        mbar_init(wfull, 1);
        fence_mbar_init();
    }
    __syncthreads();
    pdl_wait();

    if (warp < 4) {
        // ================================================================== TMA producer
        // (warp 0 stays CONVERGED and one elected lane issues: under `if (lane == 0)` the compiler has to assume an
        // arbitrary active mask and wraps every TMA instruction in an elect-and-retry loop)
        regs_dec<40>();
        if (warp != 0) return;
        if (MODE == MODE_CONV64) {
            // the weights of this CTA's output-channel tile (the grid is a multiple of num_n_tiles: nt is fixed per CTA)
            const int nblk = 9 + p.kb_aux;
            const int nt = static_cast<int>(blockIdx.x) % p.num_n_tiles;
            if (elect_one()) {
                mbar_arrive_expect_tx(wfull, nblk * BN * 128);
                for (int t = 0; t < nblk; ++t) tma_load_2d(sW + t * BN * 128, &mapB, wfull, t * TILE_K, nt * BN);
            }
            __syncwarp();
        }
        int s = 0; uint32_t ph = 0;
        for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
            const int mt = tile / p.num_n_tiles, nt = tile % p.num_n_tiles;
            int b = 0, x0 = 0, y0 = 0;
            if (AMODE == AMODE_TILES) {
                const TileOrigin org = tile_origin(p, mt);
                b = org.b; y0 = org.y0; x0 = org.x0;
            }
            for (int i = 0; i < nstage; ++i) {
                mbar_wait(&empty[s], ph ^ 1);
                uint8_t* sa = smem + s * Cfg::kStageBytes;
                uint8_t* sb = sa + Cfg::kABytes;
                if (elect_one()) {
                    if (MODE == MODE_GEMM) {
                        mbar_arrive_expect_tx(&full[s], Cfg::kStageBytes);
                        if (AMODE == AMODE_ROWS) {
                            tma_load_2d(sa, &mapA, &full[s], i * TILE_K, mt * TILE_M);
                        } else if (i < kb_taps) {
                            const int tap = i / p.kb_main, c = i % p.kb_main;
                            const int tx = (p.ntaps == 9) ? tap % 3 : 1, ty = (p.ntaps == 9) ? tap / 3 : 1;
                            tma_load_4d(sa, &mapA, &full[s], c * TILE_K, x0 + tx, y0 + ty, b);
                        } else {
                            tma_load_4d(sa, &mapAux, &full[s], (i - kb_taps) * TILE_K, x0 + 1, y0 + 1, b);
                        }
                        tma_load_2d(sb, &mapB, &full[s], i * TILE_K, nt * BN);
                    } else if (MODE == MODE_CONV64) {
                        if (i < 3) {
                            mbar_arrive_expect_tx(&full[s], Cfg::kHaloBytes);
                            tma_load_4d(sa, &mapA, &full[s], 0, x0 + i, y0, b);             // padded rows y0..y0+9 = taps dy 0..2
                        } else {
                            mbar_arrive_expect_tx(&full[s], TILE_M * 128);
                            tma_load_4d(sa, &mapAux, &full[s], 0, x0 + 1, y0 + 1, b);
                        }
                    } else {
                        // MODE_CONVH: stage i = (channel block c, horizontal tap dx): halo box + the weight blocks of dy = 0..2;
                        // the aux blocks (fused 1x1 source) follow: 8-row box + one weight block
                        const bool aux = i >= 3 * p.kb_main;
                        if (!aux) {
                            const int c = i / 3, dx = i % 3;
                            mbar_arrive_expect_tx(&full[s], Cfg::kHaloBytes + 3 * BN * 128);
                            tma_load_4d(sa, &mapA, &full[s], c * TILE_K, x0 + dx, y0, b);
                            for (int dy = 0; dy < 3; ++dy)
                                tma_load_2d(sb + dy * BN * 128, &mapB, &full[s], ((dy * 3 + dx) * p.kb_main + c) * TILE_K, nt * BN);
                        } else {
                            const int c = i - 3 * p.kb_main;
                            mbar_arrive_expect_tx(&full[s], TILE_M * 128 + BN * 128);
                            tma_load_4d(sa, &mapAux, &full[s], c * TILE_K, x0 + 1, y0 + 1, b);
                            tma_load_2d(sb, &mapB, &full[s], (9 * p.kb_main + c) * TILE_K, nt * BN);
                        }
                    }
                }
                __syncwarp();
                if (++s == S) { s = 0; ph ^= 1; }
            }
        }
    } else {
        // ================================================================== consumers: MMA, then epilogue
        regs_inc<232>();
        const int g = (warp - 4) >> 2;                  // consumer warpgroup: rows 64 g .. 64 g + 63 of the tile
        const int wl = warp & 3;
        const int ew = warp - 4;
        const int quarter = ew & 3;
        const int col_begin = (Cfg::kEpiWarps == 8) ? (ew >> 2) * (BN / 2) : 0;
        const uint32_t a_off = static_cast<uint32_t>(g) * 64 * 128;
        if (MODE == MODE_CONV64) mbar_wait(wfull, 0);
        const uint32_t w0 = smem_u32(sW);
        LnRows lnr{}, lnn{};
        const bool ln_on = AMODE == AMODE_ROWS && (EPI == EPI_STORE16 || EPI == EPI_GELU16) && p.ln_rstd != nullptr;
        if (ln_on && static_cast<int>(blockIdx.x) < total_tiles) ln_load(p, static_cast<int>(blockIdx.x) / p.num_n_tiles, quarter, lane, lnn);
        int s = 0; uint32_t ph = 0;
        for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
            const int mt = tile / p.num_n_tiles, nt = tile % p.num_n_tiles;
            if (ln_on) {        // rstd of this tile's rows (loaded one iteration ago); then issue the next tile's loads
                lnr = lnn;
                const int nxt = tile + static_cast<int>(gridDim.x);
                if (nxt < total_tiles) ln_load(p, nxt / p.num_n_tiles, quarter, lane, lnn);
            }
            float acc[BN / 2];
#pragma unroll
            for (int j = 0; j < BN / 2; ++j) acc[j] = 0.f;
            int prev = -1;
            for (int i = 0; i < nstage; ++i) {
                mbar_wait(&full[s], ph);
                const uint32_t sa = smem_u32(smem + s * Cfg::kStageBytes) + a_off;
                const uint32_t sb = smem_u32(smem + s * Cfg::kStageBytes + Cfg::kABytes);
                wgmma_fence();
                auto mma64 = [&](uint32_t a, uint32_t bb) {          // one 64-wide K block
                    const uint64_t ad = make_sdesc_sw128(a), bd = make_sdesc_sw128(bb);
#pragma unroll
                    for (int k = 0; k < TILE_K / 16; ++k) Wgmma<BN, BF16>::ss(acc, ad + 2 * k, bd + 2 * k, 1u);
                };
                if (MODE == MODE_GEMM) {
                    mma64(sa, sb);
                } else if (MODE == MODE_CONV64) {
                    if (i < 3) {
#pragma unroll
                        for (int dy = 0; dy < 3; ++dy) mma64(sa + dy * TILE_PW * 128, w0 + (dy * 3 + i) * BN * 128);
                    } else {
                        mma64(sa, w0 + 9 * BN * 128);
                    }
                } else {
                    if (i < 3 * p.kb_main) {
#pragma unroll
                        for (int dy = 0; dy < 3; ++dy) mma64(sa + dy * TILE_PW * 128, sb + dy * BN * 128);
                    } else {
                        mma64(sa, sb);
                    }
                }
                wgmma_commit();
                // the MMAs of the previous stage have completed once at most this stage's group is pending: release its slot
                wgmma_wait<1>();
                reg_fence(acc);
                if (prev >= 0 && lane == 0) mbar_arrive(&empty[prev]);
                prev = s;
                if (++s == S) { s = 0; ph ^= 1; }
            }
            wgmma_wait<0>();
            reg_fence(acc);
            if (prev >= 0 && lane == 0) mbar_arrive(&empty[prev]);
            named_sync(1, 256);                          // every epilogue warp is done reading the previous tile
            acc_stage<BN>(stg, acc, g, wl, lane);
            named_sync(1, 256);
            if (ew < Cfg::kEpiWarps) {
                if constexpr (EPI == EPI_DEC) epilogue_dec16<BN, Cfg::kColsPerWarp, AMODE, BF16, DF>(p, mt, nt, stg, quarter, lane, col_begin);
                else if constexpr (EPI == EPI_HEADOUT) epilogue_headout<BN, BF16>(p, mt, stg, quarter, lane);
                else if constexpr (EPI == EPI_NECKOUT) epilogue_neckout<BN>(p, mt, stg, quarter, lane);
                else epilogue_rows<BN, Cfg::kColsPerWarp, EPI, BF16>(p, mt, nt, stg, quarter, lane, col_begin, ln_on, lnr);
            }
        }
    }
}

}  // namespace mg
