// MoGe-1 kernels (reference moge/model/v1.py): the antialiased bicubic input resize, GroupNorm statistics and the fused
// normalise + affine + ReLU pass of the residual blocks, the input-grid UV term of the upsampling ConvTranspose, the bilinear
// resize of the last decoder map to the resized-image grid, the output block tail, and the v1 post-processing.
// Decoder maps are padded NHWC 16-bit (host_api.h Level): every kernel that writes one writes its replicated border too.
#include "common.cuh"
#include "host_api.h"
#include "moge_b200.h"
#include <math.h>
#include <algorithm>

namespace mg {

// ------------------------------------------------------------------------------------------ V1 antialiased bicubic resize
// F.interpolate(mode='bicubic', align_corners=False, antialias=True) (v1.py:275): per axis the PIL-style filter of ATen's
// _upsample_bicubic2d_aa -- support 2 * max(scale, 1), taps at (j - centre + 0.5) * min(1, 1/scale), Keys cubic with a = -0.5,
// weights normalised to sum 1, no clamping of the output.
// Tap positions and weights are computed in fp64: in fp32 the centre scale * (i + 0.5) of a 700-pixel axis is off by ~4e-5.
__host__ __device__ inline double cubic_aa(double x) {
    const double a = -0.5;
    x = fabs(x);
    if (x < 1.0) return ((a + 2.0) * x - (a + 3.0)) * x * x + 1.0;
    if (x < 2.0) return (((x - 5.0) * x + 8.0) * x - 4.0) * a;
    return 0.0;
}
struct CubicTaps { int lo, n; double centre, inv; };
__host__ __device__ inline CubicTaps cubic_taps(int in, int out, int i) {
    const double scale = static_cast<double>(in) / static_cast<double>(out);
    const double support = scale >= 1.0 ? 2.0 * scale : 2.0;
    CubicTaps t;
    t.centre = scale * (i + 0.5);
    t.inv = scale >= 1.0 ? 1.0 / scale : 1.0;
    const int lo = static_cast<int>(t.centre - support + 0.5);
    const int hi = static_cast<int>(t.centre + support + 0.5);
    t.lo = lo > 0 ? lo : 0;
    t.n = (hi < in ? hi : in) - t.lo;
    return t;
}
__host__ __device__ inline float cubic_tap_w(const CubicTaps& t, int j) { return static_cast<float>(cubic_aa((j + t.lo - t.centre + 0.5) * t.inv)); }

__device__ __forceinline__ float load_any(const void* p, int dtype, size_t idx) {
    if (dtype == MOGE_F32) return static_cast<const float*>(p)[idx];
    if (dtype == MOGE_F16) return __half2float(static_cast<const __half*>(p)[idx]);
    return __bfloat162float(static_cast<const __nv_bfloat16*>(p)[idx]);
}

// horizontal pass: rows of W pixels -> rows of Wo pixels (fp32)
__global__ void bicubic_h_kernel(const void* __restrict__ src, int dtype, size_t rows, int W, int Wo, float* __restrict__ dst) {
    pdl_prologue();
    const size_t total = rows * Wo;
    for (size_t idx = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; idx < total; idx += static_cast<size_t>(gridDim.x) * blockDim.x) {
        const int x = static_cast<int>(idx % Wo);
        const size_t r = idx / Wo;
        const CubicTaps t = cubic_taps(W, Wo, x);
        float acc = 0.f, ws = 0.f;
        for (int j = 0; j < t.n; ++j) {
            const float w = cubic_tap_w(t, j);
            ws += w;
            acc += w * load_any(src, dtype, r * W + t.lo + j);
        }
        dst[idx] = acc / ws;
    }
}
// vertical pass: planes of H x Wo -> Ho x Wo
__global__ void bicubic_v_kernel(const float* __restrict__ src, size_t planes, int H, int Ho, int Wo, float* __restrict__ dst) {
    pdl_prologue();
    const size_t total = planes * Ho * Wo;
    for (size_t idx = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; idx < total; idx += static_cast<size_t>(gridDim.x) * blockDim.x) {
        const int x = static_cast<int>(idx % Wo);
        const int y = static_cast<int>((idx / Wo) % Ho);
        const size_t p = idx / (static_cast<size_t>(Wo) * Ho);
        const CubicTaps t = cubic_taps(H, Ho, y);
        float acc = 0.f, ws = 0.f;
        for (int j = 0; j < t.n; ++j) {
            const float w = cubic_tap_w(t, j);
            ws += w;
            acc += w * src[(p * H + t.lo + j) * Wo + x];
        }
        dst[idx] = acc / ws;
    }
}

static int grid_for(size_t total) { return static_cast<int>(std::max<size_t>(1, std::min<size_t>((total + 255) / 256, 132 * 16))); }

int launch_resize_bicubic_aa(const void* image, int dtype, int B, int C, int H, int W, int Ho, int Wo, float* tmp, float* out, cudaStream_t st) {
    if (B <= 0 || C <= 0 || H <= 0 || W <= 0 || Ho <= 0 || Wo <= 0) return set_error("resize_bicubic_aa: bad shape");
    const size_t rows = static_cast<size_t>(B) * C * H;
    CUDA_TRY(launch_pdl(bicubic_h_kernel, dim3(grid_for(rows * Wo)), dim3(256), 0, st, image, dtype, rows, W, Wo, tmp));
    const size_t planes = static_cast<size_t>(B) * C;
    CUDA_TRY(launch_pdl(bicubic_v_kernel, dim3(grid_for(planes * Ho * Wo)), dim3(256), 0, st, static_cast<const float*>(tmp), planes, H, Ho, Wo, out));
    return 0;
}

int bicubic_aa_taps(int in, int out, int i, int* lo, float* w, int cap) {
    const CubicTaps t = cubic_taps(in, out, i);
    *lo = t.lo;
    if (w != nullptr) {
        if (t.n > cap) return set_error("bicubic_aa_weights: %d taps > cap %d", t.n, cap);
        float s = 0.f;
        for (int j = 0; j < t.n; ++j) s += cubic_tap_w(t, j);
        for (int j = 0; j < t.n; ++j) w[j] = cubic_tap_w(t, j) / s;
    }
    return t.n;
}

// ------------------------------------------------------------------------------------------ V6 GroupNorm
// nn.GroupNorm(G, C) (eps 1e-5, biased variance) over the interior of a padded NHWC map.  Statistics are deterministic: fixed
// pixel tiles per image, fp64 per-thread partial sums, fixed-order reductions (no atomics), fp64 finalisation.  A tile holds
// 32K elements (16 16-byte loads per thread), so that even one image of the smallest decoder level spans tens of CTAs; the tiling
// depends on the map shape only, never on the batch.
constexpr int GN_TILE_ELEMS = 32768;
static int gn_tile_px(int C) { return GN_TILE_ELEMS / C; }
int gn_tiles(int H, int W, int C) { return (H * W + gn_tile_px(C) - 1) / gn_tile_px(C); }

__device__ __forceinline__ void unpack8(uint4 q, float* f, bool bf16) {
    const uint32_t w[4] = {q.x, q.y, q.z, q.w};
#pragma unroll
    for (int e = 0; e < 4; ++e) {
        const float2 v = bf16 ? H16<true>::unpack(w[e]) : H16<false>::unpack(w[e]);
        f[2 * e] = v.x; f[2 * e + 1] = v.y;
    }
}
template <bool BF16>
__device__ __forceinline__ uint4 pack8(const float* f) {
    return make_uint4(H16<BF16>::pack(f[0], f[1]), H16<BF16>::pack(f[2], f[3]), H16<BF16>::pack(f[4], f[5]), H16<BF16>::pack(f[6], f[7]));
}
__device__ __forceinline__ size_t px_off(int b, int Y, int X, int Hp, int Wp, int C) {      // byte offset of padded pixel (Y, X)
    return ((static_cast<size_t>(b) * Hp + Y) * Wp + X) * static_cast<size_t>(C) * 2;
}

template <bool BF16>
__global__ void __launch_bounds__(256) gn_partial_kernel(const uint8_t* __restrict__ map, int Hp, int Wp, int H, int W, int C, int G, int tiles,
                                                         int tile_px, double2* __restrict__ part) {
    pdl_prologue();
    __shared__ double ss[256], sq[256];
    const int b = blockIdx.y, tile = blockIdx.x;
    const int lanes = C / 8, slots = 256 / lanes;
    const int lane = threadIdx.x % lanes, slot = threadIdx.x / lanes;
    double s = 0.0, q = 0.0;
    if (slot < slots) {
        const int p1 = min((tile + 1) * tile_px, H * W);
        for (int p = tile * tile_px + slot; p < p1; p += slots) {
            const int y = p / W, x = p % W;
            float f[8];
            unpack8(*reinterpret_cast<const uint4*>(map + px_off(b, y + 1, x + 1, Hp, Wp, C) + lane * 16), f, BF16);
#pragma unroll
            for (int e = 0; e < 8; ++e) { s += f[e]; q += static_cast<double>(f[e]) * f[e]; }
        }
    }
    ss[threadIdx.x] = s; sq[threadIdx.x] = q;
    __syncthreads();
    // fixed-order reduction: each lane over its slots, then each group over its lanes (channel octets lane*8 .. lane*8+7)
    if (threadIdx.x < lanes) {
        for (int sl = 1; sl < slots; ++sl) { s += ss[sl * lanes + threadIdx.x]; q += sq[sl * lanes + threadIdx.x]; }
        ss[threadIdx.x] = s; sq[threadIdx.x] = q;
    }
    __syncthreads();
    const int lpg = C / G / 8;
    for (int g = threadIdx.x; g < G; g += blockDim.x) {
        double a = 0.0, c = 0.0;
        for (int l = g * lpg; l < (g + 1) * lpg; ++l) { a += ss[l]; c += sq[l]; }
        part[(static_cast<size_t>(b) * tiles + tile) * G + g] = make_double2(a, c);
    }
}
// one CTA per (group, image): strided sums over the tiles, then a fixed shared-memory tree
__global__ void __launch_bounds__(256) gn_finalize_kernel(const double2* __restrict__ part, int tiles, int G, double inv_n,
                                                          float2* __restrict__ stats) {
    pdl_prologue();
    __shared__ double ss[256], sq[256];
    const int g = blockIdx.x, b = blockIdx.y;
    double s = 0.0, q = 0.0;
    for (int t = threadIdx.x; t < tiles; t += blockDim.x) {
        const double2 v = part[(static_cast<size_t>(b) * tiles + t) * G + g];
        s += v.x; q += v.y;
    }
    ss[threadIdx.x] = s; sq[threadIdx.x] = q;
    __syncthreads();
    for (int k = blockDim.x / 2; k > 0; k >>= 1) {
        if (threadIdx.x < k) { ss[threadIdx.x] += ss[threadIdx.x + k]; sq[threadIdx.x] += sq[threadIdx.x + k]; }
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        const double mean = ss[0] * inv_n;
        const double var = fmax(sq[0] * inv_n - mean * mean, 0.0);
        stats[static_cast<size_t>(b) * G + g] = make_float2(static_cast<float>(mean), static_cast<float>(1.0 / sqrt(var + 1e-5)));
    }
}
// relu(gamma * (x - mean) * rstd + beta) of every padded pixel, the border from the clamped interior pixel
template <bool BF16>
__global__ void gn_relu_kernel(const uint8_t* __restrict__ src, uint8_t* __restrict__ dst, int B, int Hp, int Wp, int H, int W, int C, int G,
                               const float2* __restrict__ stats, const float* __restrict__ gamma, const float* __restrict__ beta) {
    pdl_prologue();
    const int lanes = C / 8, cg = C / G;
    const size_t total = static_cast<size_t>(B) * (H + 2) * (W + 2) * lanes;
    for (size_t idx = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; idx < total; idx += static_cast<size_t>(gridDim.x) * blockDim.x) {
        const int lane = static_cast<int>(idx % lanes);
        const size_t pix = idx / lanes;
        const int px = static_cast<int>(pix % (W + 2));
        const int py = static_cast<int>((pix / (W + 2)) % (H + 2));
        const int b = static_cast<int>(pix / (static_cast<size_t>(W + 2) * (H + 2)));
        const int y = min(max(py - 1, 0), H - 1), x = min(max(px - 1, 0), W - 1);
        const int c0 = lane * 8;
        const float2 ms = stats[static_cast<size_t>(b) * G + c0 / cg];
        float f[8];
        unpack8(*reinterpret_cast<const uint4*>(src + px_off(b, y + 1, x + 1, Hp, Wp, C) + lane * 16), f, BF16);
#pragma unroll
        for (int e = 0; e < 8; ++e) f[e] = fmaxf((f[e] - ms.x) * ms.y * gamma[c0 + e] + beta[c0 + e], 0.f);
        *reinterpret_cast<uint4*>(dst + px_off(b, py, px, Hp, Wp, C) + lane * 16) = pack8<BF16>(f);
    }
}

int launch_gn_stats(const void* map, const Level& g, int B, int C, int G, double2* partials, float2* stats, bool bf16, cudaStream_t st) {
    if (C % 8 || C > 2048 || G <= 0 || C % G || (C / G) % 8) return set_error("group_norm: C=%d with %d groups unsupported", C, G);
    const int tiles = gn_tiles(g.H, g.W, C), tile_px = gn_tile_px(C);
    const dim3 grid(tiles, B);
    if (bf16) CUDA_TRY(launch_pdl(gn_partial_kernel<true>, grid, dim3(256), 0, st, static_cast<const uint8_t*>(map), g.Hp, g.Wp, g.H, g.W, C, G, tiles, tile_px, partials));
    else CUDA_TRY(launch_pdl(gn_partial_kernel<false>, grid, dim3(256), 0, st, static_cast<const uint8_t*>(map), g.Hp, g.Wp, g.H, g.W, C, G, tiles, tile_px, partials));
    const double inv_n = 1.0 / (static_cast<double>(g.H) * g.W * (C / G));
    CUDA_TRY(launch_pdl(gn_finalize_kernel, dim3(G, B), dim3(256), 0, st, static_cast<const double2*>(partials), tiles, G, inv_n, stats));
    return 0;
}
int launch_gn_relu(const void* src, void* dst, const Level& g, int B, int C, int G, const float2* stats, const float* gamma, const float* beta, bool bf16,
                   cudaStream_t st) {
    const size_t total = static_cast<size_t>(B) * (g.H + 2) * (g.W + 2) * (C / 8);
    const auto s = static_cast<const uint8_t*>(src);
    const auto d = static_cast<uint8_t*>(dst);
    if (bf16) CUDA_TRY(launch_pdl(gn_relu_kernel<true>, dim3(grid_for(total)), dim3(256), 0, st, s, d, B, g.Hp, g.Wp, g.H, g.W, C, G, stats, gamma, beta));
    else CUDA_TRY(launch_pdl(gn_relu_kernel<false>, dim3(grid_for(total)), dim3(256), 0, st, s, d, B, g.Hp, g.Wp, g.H, g.W, C, G, stats, gamma, beta));
    return 0;
}

// ------------------------------------------------------------------------------------------ V5 ConvTranspose UV term
// ConvTranspose2d(C_in + 2 -> C, k2 s2) over cat(x, uv) (v1.py:123-129): the UV channels add, at output pixel (2i+di, 2j+dj),
// Wu[co,di,dj] u(j) + Wv[co,di,dj] v(i) with u, v on the INPUT grid.  Added in place to the convT output map (H x W = twice the
// input grid), border included.  wuv: [2][4 phases][C] fp32.
template <bool BF16>
__global__ void uv_convT_kernel(uint8_t* __restrict__ map, int B, int Hp, int Wp, int H, int W, int C, const float* __restrict__ wuv, float su, float sv) {
    pdl_prologue();
    const int lanes = C / 8;
    const float inv_w = 2.f / W, inv_h = 2.f / H;      // input grid: W/2 x H/2
    const size_t total = static_cast<size_t>(B) * (H + 2) * (W + 2) * lanes;
    for (size_t idx = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; idx < total; idx += static_cast<size_t>(gridDim.x) * blockDim.x) {
        const int lane = static_cast<int>(idx % lanes);
        const size_t pix = idx / lanes;
        const int px = static_cast<int>(pix % (W + 2));
        const int py = static_cast<int>((pix / (W + 2)) % (H + 2));
        const int b = static_cast<int>(pix / (static_cast<size_t>(W + 2) * (H + 2)));
        const int y = min(max(py - 1, 0), H - 1), x = min(max(px - 1, 0), W - 1);
        const int ph = (y & 1) * 2 + (x & 1);
        const float u = su * ((2 * (x >> 1) + 1) * inv_w - 1.f), v = sv * ((2 * (y >> 1) + 1) * inv_h - 1.f);
        uint4* p = reinterpret_cast<uint4*>(map + px_off(b, py, px, Hp, Wp, C) + lane * 16);
        float f[8];
        unpack8(*p, f, BF16);
        const int c0 = lane * 8;
#pragma unroll
        for (int e = 0; e < 8; ++e) f[e] += wuv[ph * C + c0 + e] * u + wuv[(4 + ph) * C + c0 + e] * v;
        *p = pack8<BF16>(f);
    }
}
// wuv[k][ph][co] = w[Cin + k][co][ph] of the ConvTranspose2d weight (Cin + 2, Cout, 2, 2), ph = di * 2 + dj
__global__ void pack_convT_uv_kernel(const float* __restrict__ w, int Cin, int Cout, float* __restrict__ wuv) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= 8 * Cout) return;
    const int co = i % Cout, ph = (i / Cout) % 4, k = i / (4 * Cout);
    wuv[i] = w[(static_cast<size_t>(Cin + k) * Cout + co) * 4 + ph];
}
int launch_pack_convT_uv(const float* w, int Cin, int Cout, float* wuv, cudaStream_t st) {
    pack_convT_uv_kernel<<<(8 * Cout + 255) / 256, 256, 0, st>>>(w, Cin, Cout, wuv);
    CUDA_TRY(cudaGetLastError());
    return 0;
}
int launch_uv_convT(void* map, const Level& g, int B, int C, const float* wuv, float su, float sv, bool bf16, cudaStream_t st) {
    const size_t total = static_cast<size_t>(B) * (g.H + 2) * (g.W + 2) * (C / 8);
    const auto m = static_cast<uint8_t*>(map);
    if (bf16) CUDA_TRY(launch_pdl(uv_convT_kernel<true>, dim3(grid_for(total)), dim3(256), 0, st, m, B, g.Hp, g.Wp, g.H, g.W, C, wuv, su, sv));
    else CUDA_TRY(launch_pdl(uv_convT_kernel<false>, dim3(grid_for(total)), dim3(256), 0, st, m, B, g.Hp, g.Wp, g.H, g.W, C, wuv, su, sv));
    return 0;
}

// ------------------------------------------------------------------------------------------ V7 bilinear resize of the decoder map
// F.interpolate(bilinear, align_corners=False, antialias=False) (v1.py:132) from the last decoder level to the resized-image grid,
// padded NHWC -> padded NHWC, border included.
template <bool BF16>
__global__ void resize_bilinear_nhwc_kernel(const uint8_t* __restrict__ src, int Hps, int Wps, int Hs, int Ws, uint8_t* __restrict__ dst, int Hpd,
                                            int Wpd, int Hd, int Wd, int C, int B) {
    pdl_prologue();
    const int lanes = C / 8;
    const float ry = static_cast<float>(Hs) / Hd, rx = static_cast<float>(Ws) / Wd;
    const size_t total = static_cast<size_t>(B) * (Hd + 2) * (Wd + 2) * lanes;
    for (size_t idx = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; idx < total; idx += static_cast<size_t>(gridDim.x) * blockDim.x) {
        const int lane = static_cast<int>(idx % lanes);
        const size_t pix = idx / lanes;
        const int px = static_cast<int>(pix % (Wd + 2));
        const int py = static_cast<int>((pix / (Wd + 2)) % (Hd + 2));
        const int b = static_cast<int>(pix / (static_cast<size_t>(Wd + 2) * (Hd + 2)));
        const int Y = min(max(py - 1, 0), Hd - 1), X = min(max(px - 1, 0), Wd - 1);
        const float sy = fmaxf(ry * (Y + 0.5f) - 0.5f, 0.f), sx = fmaxf(rx * (X + 0.5f) - 0.5f, 0.f);
        const int y0 = min(static_cast<int>(sy), Hs - 1), x0 = min(static_cast<int>(sx), Ws - 1);
        const int y1 = min(y0 + 1, Hs - 1), x1 = min(x0 + 1, Ws - 1);
        const float ly = sy - y0, lx = sx - x0;
        float a[8], bq[8], c[8], d[8];
        unpack8(*reinterpret_cast<const uint4*>(src + px_off(b, y0 + 1, x0 + 1, Hps, Wps, C) + lane * 16), a, BF16);
        unpack8(*reinterpret_cast<const uint4*>(src + px_off(b, y0 + 1, x1 + 1, Hps, Wps, C) + lane * 16), bq, BF16);
        unpack8(*reinterpret_cast<const uint4*>(src + px_off(b, y1 + 1, x0 + 1, Hps, Wps, C) + lane * 16), c, BF16);
        unpack8(*reinterpret_cast<const uint4*>(src + px_off(b, y1 + 1, x1 + 1, Hps, Wps, C) + lane * 16), d, BF16);
        float f[8];
#pragma unroll
        for (int e = 0; e < 8; ++e) f[e] = (1.f - ly) * ((1.f - lx) * a[e] + lx * bq[e]) + ly * ((1.f - lx) * c[e] + lx * d[e]);
        *reinterpret_cast<uint4*>(dst + px_off(b, py, px, Hpd, Wpd, C) + lane * 16) = pack8<BF16>(f);
    }
}
int launch_resize_bilinear_nhwc(const void* src, const Level& gs, void* dst, const Level& gd, int B, int C, bool bf16, cudaStream_t st) {
    if (C % 8) return set_error("resize_bilinear_nhwc: C=%d must be a multiple of 8", C);
    const size_t total = static_cast<size_t>(B) * (gd.H + 2) * (gd.W + 2) * (C / 8);
    const auto s = static_cast<const uint8_t*>(src);
    const auto d = static_cast<uint8_t*>(dst);
    if (bf16) CUDA_TRY(launch_pdl(resize_bilinear_nhwc_kernel<true>, dim3(grid_for(total)), dim3(256), 0, st, s, gs.Hp, gs.Wp, gs.H, gs.W, d, gd.Hp, gd.Wp, gd.H, gd.W, C, B));
    else CUDA_TRY(launch_pdl(resize_bilinear_nhwc_kernel<false>, dim3(grid_for(total)), dim3(256), 0, st, s, gs.Hp, gs.Wp, gs.H, gs.W, d, gd.Hp, gd.Wp, gd.H, gd.W, C, B));
    return 0;
}

// ------------------------------------------------------------------------------------------ V7 output block tail
// Both output blocks (v1.py:103-109, 137-138) after their 3x3 conv over the 64 feature channels (one conv, N = 32 points + 32 mask
// channels): + the UV part of that conv, + ReLU, then the two 1x1 convs as one block-diagonal 64 -> 4 map.  The UV part of a 3x3
// replicate-padded conv is exact as six folded weights per channel: sum_dx (sum_dy Wu[dy,dx]) u(clamp(x+dx)) + the same for v.
// wf: [64][6] folded UV weights (u at x-1, x, x+1; v at y-1, y, y+1), [4][64] 1x1 weights, [4] biases.
constexpr int V1_OUT_PARAMS = 64 * 6 + 4 * 64 + 4;
template <bool BF16>
__global__ void __launch_bounds__(256) v1_output_kernel(const uint8_t* __restrict__ map, int B, int Hp, int Wp, int H, int W, const float* __restrict__ wf,
                                                        float su, float sv, float4* __restrict__ pts, float* __restrict__ msk) {
    pdl_prologue();
    __shared__ float s[V1_OUT_PARAMS];
    for (int i = threadIdx.x; i < V1_OUT_PARAMS; i += blockDim.x) s[i] = wf[i];
    __syncthreads();
    const float* wuv = s;
    const float* wp = s + 64 * 6;
    const float* bias = wp + 4 * 64;
    const size_t total = static_cast<size_t>(B) * H * W;
    for (size_t idx = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; idx < total; idx += static_cast<size_t>(gridDim.x) * blockDim.x) {
        const int x = static_cast<int>(idx % W);
        const int y = static_cast<int>((idx / W) % H);
        const int b = static_cast<int>(idx / (static_cast<size_t>(W) * H));
        auto uu = [&](int X) { return su * ((2 * X + 1) / static_cast<float>(W) - 1.f); };
        auto vv = [&](int Y) { return sv * ((2 * Y + 1) / static_cast<float>(H) - 1.f); };
        const float t[6] = {uu(max(x - 1, 0)), uu(x), uu(min(x + 1, W - 1)), vv(max(y - 1, 0)), vv(y), vv(min(y + 1, H - 1))};
        float o[4] = {bias[0], bias[1], bias[2], bias[3]};
        const uint4* p = reinterpret_cast<const uint4*>(map + px_off(b, y + 1, x + 1, Hp, Wp, 64));
#pragma unroll 1
        for (int q = 0; q < 8; ++q) {
            float f[8];
            unpack8(p[q], f, BF16);
#pragma unroll
            for (int e = 0; e < 8; ++e) {
                const int c = q * 8 + e;
                float h = f[e];
#pragma unroll
                for (int k = 0; k < 6; ++k) h += wuv[c * 6 + k] * t[k];
                h = fmaxf(h, 0.f);
#pragma unroll
                for (int k = 0; k < 4; ++k) o[k] += wp[k * 64 + c] * h;
            }
        }
        pts[idx] = make_float4(o[0], o[1], o[2], 0.f);
        msk[idx] = o[3];
    }
}
int launch_v1_output(const void* map, const Level& g, int B, const float* wf, float su, float sv, float4* pts, float* msk, bool bf16, cudaStream_t st) {
    const size_t total = static_cast<size_t>(B) * g.H * g.W;
    const auto m = static_cast<const uint8_t*>(map);
    if (bf16) CUDA_TRY(launch_pdl(v1_output_kernel<true>, dim3(grid_for(total)), dim3(256), 0, st, m, B, g.Hp, g.Wp, g.H, g.W, wf, su, sv, pts, msk));
    else CUDA_TRY(launch_pdl(v1_output_kernel<false>, dim3(grid_for(total)), dim3(256), 0, st, m, B, g.Hp, g.Wp, g.H, g.W, wf, su, sv, pts, msk));
    return 0;
}

// ------------------------------------------------------------------------------------------ V9 post-processing
// v1.py:356-380: mask = raw mask > mask_threshold; intrinsics; depth = z + shift; re-projection (force_projection) or
// points += (0, 0, shift); masking sets points and depth to +inf.  No `depth > 0` term and no metric scale (unlike v2).
__global__ void v1_threshold_kernel(const float* __restrict__ mask, float thr, size_t n, uint8_t* __restrict__ out) {
    pdl_prologue();
    for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < n; i += static_cast<size_t>(gridDim.x) * blockDim.x)
        out[i] = mask[i] > thr ? 1 : 0;
}
__global__ void v1_post_kernel(float* __restrict__ points, const uint8_t* __restrict__ mask, const float* __restrict__ focal,
                               const float* __restrict__ shift, int H, int W, int force_projection, int apply_mask, float* __restrict__ depth,
                               float* __restrict__ intrinsics) {
    pdl_prologue();
    const int b = blockIdx.y;
    const float aspect = static_cast<float>(W) / H;
    const float diag = sqrtf(1.f + aspect * aspect);
    const float f = focal[b];
    const float fx = f / 2.f * diag / aspect, fy = f / 2.f * diag;
    const float sft = shift[b];
    if (blockIdx.x == 0 && threadIdx.x < 9) {
        const float K[9] = {fx, 0.f, 0.5f, 0.f, fy, 0.5f, 0.f, 0.f, 1.f};
        intrinsics[b * 9 + threadIdx.x] = K[threadIdx.x];
    }
    const size_t npix = static_cast<size_t>(H) * W;
    for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < npix; i += static_cast<size_t>(gridDim.x) * blockDim.x) {
        const size_t pix = static_cast<size_t>(b) * npix + i;
        const int X = static_cast<int>(i % W), Y = static_cast<int>(i / W);
        float px = points[pix * 3], py = points[pix * 3 + 1];
        float z = points[pix * 3 + 2] + sft;
        if (force_projection) {
            px = ((X + 0.5f) / W - 0.5f) / fx * z;
            py = ((Y + 0.5f) / H - 0.5f) / fy * z;
        }
        if (apply_mask && !mask[pix]) px = py = z = INFINITY;
        points[pix * 3] = px; points[pix * 3 + 1] = py; points[pix * 3 + 2] = z;
        depth[pix] = z;
    }
}
int launch_v1_postprocess(float* points, const float* mask, float mask_threshold, const float* focal_in, int B, int H, int W, int force_projection,
                          int apply_mask, float* depth, uint8_t* mask_out, float* intrinsics, float* focal, float* shift, cudaStream_t st) {
    const size_t n = static_cast<size_t>(B) * H * W;
    CUDA_TRY(launch_pdl(v1_threshold_kernel, dim3(grid_for(n)), dim3(256), 0, st, mask, mask_threshold, n, mask_out));
    MG_TRY(launch_focal_shift(points, nullptr, mask_out, B, H, W, focal_in, focal, shift, st));
    const size_t npix = static_cast<size_t>(H) * W;
    const dim3 grid(static_cast<unsigned>(std::min<size_t>((npix + 255) / 256, 132 * 8)), B);
    CUDA_TRY(launch_pdl(v1_post_kernel, grid, dim3(256), 0, st, points, static_cast<const uint8_t*>(mask_out), static_cast<const float*>(focal),
                        static_cast<const float*>(shift), H, W, force_projection, apply_mask, depth, intrinsics));
    return 0;
}

}  // namespace mg
