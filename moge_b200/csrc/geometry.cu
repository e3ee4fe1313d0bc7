// Geometry utilities (moge/utils/geometry_torch.py of the reference): refine_depth_with_normal, dilate_with_mask,
// theshold_depth_change and gaussian_blur_2d.  Python: moge_b200.geometry; fp64 restatements and error bounds:
// oracle/geometry_port.py.  Every map is fp32 (batch, H, W) contiguous, masks uint8 (nonzero = in).  No atomics: each output
// element is written by one thread from a fixed sequence of operations, so every run gives the same bits.
//
// refine_depth_with_normal: a log kernel clamps the depth in place (the reference's depth.clamp_min_(eps)) and writes its log; a
// set-up kernel forms, per interior pixel, the normal-driven Laplacian term (grad in fp64 from the per-image inverse
// intrinsics, weights from the log-depth tile) and stores damp * log d - clamp(lap, -0.1, 0.1); then one Jacobi sweep kernel per
// iteration ping-pongs two log-depth buffers, and the last sweep writes exp() of every pixel.  The bilateral weights depend on
// the INPUT log-depth only, so the sweeps recompute them from its tile in shared memory rather than streaming a (k x k) weight
// buffer: 25 expf per pixel cost less than 100 bytes of traffic per pixel per sweep (DESIGN.md §1).  The radius-wide border
// keeps the input log-depth: a sweep reads the border of its source buffer from the log-depth map, so the buffers need no copy.
#include "host_api.h"
#include "../../include/moge_b200.h"
#include <math.h>
#include <stdint.h>

namespace mg {
namespace {

constexpr int kThreads = 256;
constexpr int kT = 32;                            // output tile: kT x kT pixels
constexpr int kMaxPoolR = (MOGE_GEOMETRY_MAX_POOL_KERNEL - 1) / 2;
constexpr int kMaxBlurR = (MOGE_GEOMETRY_MAX_BLUR_KERNEL - 1) / 2;
constexpr int64_t kMaxPixels = int64_t(1) << 30;

__device__ __forceinline__ bool interior(int i, int j, int H, int W, int r) { return i >= r && i < H - r && j >= r && j < W - r; }

// ---------------------------------------------------------------------------------------------------- refine_depth_with_normal
// Per-tap constants of a (2R + 1)^2 window in row-major tap order (tap (a, b) = offset (a - R, b - R)):
// c = 1 / (10 max(|duv|, eps)), hx / hy = duv / 2 with duv = ((b - R) / W, (a - R) / H).
struct Taps {
    float c[MOGE_GEOMETRY_MAX_REFINE_KERNEL * MOGE_GEOMETRY_MAX_REFINE_KERNEL];
    double hx[MOGE_GEOMETRY_MAX_REFINE_KERNEL * MOGE_GEOMETRY_MAX_REFINE_KERNEL];
    double hy[MOGE_GEOMETRY_MAX_REFINE_KERNEL * MOGE_GEOMETRY_MAX_REFINE_KERNEL];
};

// bilateral weight of a tap: exp(-((ld_n - ld_c) c)^2)
__device__ __forceinline__ float tap_weight(float ln, float lc, float c) {
    const float t = __fmul_rn(__fsub_rn(ln, lc), c);
    return expf(-__fmul_rn(t, t));
}

__global__ void __launch_bounds__(kThreads) log_kernel(float* __restrict__ depth, int64_t n, float eps, float* __restrict__ ld) {
    const int64_t p = static_cast<int64_t>(blockIdx.x) * kThreads + threadIdx.x;
    if (p >= n) return;
    float d = depth[p];
    if (d < eps) {                                 // clamp_min_: NaN stays NaN
        d = eps;
        depth[p] = d;
    }
    ld[p] = logf(d);
}

__global__ void __launch_bounds__(kThreads) exp_kernel(const float* __restrict__ ld, int64_t n, float* __restrict__ out) {
    const int64_t p = static_cast<int64_t>(blockIdx.x) * kThreads + threadIdx.x;
    if (p < n) out[p] = expf(ld[p]);
}

// grid (tiles x, tiles y, images).  cterm[p] = damp * ld[p] - clamp(lap, -0.1, 0.1) at interior pixels, with
// lap = sum over taps of w * ((g_n + g_c) . duv / 2) and g = -(n_xy K2) / (n_z + n_xy . (K2 uv + k)), K2 and k the upper 2 x 2
// block and the upper half of the last column of inv(intrinsics), uv = ((j + 0.5) / W, (i + 0.5) / H).
template <int R>
__global__ void __launch_bounds__(kThreads) setup_kernel(const float* __restrict__ ld, const float* __restrict__ normal,
                                                         const float* __restrict__ intrinsics, int H, int W, float damp, const Taps taps,
                                                         float* __restrict__ cterm) {
    constexpr int S = kT + 2 * R, K = 2 * R + 1;
    __shared__ float s_ld[S][S];
    __shared__ double2 s_g[S][S];
    __shared__ double s_k[6];
    const int64_t b = blockIdx.z, hw = static_cast<int64_t>(H) * W;
    const int i0 = blockIdx.y * kT, j0 = blockIdx.x * kT;
    if (threadIdx.x == 0) {                        // inverse of the 3 x 3 intrinsics by cofactors, in fp64
        const float* k = intrinsics + b * 9;
        const double a = k[0], bb = k[1], c = k[2], d = k[3], e = k[4], f = k[5], g = k[6], h = k[7], i = k[8];
        const double A = e * i - f * h, B = -(d * i - f * g), D = -(bb * i - c * h), E = a * i - c * g, G = bb * f - c * e,
                     Hh = -(a * f - c * d);
        const double det = a * A + bb * B + c * (d * h - e * g);
        s_k[0] = A / det; s_k[1] = D / det; s_k[2] = G / det;       // row 0 of the inverse
        s_k[3] = B / det; s_k[4] = E / det; s_k[5] = Hh / det;      // row 1
    }
    __syncthreads();
    const double k00 = s_k[0], k01 = s_k[1], k02 = s_k[2], k10 = s_k[3], k11 = s_k[4], k12 = s_k[5];
    for (int q = threadIdx.x; q < S * S; q += kThreads) {
        const int li = q / S, lj = q % S, i = i0 - R + li, j = j0 - R + lj;
        float l = 0.f;
        double2 g = make_double2(0.0, 0.0);
        if (i >= 0 && i < H && j >= 0 && j < W) {
            const int64_t p = b * hw + static_cast<int64_t>(i) * W + j;
            l = ld[p];
            const double nx = normal[p * 3], ny = normal[p * 3 + 1], nz = normal[p * 3 + 2];
            const double u = (j + 0.5) / W, v = (i + 0.5) / H;
            const double den = nz + nx * (k00 * u + k01 * v + k02) + ny * (k10 * u + k11 * v + k12);
            g = make_double2(-(nx * k00 + ny * k10) / den, -(nx * k01 + ny * k11) / den);
        }
        s_ld[li][lj] = l;
        s_g[li][lj] = g;
    }
    __syncthreads();
    const double clampv = static_cast<double>(0.1f);
    for (int q = threadIdx.x; q < kT * kT; q += kThreads) {
        const int oi = q / kT, oj = q % kT, i = i0 + oi, j = j0 + oj;
        if (i >= H || j >= W || !interior(i, j, H, W, R)) continue;
        const float lc = s_ld[oi + R][oj + R];
        const double2 gc = s_g[oi + R][oj + R];
        double lap = 0.0;
#pragma unroll 1
        for (int a = 0; a < K; ++a)
#pragma unroll
            for (int bb = 0; bb < K; ++bb) {
                const int t = a * K + bb;
                const float w = tap_weight(s_ld[oi + a][oj + bb], lc, taps.c[t]);
                const double2 gn = s_g[oi + a][oj + bb];
                lap += static_cast<double>(w) * ((gn.x + gc.x) * taps.hx[t] + (gn.y + gc.y) * taps.hy[t]);
            }
        lap = lap < -clampv ? -clampv : (lap > clampv ? clampv : lap);       // torch.clamp: NaN stays NaN
        cterm[b * hw + static_cast<int64_t>(i) * W + j] = __fsub_rn(__fmul_rn(damp, lc), static_cast<float>(lap));
    }
}

// grid (tiles x, tiles y, images): one Jacobi sweep
//   y = 0.1 x_c + 0.9 (cterm + sum_taps w x_n) / (sum_taps w + damp)
// at interior pixels, x = src at interior pixels and ld on the border.  The last sweep (out != null) writes exp(y) at interior
// pixels and exp(ld) on the border of the depth map `out` instead of y to dst.
template <int R>
__global__ void __launch_bounds__(kThreads) sweep_kernel(const float* __restrict__ ld, const float* __restrict__ src,
                                                         const float* __restrict__ cterm, int H, int W, float damp, const Taps taps,
                                                         float* __restrict__ dst, float* __restrict__ out) {
    constexpr int S = kT + 2 * R, K = 2 * R + 1;
    __shared__ float s_ld[S][S], s_x[S][S];
    const int64_t b = blockIdx.z, hw = static_cast<int64_t>(H) * W;
    const int i0 = blockIdx.y * kT, j0 = blockIdx.x * kT;
    for (int q = threadIdx.x; q < S * S; q += kThreads) {
        const int li = q / S, lj = q % S, i = i0 - R + li, j = j0 - R + lj;
        float l = 0.f, x = 0.f;
        if (i >= 0 && i < H && j >= 0 && j < W) {
            const int64_t p = b * hw + static_cast<int64_t>(i) * W + j;
            l = ld[p];
            x = interior(i, j, H, W, R) ? src[p] : l;
        }
        s_ld[li][lj] = l;
        s_x[li][lj] = x;
    }
    __syncthreads();
    for (int q = threadIdx.x; q < kT * kT; q += kThreads) {
        const int oi = q / kT, oj = q % kT, i = i0 + oi, j = j0 + oj;
        if (i >= H || j >= W) continue;
        const int64_t p = b * hw + static_cast<int64_t>(i) * W + j;
        if (!interior(i, j, H, W, R)) {
            if (out) out[p] = expf(s_ld[oi + R][oj + R]);
            continue;
        }
        const float lc = s_ld[oi + R][oj + R];
        float tot = 0.f, acc = 0.f;
#pragma unroll
        for (int a = 0; a < K; ++a)
#pragma unroll
            for (int bb = 0; bb < K; ++bb) {
                const float w = tap_weight(s_ld[oi + a][oj + bb], lc, taps.c[a * K + bb]);
                tot = __fadd_rn(tot, w);
                acc = __fadd_rn(acc, __fmul_rn(w, s_x[oi + a][oj + bb]));
            }
        const float q2 = __fdiv_rn(__fadd_rn(cterm[p], acc), __fadd_rn(tot, damp));
        const float y = __fadd_rn(__fmul_rn(0.1f, s_x[oi + R][oj + R]), __fmul_rn(0.9f, q2));
        if (out) out[p] = expf(y);
        else dst[p] = y;
    }
}

template <int R>
int launch_refine(float* ld, const float* normal, const float* intrinsics, int64_t batch, int H, int W, int iterations, float damp,
                  const Taps& taps, float* cterm, float* buf0, float* buf1, float* out, cudaStream_t st) {
    const dim3 grid((W + kT - 1) / kT, (H + kT - 1) / kT, static_cast<unsigned>(batch));
    setup_kernel<R><<<grid, kThreads, 0, st>>>(ld, normal, intrinsics, H, W, damp, taps, cterm);
    CUDA_TRY(cudaGetLastError());
    const float* src = ld;
    float* bufs[2] = {buf0, buf1};
    for (int it = 0; it < iterations; ++it) {
        const bool last = it + 1 == iterations;
        float* dst = bufs[it & 1];
        sweep_kernel<R><<<grid, kThreads, 0, st>>>(ld, src, cterm, H, W, damp, taps, last ? nullptr : dst, last ? out : nullptr);
        CUDA_TRY(cudaGetLastError());
        src = dst;
    }
    return 0;
}

// ---------------------------------------------------------------------------------------------------- dilate_with_mask
// grid (pixel blocks, images).  Valid pixels keep their value; an invalid pixel takes the filter of the valid pixels among its
// up, left, right and down neighbours (outside the map: invalid), and becomes valid when there is one.  With none: mean and
// median give NaN, min +inf, max -inf, as the reference's fill values do.  min / max propagate NaN (torch.min / max); mean and
// median skip NaN values (nanmean / nanmedian), median taking the lower middle of an even count.
__global__ void __launch_bounds__(kThreads) dilate_kernel(const float* __restrict__ in, const uint8_t* __restrict__ mask, int H, int W,
                                                          int filter, float* __restrict__ out, uint8_t* __restrict__ mask_out) {
    const int64_t hw = static_cast<int64_t>(H) * W, p = static_cast<int64_t>(blockIdx.x) * kThreads + threadIdx.x;
    if (p >= hw) return;
    const int64_t e = static_cast<int64_t>(blockIdx.y) * hw + p;
    if (mask[e]) {
        out[e] = in[e];
        mask_out[e] = 1;
        return;
    }
    const int i = static_cast<int>(p / W), j = static_cast<int>(p % W);
    float v[4];
    int n = 0;
    bool any = false;
    const int64_t nb[4] = {e - W, e - 1, e + 1, e + W};                   // the cross in the window's row-major order
    const bool inside[4] = {i > 0, j > 0, j + 1 < W, i + 1 < H};
    float r;
    if (filter == MOGE_DILATE_MIN || filter == MOGE_DILATE_MAX) {
        const bool mx = filter == MOGE_DILATE_MAX;
        r = mx ? -INFINITY : INFINITY;
        for (int k = 0; k < 4; ++k) {
            if (!inside[k] || !mask[nb[k]]) continue;
            any = true;
            const float x = in[nb[k]];
            if (isnan(x) || (mx ? x > r : x < r)) r = isnan(r) ? r : x;
        }
    } else {
        for (int k = 0; k < 4; ++k) {
            if (!inside[k] || !mask[nb[k]]) continue;
            any = true;
            const float x = in[nb[k]];
            if (!isnan(x)) v[n++] = x;
        }
        if (filter == MOGE_DILATE_MEAN) {
            float s = 0.f;
            for (int k = 0; k < n; ++k) s = __fadd_rn(s, v[k]);
            r = n ? __fdiv_rn(s, static_cast<float>(n)) : NAN;
        } else {
            for (int a = 1; a < n; ++a)                                   // insertion sort of at most 4 values
                for (int k = a; k > 0 && v[k - 1] > v[k]; --k) { const float t = v[k]; v[k] = v[k - 1]; v[k - 1] = t; }
            r = n ? v[(n - 1) / 2] : NAN;
        }
    }
    out[e] = r;
    mask_out[e] = any;
}

// ---------------------------------------------------------------------------------------------------- theshold_depth_change
// grid (tiles x, tiles y, images).  A separable max pool over the (2r + 1)^2 window of s = d (max) or -d (min) at masked-in
// pixels, -inf elsewhere and outside the map, NaN propagating (max_pool2d); then out = pooled > d * factor (max) or -pooled < d *
// factor (min), each product rounded once in fp32.
__device__ __forceinline__ float pool_max(float a, float b) { return (b > a || isnan(b)) ? b : a; }

__global__ void __launch_bounds__(kThreads) pool_kernel(const float* __restrict__ depth, const uint8_t* __restrict__ mask, int H, int W, int r,
                                                        int pool_max_mode, float factor, uint8_t* __restrict__ out) {
    constexpr int S = kT + 2 * kMaxPoolR;
    __shared__ float s_v[S][S], s_h[S][kT];
    const int64_t b = blockIdx.z, hw = static_cast<int64_t>(H) * W;
    const int i0 = blockIdx.y * kT, j0 = blockIdx.x * kT, Sr = kT + 2 * r;
    for (int q = threadIdx.x; q < Sr * Sr; q += kThreads) {
        const int li = q / Sr, lj = q % Sr, i = i0 - r + li, j = j0 - r + lj;
        float x = -INFINITY;
        if (i >= 0 && i < H && j >= 0 && j < W) {
            const int64_t p = b * hw + static_cast<int64_t>(i) * W + j;
            if (mask[p]) x = pool_max_mode ? depth[p] : -depth[p];
        }
        s_v[li][lj] = x;
    }
    __syncthreads();
    for (int q = threadIdx.x; q < Sr * kT; q += kThreads) {
        const int li = q / kT, oj = q % kT;
        float m = s_v[li][oj];
        for (int t = 1; t <= 2 * r; ++t) m = pool_max(m, s_v[li][oj + t]);
        s_h[li][oj] = m;
    }
    __syncthreads();
    for (int q = threadIdx.x; q < kT * kT; q += kThreads) {
        const int oi = q / kT, oj = q % kT, i = i0 + oi, j = j0 + oj;
        if (i >= H || j >= W) continue;
        float m = s_h[oi][oj];
        for (int t = 1; t <= 2 * r; ++t) m = pool_max(m, s_h[oi + t][oj]);
        const int64_t p = b * hw + static_cast<int64_t>(i) * W + j;
        const float lim = __fmul_rn(depth[p], factor);
        out[p] = pool_max_mode ? (m > lim) : (-m < lim);
    }
}

// ---------------------------------------------------------------------------------------------------- gaussian_blur_2d
// grid (tiles x, tiles y, planes): out = sum over the k x k taps (row-major) of (k1[a] * k1[b]) * x, x the input clamped to the
// map (replicate padding), the tap weight rounded once as the reference's outer product is.
struct Blur1d { float k[MOGE_GEOMETRY_MAX_BLUR_KERNEL]; };

__global__ void __launch_bounds__(kThreads) blur_kernel(const float* __restrict__ in, int H, int W, int r, const Blur1d k1,
                                                        float* __restrict__ out) {
    constexpr int S = kT + 2 * kMaxBlurR;
    __shared__ float s_x[S][S], s_k[MOGE_GEOMETRY_MAX_BLUR_KERNEL];
    const int64_t b = blockIdx.z, hw = static_cast<int64_t>(H) * W;
    const int i0 = blockIdx.y * kT, j0 = blockIdx.x * kT, Sr = kT + 2 * r, K = 2 * r + 1;
    if (threadIdx.x < MOGE_GEOMETRY_MAX_BLUR_KERNEL) s_k[threadIdx.x] = k1.k[threadIdx.x];
    for (int q = threadIdx.x; q < Sr * Sr; q += kThreads) {
        const int li = q / Sr, lj = q % Sr;
        const int i = min(max(i0 - r + li, 0), H - 1), j = min(max(j0 - r + lj, 0), W - 1);
        s_x[li][lj] = in[b * hw + static_cast<int64_t>(i) * W + j];
    }
    __syncthreads();
    for (int q = threadIdx.x; q < kT * kT; q += kThreads) {
        const int oi = q / kT, oj = q % kT, i = i0 + oi, j = j0 + oj;
        if (i >= H || j >= W) continue;
        float acc = 0.f;
        for (int a = 0; a < K; ++a) {
            const float ka = s_k[a];
            for (int bb = 0; bb < K; ++bb) acc = __fadd_rn(acc, __fmul_rn(__fmul_rn(ka, s_k[bb]), s_x[oi + a][oj + bb]));
        }
        out[b * hw + static_cast<int64_t>(i) * W + j] = acc;
    }
}

dim3 tile_grid(int64_t batch, int H, int W) { return dim3((W + kT - 1) / kT, (H + kT - 1) / kT, static_cast<unsigned>(batch)); }

int check_rows(const char* what, int H) {
    if ((H + kT - 1) / kT > 65535) return set_error("%s: %d rows is more than %d", what, H, 65535 * kT);
    return 0;
}

struct RefineLayout { size_t ld, cterm, buf0, buf1, total; };
RefineLayout refine_layout(int64_t batch, int H, int W) {
    const size_t n = static_cast<size_t>(batch) * H * W * sizeof(float);
    WsLayout ws;
    RefineLayout l;
    l.ld = ws.add(n);
    l.cterm = ws.add(n);
    l.buf0 = ws.add(n);
    l.buf1 = ws.add(n);
    l.total = ws.total;
    return l;
}

}  // namespace
}  // namespace mg

using namespace mg;

extern "C" {

int moge_geometry_workspace_bytes(int64_t batch, int H, int W, size_t* bytes) {
    if (!bytes) return set_error("null argument");
    MG_TRY(check_batch_map("refine_depth_with_normal", batch, H, W, kMaxPixels));
    *bytes = refine_layout(batch, H, W).total;
    return 0;
}

int moge_refine_depth_with_normal(float* depth, const float* normal, const float* intrinsics, int64_t batch, int H, int W,
                                  int iterations, float damp, float eps, int kernel_size, float* out, void* workspace,
                                  size_t workspace_bytes, void* stream) {
    if (!depth || !normal || !intrinsics || !out) return set_error("null argument");
    MG_TRY(check_batch_map("refine_depth_with_normal", batch, H, W, kMaxPixels));
    MG_TRY(check_rows("refine_depth_with_normal", H));
    if (kernel_size < 3 || kernel_size > MOGE_GEOMETRY_MAX_REFINE_KERNEL || kernel_size % 2 == 0)
        return set_error("refine_depth_with_normal: kernel_size %d is not an odd size from 3 to %d", kernel_size,
                         MOGE_GEOMETRY_MAX_REFINE_KERNEL);
    if (iterations < 0) return set_error("refine_depth_with_normal: iterations %d is negative", iterations);
    const RefineLayout l = refine_layout(batch, H, W);
    MG_TRY(check_workspace(l.total, workspace, workspace_bytes, "refine_depth_with_normal"));
    MG_TRY(check_device("refine_depth_with_normal"));
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    char* ws = static_cast<char*>(workspace);
    float* ld = reinterpret_cast<float*>(ws + l.ld);
    const int64_t n = batch * H * W;
    const unsigned blocks = static_cast<unsigned>((n + kThreads - 1) / kThreads);
    log_kernel<<<blocks, kThreads, 0, st>>>(depth, n, eps, ld);
    CUDA_TRY(cudaGetLastError());
    const int R = kernel_size / 2;
    if (iterations == 0 || H <= 2 * R || W <= 2 * R) {             // no sweep, or no interior pixel: exp(log(depth))
        exp_kernel<<<blocks, kThreads, 0, st>>>(ld, n, out);
        CUDA_TRY(cudaGetLastError());
        return 0;
    }
    Taps taps;
    const int K = kernel_size;
    for (int a = 0; a < K; ++a)
        for (int b = 0; b < K; ++b) {
            const double dx = static_cast<double>(b - R) / W, dy = static_cast<double>(a - R) / H;
            taps.c[a * K + b] = static_cast<float>(1.0 / (10.0 * fmax(sqrt(dx * dx + dy * dy), static_cast<double>(eps))));
            taps.hx[a * K + b] = dx / 2;
            taps.hy[a * K + b] = dy / 2;
        }
    float* cterm = reinterpret_cast<float*>(ws + l.cterm);
    float* b0 = reinterpret_cast<float*>(ws + l.buf0);
    float* b1 = reinterpret_cast<float*>(ws + l.buf1);
    switch (R) {
        case 1: return launch_refine<1>(ld, normal, intrinsics, batch, H, W, iterations, damp, taps, cterm, b0, b1, out, st);
        case 2: return launch_refine<2>(ld, normal, intrinsics, batch, H, W, iterations, damp, taps, cterm, b0, b1, out, st);
        case 3: return launch_refine<3>(ld, normal, intrinsics, batch, H, W, iterations, damp, taps, cterm, b0, b1, out, st);
        default: return launch_refine<4>(ld, normal, intrinsics, batch, H, W, iterations, damp, taps, cterm, b0, b1, out, st);
    }
}

int moge_dilate_with_mask(const float* input, const uint8_t* mask, int64_t batch, int H, int W, int filter, float* out,
                          uint8_t* mask_out, void* stream) {
    if (!input || !mask || !out || !mask_out) return set_error("null argument");
    MG_TRY(check_batch_map("dilate_with_mask", batch, H, W, kMaxPixels));
    if (filter < MOGE_DILATE_MEAN || filter > MOGE_DILATE_MEDIAN) return set_error("dilate_with_mask: unknown filter %d", filter);
    MG_TRY(check_device("dilate_with_mask"));
    const int64_t blocks = (static_cast<int64_t>(H) * W + kThreads - 1) / kThreads;
    dilate_kernel<<<dim3(static_cast<unsigned>(blocks), static_cast<unsigned>(batch)), kThreads, 0, static_cast<cudaStream_t>(stream)>>>(
        input, mask, H, W, filter, out, mask_out);
    CUDA_TRY(cudaGetLastError());
    return 0;
}

int moge_threshold_depth_change(const float* depth, const uint8_t* mask, int64_t batch, int H, int W, int pool_max, float factor,
                                int kernel_size, uint8_t* out, void* stream) {
    if (!depth || !mask || !out) return set_error("null argument");
    MG_TRY(check_batch_map("theshold_depth_change", batch, H, W, kMaxPixels));
    MG_TRY(check_rows("theshold_depth_change", H));
    if (kernel_size < 1 || kernel_size > MOGE_GEOMETRY_MAX_POOL_KERNEL || kernel_size % 2 == 0)
        return set_error("theshold_depth_change: kernel_size %d is not an odd size from 1 to %d", kernel_size, MOGE_GEOMETRY_MAX_POOL_KERNEL);
    MG_TRY(check_device("theshold_depth_change"));
    pool_kernel<<<tile_grid(batch, H, W), kThreads, 0, static_cast<cudaStream_t>(stream)>>>(depth, mask, H, W, kernel_size / 2, pool_max ? 1 : 0,
                                                                                          factor, out);
    CUDA_TRY(cudaGetLastError());
    return 0;
}

int moge_gaussian_blur_2d(const float* input, int64_t planes, int H, int W, const float* kernel1d, int kernel_size, float* out,
                          void* stream) {
    if (!input || !kernel1d || !out) return set_error("null argument");
    MG_TRY(check_batch_map("gaussian_blur_2d", planes, H, W, kMaxPixels));
    MG_TRY(check_rows("gaussian_blur_2d", H));
    if (kernel_size < 1 || kernel_size > MOGE_GEOMETRY_MAX_BLUR_KERNEL || kernel_size % 2 == 0)
        return set_error("gaussian_blur_2d: kernel_size %d is not an odd size from 1 to %d", kernel_size, MOGE_GEOMETRY_MAX_BLUR_KERNEL);
    MG_TRY(check_device("gaussian_blur_2d"));
    Blur1d k1 = {};
    for (int a = 0; a < kernel_size; ++a) k1.k[a] = kernel1d[a];
    blur_kernel<<<tile_grid(planes, H, W), kThreads, 0, static_cast<cudaStream_t>(stream)>>>(input, H, W, kernel_size / 2, k1, out);
    CUDA_TRY(cudaGetLastError());
    return 0;
}

}  // extern "C"
