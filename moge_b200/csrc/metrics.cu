// Evaluation metrics (moge/test/metrics.py of the reference): masked nearest resize + compaction, a statistics pass, one metric
// pass over every requested variant, and boundary-F1 counts.  Every image of a batch is independent of the others.
//
// Floating-point reductions give the same bits on every run and for any batch composition: the pixels of an image are cut into
// fixed tiles (set by H x W only), each CTA reduces its tile in fp64 in a fixed order and writes a partial, and a finalize kernel
// adds the partials of an image in tile order.  Only integer counters and order-independent min/max use atomics.  Per-pixel values
// are formed in the reference's fp32 arithmetic with explicit roundings (__fmul_rn / __fadd_rn / __fdiv_rn: nvcc would otherwise
// contract `p * s + b` into an FMA, which the reference never does).
#include "common.cuh"
#include "host_api.h"
#include "../../include/moge_b200.h"
#include <math.h>
#include <stdint.h>
#include <string.h>
#include <algorithm>

namespace mg {
namespace {

constexpr int kThreads = 256;
constexpr int kWarps = kThreads / 32;
constexpr int kTilePx = 8192;                 // pixels per reduction tile (32 per thread)
constexpr int64_t kMaxPixels = int64_t(1) << 29;
constexpr int kMaxSeg = MOGE_METRICS_MAX_SEGMENTS;
constexpr int kMaxVar = MOGE_METRICS_MAX_VARIANTS;
constexpr int kStatQ = 5;                     // sum x, sum y, sum x^2, sum xy, n
constexpr int kEvalQ = 2 * kMaxVar + 1;       // per variant (rel sum, delta1 count), then the mask count
constexpr int kResizeThreads = 1024;
constexpr int kBT = 32;                       // boundary tile: kBT x kBT centres, 3-pixel halo
constexpr int kHalo = 3;
constexpr int kBS = kBT + 2 * kHalo;

struct Variants { moge_metric_variant_t v[kMaxVar]; int n; };
struct Thresholds { float t[MOGE_METRICS_F1_THRESHOLDS]; };

__device__ __forceinline__ float norm3(float x, float y, float z) {
    return sqrtf(__fadd_rn(__fadd_rn(__fmul_rn(x, x), __fmul_rn(y, y)), __fmul_rn(z, z)));
}

// the aligned depth of a depth / disparity variant at pixel `pix` of image b (params: scale, shift, clamp, -)
__device__ __forceinline__ float aligned_depth(const moge_metric_variant_t& v, int64_t b, int64_t hw, int64_t pix) {
    const float x = v.src[b * hw + pix];
    if (v.kind == MOGE_MV_DEPTH) return x;
    const float* p = v.params + b * 4;
    if (v.kind == MOGE_MV_DEPTH_SCALE) return __fmul_rn(x, p[0]);
    if (v.kind == MOGE_MV_DEPTH_AFFINE) return __fadd_rn(__fmul_rn(x, p[0]), p[1]);
    const float d = v.kind == MOGE_MV_DISPARITY_FROM_DEPTH ? __fdiv_rn(1.f, x) : x;
    float a = __fadd_rn(__fmul_rn(d, p[0]), p[1]);
    if (a < p[2]) a = p[2];                   // clamp_min: NaN stays NaN
    return __fdiv_rn(1.f, a);
}

// the aligned point of a points variant (params: scale, shift x, y, z)
__device__ __forceinline__ void aligned_point(const moge_metric_variant_t& v, int64_t b, int64_t hw, int64_t pix, float* o) {
    const float* s = v.src + (b * hw + pix) * 3;
    const float* p = v.params + b * 4;
    for (int c = 0; c < 3; ++c) {
        if (v.kind == MOGE_MV_POINTS_SHIFT) o[c] = __fadd_rn(s[c], p[1 + c]);
        else if (v.kind == MOGE_MV_POINTS_SCALE) o[c] = __fmul_rn(s[c], p[0]);
        else o[c] = __fadd_rn(__fmul_rn(s[c], p[0]), p[1 + c]);
    }
}

__device__ __forceinline__ bool is_points(int kind) { return kind >= MOGE_MV_POINTS_SHIFT; }

// slot of segment id `id` in the sorted table ids[0, n), or -1
__device__ __forceinline__ int find_slot(const int32_t* ids, int n, int32_t id) {
    int lo = 0, hi = n;
    while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (ids[mid] < id) lo = mid + 1; else hi = mid;
    }
    return (lo < n && ids[lo] == id) ? lo : -1;
}

// ---------------------------------------------------------------------------------------------------- masked nearest resize
// One CTA per image.  Target pixel (i, j) has centre (cx, cy) = ((j + .5) / tw * W, (i + .5) / th * H) in fp32 and a window of
// fh x fw source pixels whose top-left is round-half-even(c - half); the output is the valid window pixel of least fp32 distance
// sqrt(dx dx + dy dy) between pixel centres, ties to the first in row-major window order (torch.argmin).  A window without a
// valid pixel returns its first pixel's index (0 when that lies outside the image).  Valid targets are then listed in row-major
// order and the list is padded to th*tw with its first entry at weight 0.
__global__ void __launch_bounds__(kResizeThreads) resize_kernel(const uint8_t* __restrict__ mask, int H, int W, int th, int tw, int fh,
                                                                 int fw, float half_h, float half_w, uint8_t* lr_mask, int64_t* lr_index,
                                                                 int64_t* list, float* list_w, int32_t* count) {
    __shared__ int warp_tot[kResizeThreads / 32];
    __shared__ int64_t first;
    const int64_t b = blockIdx.x;
    const int n = th * tw;
    const uint8_t* m = mask + b * static_cast<int64_t>(H) * W;
    const int chunk = (n + blockDim.x - 1) / blockDim.x, c0 = min(n, static_cast<int>(threadIdx.x) * chunk), c1 = min(n, c0 + chunk);
    int local = 0;
    for (int t = c0; t < c1; ++t) {
        const int i = t / tw, j = t % tw;
        const float cx = __fmul_rn(__fdiv_rn(static_cast<float>(j) + 0.5f, static_cast<float>(tw)), static_cast<float>(W));
        const float cy = __fmul_rn(__fdiv_rn(static_cast<float>(i) + 0.5f, static_cast<float>(th)), static_cast<float>(H));
        const int r0 = static_cast<int>(rintf(__fsub_rn(cy, half_h))), q0 = static_cast<int>(rintf(__fsub_rn(cx, half_w)));
        float best = INFINITY;
        int64_t best_idx = -1, first_idx = 0;
        for (int a = 0; a < fh; ++a) {
            for (int c = 0; c < fw; ++c) {
                const int r = r0 + a, q = q0 + c;
                const bool inside = r >= 0 && r < H && q >= 0 && q < W;
                const int64_t idx = inside ? static_cast<int64_t>(r) * W + q : 0;
                if (a == 0 && c == 0) first_idx = idx;
                if (!inside || !m[idx]) continue;
                const float dx = __fsub_rn(static_cast<float>(q) + 0.5f, cx), dy = __fsub_rn(static_cast<float>(r) + 0.5f, cy);
                const float d = sqrtf(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)));
                if (d < best) { best = d; best_idx = idx; }
            }
        }
        const bool valid = best_idx >= 0;
        lr_mask[b * n + t] = valid;
        lr_index[b * n + t] = valid ? best_idx : first_idx;
        local += valid;
    }
    // exclusive scan of the per-thread counts
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    int inc = local;
    for (int o = 1; o < 32; o <<= 1) {
        const int v = __shfl_up_sync(0xffffffffu, inc, o);
        if (lane >= o) inc += v;
    }
    if (lane == 31) warp_tot[warp] = inc;
    __syncthreads();
    int base = 0, total = 0;
    for (int w = 0; w < static_cast<int>(blockDim.x >> 5); ++w) { if (w < warp) base += warp_tot[w]; total += warp_tot[w]; }
    int pos = base + inc - local;
    for (int t = c0; t < c1; ++t) {
        if (!lr_mask[b * n + t]) continue;
        const int64_t idx = lr_index[b * n + t];
        if (pos == 0) first = idx;
        list[b * n + pos] = idx;
        list_w[b * n + pos] = 1.f;
        ++pos;
    }
    __syncthreads();
    const int64_t pad = total > 0 ? first : 0;
    for (int k = total + threadIdx.x; k < n; k += blockDim.x) { list[b * n + k] = pad; list_w[b * n + k] = 0.f; }
    if (threadIdx.x == 0) count[b] = total;
}

// ---------------------------------------------------------------------------------------------------- statistics pass
// grid (tiles, images).  Partials: kStatQ doubles per (image, tile).  gmax: ordered key of the masked GT max; bbox: per (image,
// slot) the ordered keys of the min of the GT points over (segment == id) & mask (3), then the complements of the keys of the max
// (3), so that both halves reduce with atomicMin from all-ones.
__global__ void __launch_bounds__(kThreads) stats_kernel(const float* __restrict__ gt_depth, const float* __restrict__ gt_points,
                                                         const uint8_t* __restrict__ mask, const float* __restrict__ disp_src,
                                                         int disp_from_depth, const int32_t* __restrict__ seg, const int32_t* __restrict__ seg_ids,
                                                         const int32_t* __restrict__ seg_count, int S, int64_t hw, int tiles,
                                                         double* part, uint32_t* gmax, uint32_t* bbox) {
    __shared__ double red[kWarps];
    __shared__ int32_t s_ids[kMaxSeg];
    __shared__ uint32_t s_box[kMaxSeg * 6];
    const int64_t b = blockIdx.y;
    const int ns = seg ? seg_count[b] : 0;
    for (int s = threadIdx.x; s < ns; s += blockDim.x) s_ids[s] = seg_ids[b * S + s];
    for (int k = threadIdx.x; k < ns * 6; k += blockDim.x) s_box[k] = 0xffffffffu;
    __syncthreads();
    double sx = 0.0, sy = 0.0, sxx = 0.0, sxy = 0.0, cnt = 0.0;
    uint32_t mx = 0;
    const int64_t p0 = static_cast<int64_t>(blockIdx.x) * kTilePx;
    for (int k = threadIdx.x; k < kTilePx; k += blockDim.x) {
        const int64_t pix = p0 + k;
        if (pix >= hw || !mask[b * hw + pix]) continue;
        const float g = gt_depth[b * hw + pix];
        if (g == g) mx = max(mx, order_key(g));
        if (disp_src) {
            const float s = disp_src[b * hw + pix];
            const double x = disp_from_depth ? __fdiv_rn(1.f, s) : s, y = __fdiv_rn(1.f, g);
            sx += x; sy += y; sxx += x * x; sxy += x * y; cnt += 1.0;
        }
        if (ns) {
            const int slot = find_slot(s_ids, ns, seg[b * hw + pix]);
            if (slot >= 0) {
                const float* q = gt_points + (b * hw + pix) * 3;
                for (int c = 0; c < 3; ++c) {
                    if (!(q[c] == q[c])) continue;
                    const uint32_t key = order_key(q[c]);
                    atomicMin(&s_box[slot * 6 + c], key);
                    atomicMin(&s_box[slot * 6 + 3 + c], ~key);
                }
            }
        }
    }
    if (mx) atomicMax(gmax + b, mx);
    if (disp_src) {
        double* out = part + (b * tiles + blockIdx.x) * kStatQ;
        sx = block_sum<kThreads>(sx, red); sy = block_sum<kThreads>(sy, red); sxx = block_sum<kThreads>(sxx, red);
        sxy = block_sum<kThreads>(sxy, red); cnt = block_sum<kThreads>(cnt, red);
        if (threadIdx.x == 0) { out[0] = sx; out[1] = sy; out[2] = sxx; out[3] = sxy; out[4] = cnt; }
    }
    __syncthreads();
    for (int k = threadIdx.x; k < ns * 6; k += blockDim.x) {
        if (s_box[k] != 0xffffffffu) atomicMin(bbox + (b * kMaxSeg) * 6 + k, s_box[k]);
    }
}

// one CTA per image: the disparity least-squares solve (fp64 normal equations, as the alignment lstsq kernel solves them), the
// clamp 1 / max GT depth, and the segment diameters max_c (max_c - min_c).
__global__ void __launch_bounds__(kThreads) stats_finalize_kernel(const double* __restrict__ part, int tiles, int has_disp,
                                                                  const uint32_t* __restrict__ gmax, const uint32_t* __restrict__ bbox,
                                                                  const int32_t* __restrict__ seg_count, int S, float* disp_params,
                                                                  float* diameter) {
    const int64_t b = blockIdx.x;
    if (threadIdx.x == 0) {
        const float mx = gmax[b] ? key_value(gmax[b]) : __int_as_float(0x7fc00000);
        float a = __int_as_float(0x7fc00000), sh = a;
        if (has_disp) {
            double q[kStatQ] = {0, 0, 0, 0, 0};
            for (int t = 0; t < tiles; ++t)
                for (int k = 0; k < kStatQ; ++k) q[k] += part[(b * tiles + t) * kStatQ + k];
            const double su = q[0], sv = q[1], su2 = q[2], suv = q[3], nn = q[4], det = su2 * nn - su * su;
            a = static_cast<float>((nn * suv - su * sv) / det);
            sh = static_cast<float>((su2 * sv - su * suv) / det);
        }
        disp_params[b * 4 + 0] = a;
        disp_params[b * 4 + 1] = sh;
        disp_params[b * 4 + 2] = static_cast<float>(1.0 / static_cast<double>(mx));   // Python's 1 / gt.max().item(), then fp32
        disp_params[b * 4 + 3] = mx;
    }
    if (diameter) {
        const int ns = seg_count[b];
        for (int s = threadIdx.x; s < S; s += blockDim.x) {
            float d = __int_as_float(0x7fc00000);
            if (s < ns) {
                const uint32_t* k = bbox + (b * kMaxSeg + s) * 6;
                if (k[0] != 0xffffffffu) {
                    d = -INFINITY;
                    for (int c = 0; c < 3; ++c) d = nan_max(d, __fsub_rn(key_value(~k[3 + c]), key_value(k[c])));
                }
            }
            diameter[b * S + s] = d;
        }
    }
}

// ---------------------------------------------------------------------------------------------------- metric pass
// grid (tiles, images).  Per masked pixel and variant: rel (|p - g| / (g + 1e-6), or |p - g| / (|g| + 1e-6) for points) and
// delta1 (max(g / p, p / g) < 1.25, or |p - g| < 0.25 min(|g|, |p|)).  Per segment slot: |p_s - g| / diameter and
// |p_s - g| < 0.25 diameter with the segment's own scale and shift.  Per-segment rel sums are summed per warp in lane order
// (lanes of one slot are combined by the lowest lane), then over warps in order; counts use integer atomics.
__global__ void __launch_bounds__(kThreads) eval_kernel(const float* __restrict__ gt_depth, const float* __restrict__ gt_points,
                                                        const uint8_t* __restrict__ mask, const Variants vars, const float* __restrict__ local_src,
                                                        const int32_t* __restrict__ seg, const int32_t* __restrict__ seg_ids,
                                                        const int32_t* __restrict__ seg_count, int S, const float* __restrict__ seg_params,
                                                        const float* __restrict__ seg_diam, int64_t hw, int tiles, double* part,
                                                        double* seg_part) {
    __shared__ double red[kWarps];
    __shared__ int32_t s_ids[kMaxSeg];
    __shared__ float s_par[kMaxSeg * 5];
    __shared__ double s_rel[kWarps][kMaxSeg];
    __shared__ uint32_t s_cnt[kMaxSeg * 2];
    const int64_t b = blockIdx.y;
    const int ns = seg ? seg_count[b] : 0;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (int s = threadIdx.x; s < ns; s += blockDim.x) {
        s_ids[s] = seg_ids[b * S + s];
        for (int c = 0; c < 4; ++c) s_par[s * 5 + c] = seg_params[(b * S + s) * 4 + c];
        s_par[s * 5 + 4] = seg_diam[b * S + s];
        s_cnt[2 * s] = 0; s_cnt[2 * s + 1] = 0;
    }
    for (int k = threadIdx.x; k < kWarps * kMaxSeg; k += blockDim.x) s_rel[k / kMaxSeg][k % kMaxSeg] = 0.0;
    __syncthreads();
    double rel[kMaxVar];
    int cnt[kMaxVar];
    int n = 0;
#pragma unroll
    for (int v = 0; v < kMaxVar; ++v) { rel[v] = 0.0; cnt[v] = 0; }
    const int64_t p0 = static_cast<int64_t>(blockIdx.x) * kTilePx;
    for (int k = threadIdx.x; k < kTilePx; k += blockDim.x) {
        const int64_t pix = p0 + k;
        const bool on = pix < hw && mask[b * hw + pix];
        int slot = -1;
        float lrel = 0.f;
        if (on) {
            ++n;
            const float g = gt_depth[b * hw + pix];
            const float* gp = gt_points + (b * hw + pix) * 3;
            const float gn = norm3(gp[0], gp[1], gp[2]);
#pragma unroll
            for (int v = 0; v < kMaxVar; ++v) {
                if (v >= vars.n) break;
                const moge_metric_variant_t& var = vars.v[v];
                if (!is_points(var.kind)) {
                    const float p = aligned_depth(var, b, hw, pix);
                    rel[v] += __fdiv_rn(fabsf(__fsub_rn(p, g)), __fadd_rn(g, 1e-6f));
                    cnt[v] += nan_max(__fdiv_rn(g, p), __fdiv_rn(p, g)) < 1.25f;
                } else {
                    float p[3];
                    aligned_point(var, b, hw, pix, p);
                    const float err = norm3(__fsub_rn(p[0], gp[0]), __fsub_rn(p[1], gp[1]), __fsub_rn(p[2], gp[2]));
                    rel[v] += __fdiv_rn(err, __fadd_rn(gn, 1e-6f));
                    cnt[v] += err < __fmul_rn(0.25f, nan_min(gn, norm3(p[0], p[1], p[2])));
                }
            }
            if (ns) {
                slot = find_slot(s_ids, ns, seg[b * hw + pix]);
                if (slot >= 0) {
                    const float* q = local_src + (b * hw + pix) * 3;
                    const float* sp = s_par + slot * 5;
                    float e[3];
                    for (int c = 0; c < 3; ++c) e[c] = __fsub_rn(__fadd_rn(__fmul_rn(q[c], sp[0]), sp[1 + c]), gp[c]);
                    const float err = norm3(e[0], e[1], e[2]);
                    lrel = __fdiv_rn(err, sp[4]);
                    atomicAdd(&s_cnt[2 * slot], 1u);
                    if (err < __fmul_rn(0.25f, sp[4])) atomicAdd(&s_cnt[2 * slot + 1], 1u);
                }
            }
        }
        if (ns && __any_sync(0xffffffffu, slot >= 0)) {
            double sum = 0.0;
            for (int l = 0; l < 32; ++l) {
                const int sl = __shfl_sync(0xffffffffu, slot, l);
                const float vl = __shfl_sync(0xffffffffu, lrel, l);
                if (sl == slot) sum += vl;
            }
            const unsigned grp = __match_any_sync(0xffffffffu, slot);
            if (slot >= 0 && lane == __ffs(grp) - 1) s_rel[warp][slot] += sum;
        }
    }
    double* out = part + (b * tiles + blockIdx.x) * kEvalQ;
    for (int v = 0; v < vars.n; ++v) {
        const double r = block_sum<kThreads>(rel[v], red), c = block_sum<kThreads>(static_cast<double>(cnt[v]), red);
        if (threadIdx.x == 0) { out[2 * v] = r; out[2 * v + 1] = c; }
    }
    const double nn = block_sum<kThreads>(static_cast<double>(n), red);
    if (threadIdx.x == 0) out[2 * kMaxVar] = nn;
    __syncthreads();
    for (int s = threadIdx.x; s < ns; s += blockDim.x) {
        double r = 0.0;
        for (int w = 0; w < kWarps; ++w) r += s_rel[w][s];
        double* o = seg_part + ((b * tiles + blockIdx.x) * S + s) * 3;
        o[0] = r; o[1] = s_cnt[2 * s + 1]; o[2] = s_cnt[2 * s];
    }
}

// one CTA per image: the tile partials in tile order, into out (see moge_metrics_eval)
__global__ void __launch_bounds__(kThreads) eval_finalize_kernel(const double* __restrict__ part, const double* __restrict__ seg_part,
                                                                 const int32_t* __restrict__ seg_count, int S, int tiles, double* out,
                                                                 int64_t stride) {
    const int64_t b = blockIdx.x;
    const int ns = seg_part ? seg_count[b] : 0;
    double* o = out + b * stride;
    for (int q = threadIdx.x; q < kEvalQ + 3 * ns; q += blockDim.x) {
        double s = 0.0;
        if (q < kEvalQ) for (int t = 0; t < tiles; ++t) s += part[(b * tiles + t) * kEvalQ + q];
        else {
            const int k = q - kEvalQ;
            for (int t = 0; t < tiles; ++t) s += seg_part[((b * tiles + t) * S + k / 3) * 3 + k % 3];
        }
        o[q < kEvalQ ? q : MOGE_METRICS_OUT_SEGMENTS + (q - kEvalQ)] = s;
    }
}

// ---------------------------------------------------------------------------------------------------- boundary F1
// grid (tiles x, tiles y, images).  A centre (i, j) counts for radius r when r <= i < H - r and r <= j < W - r; each of the 28
// offsets of the radius-3 disc is evaluated once and added to every radius whose disc (dx^2 + dy^2 <= r^2) contains it.  A ratio
// feeds the first k of the sorted thresholds; per (radius, kind) a histogram over k is kept in shared memory and turned into
// per-threshold counts at the end.
__global__ void __launch_bounds__(kThreads) boundary_kernel(const float* __restrict__ gt_depth, const uint8_t* __restrict__ mask,
                                                            const moge_metric_variant_t var, int H, int W, const Thresholds thr,
                                                            int64_t* counts, int64_t stride) {
    constexpr int NT = MOGE_METRICS_F1_THRESHOLDS;
    __shared__ float s_p[kBS * kBS], s_g[kBS * kBS];
    __shared__ uint8_t s_m[kBS * kBS];
    __shared__ uint32_t hist[3][3][NT + 1];
    const int64_t b = blockIdx.z, hw = static_cast<int64_t>(H) * W;
    const int i0 = blockIdx.y * kBT - kHalo, j0 = blockIdx.x * kBT - kHalo;
    for (int k = threadIdx.x; k < 3 * 3 * (NT + 1); k += blockDim.x) (&hist[0][0][0])[k] = 0;
    for (int k = threadIdx.x; k < kBS * kBS; k += blockDim.x) {
        const int i = i0 + k / kBS, j = j0 + k % kBS;
        const bool in = i >= 0 && i < H && j >= 0 && j < W;
        const int64_t pix = static_cast<int64_t>(i) * W + j;
        const bool m = in && mask[b * hw + pix];
        s_m[k] = m;
        s_p[k] = m ? aligned_depth(var, b, hw, pix) : 0.f;
        s_g[k] = m ? gt_depth[b * hw + pix] : 0.f;
    }
    __syncthreads();
    for (int k = threadIdx.x; k < kBT * kBT; k += blockDim.x) {
        const int li = k / kBT + kHalo, lj = k % kBT + kHalo, i = i0 + li, j = j0 + lj;
        if (i >= H || j >= W || !s_m[li * kBS + lj]) continue;
        const int rc = min(min(i, H - 1 - i), min(j, W - 1 - j));     // the largest radius this centre counts for
        if (rc < 1) continue;
        const float pc = s_p[li * kBS + lj], gc = s_g[li * kBS + lj];
        for (int dy = -3; dy <= 3; ++dy) {
            for (int dx = -3; dx <= 3; ++dx) {
                const int d2 = dx * dx + dy * dy;
                if (d2 == 0 || d2 > 9) continue;
                const int rmin = d2 <= 1 ? 1 : (d2 <= 4 ? 2 : 3);
                if (rmin > rc) continue;
                const int q = (li + dy) * kBS + lj + dx;
                if (!s_m[q]) continue;
                const float rp = __fdiv_rn(s_p[q], pc), rg = __fdiv_rn(s_g[q], gc);
                int kp = 0, kg = 0;
#pragma unroll
                for (int t = 0; t < NT; ++t) { kp += rp > thr.t[t]; kg += rg > thr.t[t]; }
                if (!(kp | kg)) continue;
                const int kt = min(kp, kg), rmax = min(rc, 3);
                for (int r = rmin; r <= rmax; ++r) {
                    if (kt) atomicAdd(&hist[r - 1][0][kt], 1u);
                    if (kg) atomicAdd(&hist[r - 1][1][kg], 1u);
                    if (kp) atomicAdd(&hist[r - 1][2][kp], 1u);
                }
            }
        }
    }
    __syncthreads();
    for (int k = threadIdx.x; k < 3 * NT * 3; k += blockDim.x) {
        const int r = k / (NT * 3), t = (k / 3) % NT, kind = k % 3;
        unsigned long long c = 0;
        for (int h = t + 1; h <= NT; ++h) c += hist[r][kind][h];
        if (c) atomicAdd(reinterpret_cast<unsigned long long*>(counts + b * stride + k), c);
    }
}

int num_tiles(int H, int W) { return static_cast<int>((static_cast<int64_t>(H) * W + kTilePx - 1) / kTilePx); }

// workspace layout: stats partials, gmax keys, bbox keys, eval partials, segment partials
struct Layout { size_t stat, gmax, bbox, eval, seg, total; };
Layout layout(int64_t batch, int H, int W, int S) {
    const size_t t = static_cast<size_t>(num_tiles(H, W)), B = static_cast<size_t>(batch);
    WsLayout ws;
    Layout l;
    l.stat = ws.add(B * t * kStatQ * 8);
    l.gmax = ws.add(B * 4);
    l.bbox = ws.add(B * kMaxSeg * 6 * 4);
    l.eval = ws.add(B * t * kEvalQ * 8);
    l.seg = ws.add(B * t * static_cast<size_t>(S) * 3 * 8);
    l.total = ws.total;
    return l;
}

int check_segments(const char* what, const int32_t* seg, const int32_t* ids, const int32_t* count, int S) {
    if (!seg) return S == 0 ? 0 : set_error("%s: segment ids given without a segmentation map", what);
    if (!ids || !count) return set_error("%s: a segmentation map needs its id table and counts", what);
    if (S < 1 || S > kMaxSeg) return set_error("%s: %d segment slots per image is outside [1, %d]", what, S, kMaxSeg);
    return 0;
}

int check_variant(const char* what, const moge_metric_variant_t& v) {
    if (v.kind < MOGE_MV_DEPTH || v.kind > MOGE_MV_POINTS_AFFINE) return set_error("%s: unknown variant kind %d", what, v.kind);
    if (!v.src) return set_error("%s: variant without a source map", what);
    if (v.kind != MOGE_MV_DEPTH && !v.params) return set_error("%s: variant kind %d needs params", what, v.kind);
    return 0;
}

}  // namespace
}  // namespace mg

using namespace mg;

extern "C" {

int moge_metrics_workspace_bytes(int64_t batch, int H, int W, int S, size_t* bytes) {
    if (!bytes) return set_error("null argument");
    MG_TRY(check_batch_map("metrics", batch, H, W, kMaxPixels));
    if (S < 0 || S > kMaxSeg) return set_error("metrics: %d segment slots per image is outside [0, %d]", S, kMaxSeg);
    *bytes = layout(batch, H, W, S).total;
    return 0;
}

int moge_metrics_resize(const uint8_t* mask, int64_t batch, int H, int W, int th, int tw, uint8_t* lr_mask, int64_t* lr_index,
                        int64_t* list, float* list_w, int32_t* count, void* stream) {
    if (!mask || !lr_mask || !lr_index || !list || !list_w || !count) return set_error("null argument");
    MG_TRY(check_batch_map("masked_nearest_resize", batch, H, W, kMaxPixels));
    if (th <= 0 || tw <= 0 || static_cast<int64_t>(th) * tw > (1 << 22))
        return set_error("masked_nearest_resize: bad target size %d x %d", th, tw);
    MG_TRY(check_device("masked_nearest_resize"));
    const double fh = std::max(1.0, static_cast<double>(H) / th), fw = std::max(1.0, static_cast<double>(W) / tw);
    const int fhi = static_cast<int>(ceil(fh)), fwi = static_cast<int>(ceil(fw));
    resize_kernel<<<static_cast<unsigned>(batch), kResizeThreads, 0, static_cast<cudaStream_t>(stream)>>>(
        mask, H, W, th, tw, fhi, fwi, static_cast<float>(fh / 2), static_cast<float>(fw / 2), lr_mask, lr_index, list, list_w, count);
    CUDA_TRY(cudaGetLastError());
    return 0;
}

int moge_metrics_stats(const float* gt_depth, const float* gt_points, const uint8_t* mask, const float* disp_src, int disp_from_depth,
                       const int32_t* seg, const int32_t* seg_ids, const int32_t* seg_count, int S, int64_t batch, int H, int W,
                       float* disp_params, float* diameter, void* workspace, size_t workspace_bytes, void* stream) {
    if (!gt_depth || !mask || !disp_params) return set_error("null argument");
    MG_TRY(check_batch_map("metrics_stats", batch, H, W, kMaxPixels));
    MG_TRY(check_segments("metrics_stats", seg, seg_ids, seg_count, S));
    if (seg && (!gt_points || !diameter)) return set_error("metrics_stats: segments need the GT points and a diameter output");
    const Layout l = layout(batch, H, W, S);
    MG_TRY(check_workspace(l.total, workspace, workspace_bytes, "metrics_stats"));
    MG_TRY(check_device("metrics_stats"));
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    char* ws = static_cast<char*>(workspace);
    uint32_t* gmax = reinterpret_cast<uint32_t*>(ws + l.gmax);
    uint32_t* bbox = reinterpret_cast<uint32_t*>(ws + l.bbox);
    CUDA_TRY(cudaMemsetAsync(gmax, 0, static_cast<size_t>(batch) * 4, st));
    if (seg) CUDA_TRY(cudaMemsetAsync(bbox, 0xff, static_cast<size_t>(batch) * kMaxSeg * 6 * 4, st));
    const int tiles = num_tiles(H, W);
    const int64_t hw = static_cast<int64_t>(H) * W;
    stats_kernel<<<dim3(tiles, static_cast<unsigned>(batch)), kThreads, 0, st>>>(gt_depth, gt_points, mask, disp_src, disp_from_depth, seg,
                                                                                  seg_ids, seg_count, S, hw, tiles,
                                                                                  reinterpret_cast<double*>(ws + l.stat), gmax, bbox);
    CUDA_TRY(cudaGetLastError());
    stats_finalize_kernel<<<static_cast<unsigned>(batch), kThreads, 0, st>>>(reinterpret_cast<const double*>(ws + l.stat), tiles,
                                                                              disp_src != nullptr, gmax, bbox, seg_count, S, disp_params,
                                                                              seg ? diameter : nullptr);
    CUDA_TRY(cudaGetLastError());
    return 0;
}

int moge_metrics_eval(const float* gt_depth, const float* gt_points, const uint8_t* mask, const moge_metric_variant_t* variants,
                      int num_variants, const float* local_src, const int32_t* seg, const int32_t* seg_ids, const int32_t* seg_count, int S,
                      const float* seg_params, const float* seg_diameter, int64_t batch, int H, int W, double* out, int64_t out_stride,
                      void* workspace, size_t workspace_bytes, void* stream) {
    if (!gt_depth || !gt_points || !mask || !out || (num_variants && !variants)) return set_error("null argument");
    MG_TRY(check_batch_map("metrics_eval", batch, H, W, kMaxPixels));
    if (num_variants < 0 || num_variants > kMaxVar) return set_error("metrics_eval: %d variants is outside [0, %d]", num_variants, kMaxVar);
    MG_TRY(check_segments("metrics_eval", seg, seg_ids, seg_count, S));
    if (seg && (!local_src || !seg_params || !seg_diameter)) return set_error("metrics_eval: segments need local points, params and diameters");
    if (out_stride < MOGE_METRICS_OUT_SEGMENTS + 3 * S) return set_error("metrics_eval: out_stride %lld is too small", static_cast<long long>(out_stride));
    Variants vars;
    memset(&vars, 0, sizeof(vars));
    vars.n = num_variants;
    for (int v = 0; v < num_variants; ++v) {
        MG_TRY(check_variant("metrics_eval", variants[v]));
        vars.v[v] = variants[v];
    }
    const Layout l = layout(batch, H, W, S);
    MG_TRY(check_workspace(l.total, workspace, workspace_bytes, "metrics_eval"));
    MG_TRY(check_device("metrics_eval"));
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    char* ws = static_cast<char*>(workspace);
    const int tiles = num_tiles(H, W);
    double* part = reinterpret_cast<double*>(ws + l.eval);
    double* seg_part = seg ? reinterpret_cast<double*>(ws + l.seg) : nullptr;
    eval_kernel<<<dim3(tiles, static_cast<unsigned>(batch)), kThreads, 0, st>>>(gt_depth, gt_points, mask, vars, local_src, seg, seg_ids, seg_count,
                                                                                 S, seg_params, seg_diameter, static_cast<int64_t>(H) * W, tiles,
                                                                                 part, seg_part);
    CUDA_TRY(cudaGetLastError());
    eval_finalize_kernel<<<static_cast<unsigned>(batch), kThreads, 0, st>>>(part, seg_part, seg_count, S, tiles, out, out_stride);
    CUDA_TRY(cudaGetLastError());
    return 0;
}

int moge_metrics_boundary(const float* gt_depth, const uint8_t* mask, const moge_metric_variant_t* aligned, const float* thresholds,
                          int64_t batch, int H, int W, int64_t* counts, int64_t counts_stride, void* stream) {
    if (!gt_depth || !mask || !aligned || !thresholds || !counts) return set_error("null argument");
    MG_TRY(check_batch_map("metrics_boundary", batch, H, W, kMaxPixels));
    MG_TRY(check_variant("metrics_boundary", *aligned));
    if (aligned->kind >= MOGE_MV_POINTS_SHIFT) return set_error("metrics_boundary: the aligned prediction must be a depth variant");
    if (counts_stride < MOGE_METRICS_F1_COUNTS) return set_error("metrics_boundary: counts_stride %lld is too small", static_cast<long long>(counts_stride));
    Thresholds thr;
    for (int t = 0; t < MOGE_METRICS_F1_THRESHOLDS; ++t) {
        thr.t[t] = thresholds[t];
        if (!(t == 0 || thr.t[t] >= thr.t[t - 1])) return set_error("metrics_boundary: thresholds must be sorted ascending");
    }
    MG_TRY(check_device("metrics_boundary"));
    const dim3 grid((W + kBT - 1) / kBT, (H + kBT - 1) / kBT, static_cast<unsigned>(batch));
    boundary_kernel<<<grid, kThreads, 0, static_cast<cudaStream_t>(stream)>>>(gt_depth, mask, *aligned, H, W, thr, counts, counts_stride);
    CUDA_TRY(cudaGetLastError());
    return 0;
}

}  // extern "C"
