// Training losses (moge/train/losses.py of the reference): the per-pixel mask losses, the edge and normal stencil losses and the
// per-pixel passes of the affine-invariant global loss, forward and backward; and the sampled local loss: its per-pixel anchor
// counts, its patch masks, and its per-patch sums and per-pixel gradient.  Every image of a batch is independent, except that
// the local loss's anchors are drawn (by torch, outside these kernels) over the whole batch.
//
// Reductions follow metrics.cu: the pixels of an image are cut into fixed tiles (set by H x W only), each CTA reduces its tile in
// fp64 in a fixed order into one partial per quantity, and a finalize kernel adds an image's partials in tile order.  Backward
// passes write each pixel's gradient from one thread: a stencil pixel gathers the terms of the pairs / quads it belongs to
// instead of scattering into them, so no float atomics are used anywhere and gradients are bitwise reproducible.
#include "common.cuh"
#include "host_api.h"
#include "../../include/moge_b200.h"
#include <math.h>
#include <stdint.h>

namespace mg {
namespace {

constexpr int kThreads = 256;
constexpr int kWarps = kThreads / 32;
constexpr int kTilePx = 8192;                 // pixels per reduction tile (32 per thread)
constexpr int64_t kMaxPixels = int64_t(1) << 29;
constexpr int kQ = MOGE_LOSS_SUMS;

// Op(b, pix, acc) adds pixel pix of image b into acc[kQ] (and may write its gradient).  part == nullptr: no reduction.
template <class Op>
__global__ void __launch_bounds__(kThreads) tile_kernel(Op op, int64_t hw, int tiles, double* part) {
    __shared__ double red[kQ][kWarps];
    const int64_t b = blockIdx.y;
    double acc[kQ] = {0.0, 0.0, 0.0, 0.0};
    const int64_t p0 = static_cast<int64_t>(blockIdx.x) * kTilePx;
    for (int k = threadIdx.x; k < kTilePx; k += kThreads) {
        const int64_t pix = p0 + k;
        if (pix < hw) op(b, pix, acc);
    }
    if (!part) return;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int q = 0; q < kQ; ++q) {
        const double v = warp_sum(acc[q]);
        if (lane == 0) red[q][warp] = v;
    }
    __syncthreads();
    if (threadIdx.x < kQ) {
        double s = 0.0;
        for (int w = 0; w < kWarps; ++w) s += red[threadIdx.x][w];
        part[(b * tiles + blockIdx.x) * kQ + threadIdx.x] = s;
    }
}

// sums[b, q] = the partials of image b added in tile order
__global__ void finalize_kernel(const double* __restrict__ part, int tiles, double* sums) {
    const int64_t b = blockIdx.x;
    const int q = threadIdx.x;
    if (q >= kQ) return;
    double s = 0.0;
    for (int t = 0; t < tiles; ++t) s += part[(b * tiles + t) * kQ + q];
    sums[b * kQ + q] = s;
}

// ---------------------------------------------------------------------------------------------------- mask losses
struct MaskOp {
    int kind;
    const float* x; const float* a; const float* bb;
    int64_t hw;
    const float* coef; float* grad;
    __device__ void operator()(int64_t b, int64_t pix, double* acc) const {
        const int64_t i = b * hw + pix;
        const float x = this->x[i], a = this->a[i], t = bb[i];
        if (kind == MOGE_LOSS_MASK_L2) {
            if (grad) {
                const float g = __fsub_rn(__fmul_rn(a, 2.f * x), __fmul_rn(t, 2.f * __fsub_rn(1.f, x)));
                grad[i] = __fmul_rn(coef[b], g);
            } else {
                const float y = __fsub_rn(1.f, x);
                acc[0] += __fadd_rn(__fmul_rn(a, __fmul_rn(x, x)), __fmul_rn(t, __fmul_rn(y, y)));
            }
        } else {
            if (grad) {
                const float den = fmaxf(__fmul_rn(__fsub_rn(1.f, x), x), 1e-12f);
                grad[i] = __fmul_rn(__fmul_rn(coef[b], a), __fdiv_rn(__fsub_rn(x, t), den));
            } else {
                const float lx = fmaxf(logf(x), -100.f), l1 = fmaxf(log1pf(-x), -100.f);
                const float bce = __fsub_rn(__fmul_rn(__fsub_rn(t, 1.f), l1), __fmul_rn(t, lx));
                acc[0] += __fmul_rn(a, bce);
            }
        }
    }
};

// ---------------------------------------------------------------------------------------------------- angle terms
struct Angle { float lo, hi, beta, half_beta; };

__device__ __forceinline__ void cross3(const float* a, const float* b, float* c) {
    c[0] = __fsub_rn(__fmul_rn(a[1], b[2]), __fmul_rn(a[2], b[1]));
    c[1] = __fsub_rn(__fmul_rn(a[2], b[0]), __fmul_rn(a[0], b[2]));
    c[2] = __fsub_rn(__fmul_rn(a[0], b[1]), __fmul_rn(a[1], b[0]));
}
__device__ __forceinline__ float dot3(const float* a, const float* b) {
    return __fadd_rn(__fadd_rn(__fmul_rn(a[0], b[0]), __fmul_rn(a[1], b[1])), __fmul_rn(a[2], b[2]));
}

// The term smooth(clamp(atan2(|v x u| + 1e-12, v . u), lo, hi)) of predicted vector v and GT vector u.  With gv, adds coef times
// its gradient with respect to v into gv (torch autograd's rules: clamp passes the gradient at its bounds inclusively, the norm of
// a zero vector has gradient 0, a where() sends it to the branch it took).
__device__ float angle_term(const float* v, const float* u, const Angle& ag, float coef, float* gv) {
    float c[3];
    cross3(v, u, c);
    const float n = sqrtf(dot3(c, c)), d = dot3(v, u);
    const float y = __fadd_rn(n, 1e-12f);
    const float th = atan2f(y, d);
    const float tc = th < ag.lo ? ag.lo : (th > ag.hi ? ag.hi : th);     // NaN stays NaN
    const bool quad = tc < ag.beta;
    const float f = quad ? __fdiv_rn(__fmul_rn(0.5f, __fmul_rn(tc, tc)), ag.beta) : __fsub_rn(tc, ag.half_beta);
    if (gv && th >= ag.lo && th <= ag.hi) {
        const float gt = quad ? __fmul_rn(coef, __fdiv_rn(tc, ag.beta)) : coef;
        const float den = __fadd_rn(__fmul_rn(y, y), __fmul_rn(d, d));
        const float gy = __fdiv_rn(__fmul_rn(gt, d), den), gd = __fdiv_rn(__fmul_rn(-gt, y), den);
        const float s = n > 0.f ? __fdiv_rn(gy, n) : 0.f;
        const float gc[3] = {__fmul_rn(s, c[0]), __fmul_rn(s, c[1]), __fmul_rn(s, c[2])};
        float uxg[3];
        cross3(u, gc, uxg);                   // d(v x u)/dv applied to gc
        for (int k = 0; k < 3; ++k) gv[k] = __fadd_rn(gv[k], __fadd_rn(uxg[k], __fmul_rn(gd, u[k])));
    }
    return f;
}

// point k of image b, and its GT point with the reference's substitution of (1, 1, 1) for an invalid one
struct Maps {
    const float* p; const float* g; int H, W; int64_t hw;
    __device__ __forceinline__ void load(int64_t b, int i, int j, float* pp, float* gg, bool* m) const {
        const int64_t o = (b * hw + static_cast<int64_t>(i) * W + j) * 3;
        for (int k = 0; k < 3; ++k) pp[k] = p[o + k];
        *m = isfinite(g[o]) && isfinite(g[o + 1]) && isfinite(g[o + 2]);
        for (int k = 0; k < 3; ++k) gg[k] = *m ? g[o + k] : 1.f;
    }
};

// ---------------------------------------------------------------------------------------------------- edge loss
// pair (i, j)-(i+1, j) is `dx` (sums[0]), pair (i, j)-(i, j+1) is `dy` (sums[1]); v = first - second
struct EdgeOp {
    Maps mp; Angle ag; const float* coef; float* grad;
    __device__ float pair(int64_t b, int i0, int j0, int i1, int j1, float cf, float* g0, float* g1) const {
        float p0[3], q0[3], p1[3], q1[3], v[3], u[3];
        bool m0, m1;
        mp.load(b, i0, j0, p0, q0, &m0);
        mp.load(b, i1, j1, p1, q1, &m1);
        for (int k = 0; k < 3; ++k) { v[k] = __fsub_rn(p0[k], p1[k]); u[k] = __fsub_rn(q0[k], q1[k]); }
        const float mask = (m0 && m1) ? 1.f : 0.f;
        float gv[3] = {0.f, 0.f, 0.f};
        const float f = angle_term(v, u, ag, __fmul_rn(cf, mask), g0 ? gv : nullptr);
        if (g0) for (int k = 0; k < 3; ++k) { g0[k] = __fadd_rn(g0[k], gv[k]); g1[k] = __fsub_rn(g1[k], gv[k]); }
        return __fmul_rn(mask, f);
    }
    __device__ void operator()(int64_t b, int64_t pix, double* acc) const {
        const int i = static_cast<int>(pix / mp.W), j = static_cast<int>(pix % mp.W);
        if (!grad) {
            if (i + 1 < mp.H) acc[0] += pair(b, i, j, i + 1, j, 0.f, nullptr, nullptr);
            if (j + 1 < mp.W) acc[1] += pair(b, i, j, i, j + 1, 0.f, nullptr, nullptr);
            return;
        }
        // this pixel is the second point of the pairs above / left of it and the first of those below / right, in that order
        float g[3] = {0.f, 0.f, 0.f}, dummy[3] = {0.f, 0.f, 0.f};
        const float cx = coef[2 * b], cy = coef[2 * b + 1];
        if (i > 0) pair(b, i - 1, j, i, j, cx, dummy, g);
        if (i + 1 < mp.H) pair(b, i, j, i + 1, j, cx, g, dummy);
        if (j > 0) pair(b, i, j - 1, i, j, cy, dummy, g);
        if (j + 1 < mp.W) pair(b, i, j, i, j + 1, cy, g, dummy);
        for (int k = 0; k < 3; ++k) grad[pix * 3 + b * mp.hw * 3 + k] = g[k];
    }
};

// ---------------------------------------------------------------------------------------------------- normal loss
// The quad with top-left (i, j) has corners 0 = (i, j), 1 = (i, j+1), 2 = (i+1, j), 3 = (i+1, j+1); its triangles (P, Q, R) give
// the normal (P - R) x (Q - R): upxleft (1, 2, 3), leftxdown (0, 3, 1), downxright (2, 1, 0), rightxup (3, 0, 2).
__constant__ int kTri[4][3] = {{1, 2, 3}, {0, 3, 1}, {2, 1, 0}, {3, 0, 2}};

struct NormalOp {
    Maps mp; Angle ag; const float* coef; float* grad;
    // the quad's loss; with corner >= 0, adds cf times the gradient with respect to that corner into gk
    __device__ float quad(int64_t b, int i, int j, float cf, int corner, float* gk) const {
        float p[4][3], q[4][3];
        bool m[4];
        for (int c = 0; c < 4; ++c) mp.load(b, i + (c >> 1), j + (c & 1), p[c], q[c], &m[c]);
        float total = 0.f;
        for (int t = 0; t < 4; ++t) {
            const int P = kTri[t][0], Q = kTri[t][1], R = kTri[t][2];
            float a[3], bv[3], ga[3], gb[3], v[3], u[3];
            for (int k = 0; k < 3; ++k) { a[k] = __fsub_rn(p[P][k], p[R][k]); bv[k] = __fsub_rn(p[Q][k], p[R][k]); }
            cross3(a, bv, v);
            for (int k = 0; k < 3; ++k) { ga[k] = __fsub_rn(q[P][k], q[R][k]); gb[k] = __fsub_rn(q[Q][k], q[R][k]); }
            cross3(ga, gb, u);
            const float mask = (m[P] && m[Q] && m[R]) ? 1.f : 0.f;
            const bool want = corner == P || corner == Q || corner == R;
            float gv[3] = {0.f, 0.f, 0.f};
            const float f = angle_term(v, u, ag, __fmul_rn(cf, mask), want ? gv : nullptr);
            if (t == 0) total = __fmul_rn(mask, f);
            else total = __fadd_rn(total, __fmul_rn(mask, f));
            if (!want) continue;
            float da[3], db[3];
            cross3(bv, gv, da);               // d(a x b)/da applied to gv
            cross3(gv, a, db);                // d(a x b)/db applied to gv
            for (int k = 0; k < 3; ++k) {
                const float d = corner == P ? da[k] : (corner == Q ? db[k] : -__fadd_rn(da[k], db[k]));
                gk[k] = __fadd_rn(gk[k], d);
            }
        }
        return total;
    }
    __device__ void operator()(int64_t b, int64_t pix, double* acc) const {
        const int i = static_cast<int>(pix / mp.W), j = static_cast<int>(pix % mp.W);
        if (!grad) {
            if (i + 1 < mp.H && j + 1 < mp.W) acc[0] += quad(b, i, j, 0.f, -1, nullptr);
            return;
        }
        // the quads touching this pixel in row-major order of their top-left corner, the pixel being corner 3, 2, 1, 0 of them
        float g[3] = {0.f, 0.f, 0.f};
        const float cf = coef[2 * b];
        for (int c = 3; c >= 0; --c) {
            const int qi = i - (c >> 1), qj = j - (c & 1);
            if (qi >= 0 && qj >= 0 && qi + 1 < mp.H && qj + 1 < mp.W) quad(b, qi, qj, cf, c, g);
        }
        for (int k = 0; k < 3; ++k) grad[(b * mp.hw + pix) * 3 + k] = g[k];
    }
};

// ---------------------------------------------------------------------------------------------------- global loss
struct GlobalOp {
    const float* p; const float* g; const float* params; float beta; int pass; int64_t hw; float* grad;
    __device__ void operator()(int64_t b, int64_t pix, double* acc) const {
        const int64_t o = (b * hw + pix) * 3;
        const float* pr = params + b * 8;
        const bool m = isfinite(g[o]) && isfinite(g[o + 1]) && isfinite(g[o + 2]);
        float gg[3];
        for (int k = 0; k < 3; ++k) gg[k] = m ? g[o + k] : 1.f;
        float w = __fdiv_rn((pr[4] != 0.f && m) ? 1.f : 0.f, fmaxf(gg[2], 1e-5f));
        if (pass == 0) {
            acc[0] += w;
            acc[1] += m ? 1.0 : 0.0;
            return;
        }
        if (w > pr[5]) w = pr[5];             // clamp_max(cap)
        const float s = pr[0];
        float diff[3], sq = 0.f, gsum[3];
        float gscale = 0.f;
        for (int k = 0; k < 3; ++k) {
            const float q = __fadd_rn(__fmul_rn(s, p[o + k]), pr[1 + k]);
            diff[k] = __fsub_rn(q, gg[k]);
            sq = __fadd_rn(sq, __fmul_rn(diff[k], diff[k]));
            const float e = __fmul_rn(fabsf(diff[k]), w);
            const bool quad = beta > 0.f && e < beta;
            if (pass == 1) {
                acc[0] += beta > 0.f ? (quad ? __fdiv_rn(__fmul_rn(0.5f, __fmul_rn(e, e)), beta) : __fsub_rn(e, 0.5f * beta)) : e;
            } else {
                const float sgn = diff[k] > 0.f ? 1.f : (diff[k] < 0.f ? -1.f : 0.f);
                const float de = quad ? __fdiv_rn(e, beta) : 1.f;
                const float gq = __fmul_rn(__fmul_rn(__fmul_rn(pr[6], de), w), sgn);     // dL/dq
                gsum[k] = gq;
                grad[o + k] = __fmul_rn(gq, s);
                gscale = __fadd_rn(gscale, __fmul_rn(gq, p[o + k]));
            }
        }
        if (pass == 1) {
            if (m) {
                const float err = __fdiv_rn(sqrtf(sq), gg[2]);
                acc[1] += err > 1.f ? 1.f : err;
                acc[2] += err < 1.f ? 1.0 : 0.0;
            }
        } else {
            acc[0] += gscale;
            for (int k = 0; k < 3; ++k) acc[1 + k] += gsum[k];
        }
    }
};

// ---------------------------------------------------------------------------------------------------- local loss
// |a - b| in fp32, summed as ((x^2 + y^2) + z^2); the fp64 square root rounded to fp32 is the fp32 square root (53 >= 2 * 24 + 2
// bits: the double rounding is innocuous), without the fp32 slow path's call
__device__ __forceinline__ float dist3(const float* a, const float* b) {
    const float dx = __fsub_rn(a[0], b[0]), dy = __fsub_rn(a[1], b[1]), dz = __fsub_rn(a[2], b[2]);
    return static_cast<float>(sqrt(static_cast<double>(__fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz)))));
}

// compute_anchor_sampling_weight: pixel (b, i, j) counts its num_test offsets (di, dj shared by the images) whose clamped target
// is inside the map, valid and within radius[b, i, j] of it; weight = mask ? 1 / max(count, 1) : 0
__global__ void __launch_bounds__(kThreads) anchor_weight_kernel(const float* __restrict__ points, const uint8_t* __restrict__ mask,
                                                                 const int64_t* __restrict__ di, const int64_t* __restrict__ dj,
                                                                 const float* __restrict__ radius, int64_t batch, int H, int W,
                                                                 int num_test, float* __restrict__ weight) {
    const int64_t hw = static_cast<int64_t>(H) * W;
    const int64_t t = static_cast<int64_t>(blockIdx.x) * kThreads + threadIdx.x;
    if (t >= batch * hw) return;
    const int64_t b = t / hw, pix = t % hw;
    const int i = static_cast<int>(pix / W), j = static_cast<int>(pix % W);
    if (!mask[t]) { weight[t] = 0.f; return; }
    const float* p = points + t * 3;
    const float r = radius[t];
    int count = 0;
    for (int k = 0; k < num_test; ++k) {
        const int64_t ti = i + di[pix * num_test + k], tj = j + dj[pix * num_test + k];
        if (ti < 0 || ti >= H || tj < 0 || tj >= W) continue;
        const int64_t q = b * hw + ti * W + tj;
        if (mask[q] && dist3(points + q * 3, p) <= r) ++count;
    }
    weight[t] = __frcp_rn(static_cast<float>(count > 1 ? count : 1));
}

// the patches of the local loss: patch p = (image, anchor i, anchor j) = anchor[3 p ..], side S = 2 r + 1.  Position (u, v) is
// pixel (ai - r + u, aj - r + v); it is in the patch mask when that pixel is inside the map, valid, and within the anchor's 3D
// radius = (1 / focal) * half_level * anchor z (torch's `half_level / focal * z`).
constexpr int kPatchPx = 4096;                  // positions per CTA of the patch-mask kernel

__global__ void __launch_bounds__(kThreads) patch_mask_kernel(const float* __restrict__ gt, const uint8_t* __restrict__ mask,
                                                              const int64_t* __restrict__ anchor, const float* __restrict__ focal,
                                                              float half_level, int H, int W, int r, uint8_t* __restrict__ pmask,
                                                              int* __restrict__ count, float* __restrict__ radius) {
    __shared__ int red[kWarps];
    const int64_t p = blockIdx.y;
    const int S = 2 * r + 1;
    const int64_t hw = static_cast<int64_t>(H) * W;
    const int64_t b = anchor[p * 3], ai = anchor[p * 3 + 1], aj = anchor[p * 3 + 2];
    const float* g0 = gt + (b * hw + ai * W + aj) * 3;
    const float rad = __fmul_rn(__fmul_rn(__frcp_rn(focal[b]), half_level), g0[2]);
    if (blockIdx.x == 0 && threadIdx.x == 0) radius[p] = rad;
    int n = 0;
    const int64_t k0 = static_cast<int64_t>(blockIdx.x) * kPatchPx, S2 = static_cast<int64_t>(S) * S;
    for (int64_t k = k0 + threadIdx.x; k < k0 + kPatchPx && k < S2; k += kThreads) {
        const int64_t i = ai - r + k / S, j = aj - r + k % S;
        bool m = i >= 0 && i < H && j >= 0 && j < W;
        if (m) {
            const int64_t q = b * hw + i * W + j;
            m = mask[q] && dist3(gt + q * 3, g0) <= rad;
        }
        pmask[p * S2 + k] = m;
        n += m;
    }
    for (int o = 16; o > 0; o >>= 1) n += __shfl_xor_sync(0xffffffffu, n, o);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = n;
    __syncthreads();
    if (threadIdx.x == 0) {
        int s = 0;
        for (int w = 0; w < kWarps; ++w) s += red[w];
        atomicAdd(count + p, s);                // integer: the same total in any order
    }
}

// per-patch parameters of the local loss (MOGE_LOSS_LOCAL_PARAMS floats)
enum { LP_SCALE = 0, LP_SHIFT = 1, LP_VALID = 4, LP_CAP = 5, LP_RADIUS = 6, LP_COEF = 7 };

struct LocalArgs {
    const float* p; const float* g; const int64_t* anchor; const float* params; const uint8_t* pmask;
    float beta; int H, W, r; int64_t P;
};

// d(smooth(|q - g| w))/dq for one coordinate, times coef; with val, also the term itself
__device__ __forceinline__ float local_term(float diff, float w, float beta, float coef, float* val) {
    const float e = __fmul_rn(fabsf(diff), w);
    const bool quad = beta > 0.f && e < beta;
    if (val) *val = beta > 0.f ? (quad ? __fdiv_rn(__fmul_rn(0.5f, __fmul_rn(e, e)), beta) : __fsub_rn(e, 0.5f * beta)) : e;
    const float sgn = diff > 0.f ? 1.f : (diff < 0.f ? -1.f : 0.f);
    return __fmul_rn(__fmul_rn(__fmul_rn(coef, quad ? __fdiv_rn(e, beta) : 1.f), w), sgn);
}

// pass 0: per image, (sum over valid GT of 1 / (z + 1e-7), valid count), for the harmonic mean of the GT depth
struct HarmonicOp {
    const float* g; int64_t hw;
    __device__ void operator()(int64_t b, int64_t pix, double* acc) const {
        const float* q = g + (b * hw + pix) * 3;
        if (!(isfinite(q[0]) && isfinite(q[1]) && isfinite(q[2]))) return;
        acc[0] += __frcp_rn(__fadd_rn(q[2], 1e-7f));
        acc[1] += 1.0;
    }
};

// passes 1 and 2 over the positions of a patch (its `b` is the patch), masked positions only: with q = scale p + shift,
// pass 1: (sum of smooth(|q - g| w) over xyz, mask count, sum of min(err, 1), count of err < 1), err = |q - g| / radius;
// pass 2: (dL/dscale, dL/dshift x, y, z) with dL/dterm = coef.
struct PatchOp {
    LocalArgs a; int pass;
    __device__ void operator()(int64_t p, int64_t k, double* acc) const {
        const int S = 2 * a.r + 1;
        const float* pr = a.params + p * MOGE_LOSS_LOCAL_PARAMS;
        if (pr[LP_VALID] == 0.f || !a.pmask[p * S * S + k]) return;
        const int64_t b = a.anchor[p * 3];
        const int64_t i = a.anchor[p * 3 + 1] - a.r + k / S, j = a.anchor[p * 3 + 2] - a.r + k % S;
        const int64_t o = ((b * a.H + i) * a.W + j) * 3;
        const float w = __frcp_rn(fmaxf(a.g[o + 2], pr[LP_CAP]));
        float sq = 0.f, gscale = 0.f, loss = 0.f;
        for (int c = 0; c < 3; ++c) {
            const float diff = __fsub_rn(__fadd_rn(__fmul_rn(pr[LP_SCALE], a.p[o + c]), pr[LP_SHIFT + c]), a.g[o + c]);
            if (pass == 1) {
                float v;
                local_term(diff, w, a.beta, 0.f, &v);
                loss = __fadd_rn(loss, v);
                sq = __fadd_rn(sq, __fmul_rn(diff, diff));
            } else {
                const float gq = local_term(diff, w, a.beta, pr[LP_COEF], nullptr);
                gscale = __fadd_rn(gscale, __fmul_rn(gq, a.p[o + c]));
                acc[1 + c] += gq;
            }
        }
        if (pass == 1) {
            const float err = __fdiv_rn(sqrtf(sq), pr[LP_RADIUS]);
            acc[0] += loss;
            acc[1] += 1.0;
            acc[2] += err > 1.f ? 1.f : err;
            acc[3] += err < 1.f ? 1.0 : 0.0;
        } else {
            acc[0] += gscale;
        }
    }
};

// dL/dpred of the local loss: one thread per pixel gathers, in patch order, the terms of every patch position on it.  A CTA
// covers a kTile x kTile pixel tile of one image; it scans the patches kThreads at a time and lists, in patch order, those of
// its image whose box meets the tile, then each thread adds the listed patches' terms at its pixels.
constexpr int kTile = 16;
constexpr int kRows = kTile * kTile / kThreads;  // pixels per thread

__global__ void __launch_bounds__(kThreads) local_grad_kernel(LocalArgs a, float* __restrict__ grad) {
    __shared__ int list[kThreads];
    __shared__ int listed;
    const int64_t b = blockIdx.z;
    const int i0 = blockIdx.y * kTile, j0 = blockIdx.x * kTile;
    const int lane = threadIdx.x & 31;
    const int S = 2 * a.r + 1;
    float g[kRows][3] = {};
    for (int64_t c0 = 0; c0 < a.P; c0 += kThreads) {
        if (threadIdx.x < 32) {                 // warp 0 lists the chunk's patches that meet the tile, in order
            int n = 0;
            for (int s = 0; s < kThreads; s += 32) {
                const int64_t p = c0 + s + lane;
                bool hit = false;
                if (p < a.P && a.anchor[p * 3] == b && a.params[p * MOGE_LOSS_LOCAL_PARAMS + LP_VALID] != 0.f) {
                    const int64_t ai = a.anchor[p * 3 + 1], aj = a.anchor[p * 3 + 2];
                    hit = ai + a.r >= i0 && ai - a.r < i0 + kTile && aj + a.r >= j0 && aj - a.r < j0 + kTile;
                }
                const unsigned bal = __ballot_sync(0xffffffffu, hit);
                if (hit) list[n + __popc(bal & ((1u << lane) - 1u))] = static_cast<int>(p);
                n += __popc(bal);
            }
            if (lane == 0) listed = n;
        }
        __syncthreads();
        const int n = listed;
        for (int e = 0; e < n; ++e) {
            const int64_t q = list[e];
            const float* pr = a.params + q * MOGE_LOSS_LOCAL_PARAMS;
            const int64_t u0 = a.anchor[q * 3 + 1] - a.r, v0 = a.anchor[q * 3 + 2] - a.r;
#pragma unroll
            for (int k = 0; k < kRows; ++k) {
                const int i = i0 + (threadIdx.x / kTile) + k * (kThreads / kTile), j = j0 + (threadIdx.x % kTile);
                const int64_t u = i - u0, v = j - v0;
                if (i >= a.H || j >= a.W || u < 0 || u >= S || v < 0 || v >= S || !a.pmask[(q * S + u) * S + v]) continue;
                const int64_t o = ((b * a.H + i) * a.W + j) * 3;
                const float w = __frcp_rn(fmaxf(a.g[o + 2], pr[LP_CAP]));
                for (int c = 0; c < 3; ++c) {
                    const float diff = __fsub_rn(__fadd_rn(__fmul_rn(pr[LP_SCALE], a.p[o + c]), pr[LP_SHIFT + c]), a.g[o + c]);
                    g[k][c] = __fadd_rn(g[k][c], __fmul_rn(local_term(diff, w, a.beta, pr[LP_COEF], nullptr), pr[LP_SCALE]));
                }
            }
        }
        __syncthreads();
    }
#pragma unroll
    for (int k = 0; k < kRows; ++k) {
        const int i = i0 + (threadIdx.x / kTile) + k * (kThreads / kTile), j = j0 + (threadIdx.x % kTile);
        if (i >= a.H || j >= a.W) continue;
        for (int c = 0; c < 3; ++c) grad[((b * a.H + i) * a.W + j) * 3 + c] = g[k][c];
    }
}

int num_tiles(int H, int W) { return static_cast<int>((static_cast<int64_t>(H) * W + kTilePx - 1) / kTilePx); }

size_t workspace_size(int64_t batch, int H, int W) { return WsLayout::up(static_cast<size_t>(batch) * num_tiles(H, W) * kQ * 8); }

// one pass of op over every pixel; reduces into sums unless grad mode
template <class Op>
int run(const char* what, const Op& op, bool reduce, int64_t batch, int H, int W, double* sums, void* workspace, size_t workspace_bytes,
        void* stream) {
    if (reduce) {
        if (!sums) return set_error("%s: null sums", what);
        MG_TRY(check_workspace(workspace_size(batch, H, W), workspace, workspace_bytes, what));
    }
    MG_TRY(check_device(what));
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const int tiles = num_tiles(H, W);
    double* part = reduce ? static_cast<double*>(workspace) : nullptr;
    tile_kernel<Op><<<dim3(tiles, static_cast<unsigned>(batch)), kThreads, 0, st>>>(op, static_cast<int64_t>(H) * W, tiles, part);
    CUDA_TRY(cudaGetLastError());
    if (reduce) {
        finalize_kernel<<<static_cast<unsigned>(batch), 32, 0, st>>>(part, tiles, sums);
        CUDA_TRY(cudaGetLastError());
    }
    return 0;
}

constexpr double kDeg = 3.14159265358979323846 / 180.0;

}  // namespace
}  // namespace mg

using namespace mg;

extern "C" {

int moge_loss_workspace_bytes(int64_t batch, int H, int W, size_t* bytes) {
    if (!bytes) return set_error("null argument");
    MG_TRY(check_batch_map("loss", batch, H, W, kMaxPixels));
    *bytes = workspace_size(batch, H, W);
    return 0;
}

int moge_loss_mask(int kind, const float* pred, const float* a, const float* b, int64_t batch, int H, int W, const float* coef,
                   float* grad, double* sums, void* workspace, size_t workspace_bytes, void* stream) {
    if (!pred || !a || !b || (coef && !grad)) return set_error("null argument");
    if (kind != MOGE_LOSS_MASK_L2 && kind != MOGE_LOSS_MASK_BCE) return set_error("loss_mask: unknown kind %d", kind);
    MG_TRY(check_batch_map("loss_mask", batch, H, W, kMaxPixels));
    const MaskOp op{kind, pred, a, b, static_cast<int64_t>(H) * W, coef, coef ? grad : nullptr};
    return run("loss_mask", op, coef == nullptr, batch, H, W, sums, workspace, workspace_bytes, stream);
}

int moge_loss_stencil(int kind, const float* points, const float* gt, int64_t batch, int H, int W, const float* coef, float* grad,
                      double* sums, void* workspace, size_t workspace_bytes, void* stream) {
    if (!points || !gt || (coef && !grad)) return set_error("null argument");
    MG_TRY(check_batch_map("loss_stencil", batch, H, W, kMaxPixels));
    const Maps mp{points, gt, H, W, static_cast<int64_t>(H) * W};
    const float beta = static_cast<float>(3 * kDeg);
    if (kind == MOGE_LOSS_EDGE) {
        const Angle ag{static_cast<float>(0.1 * kDeg), static_cast<float>(90 * kDeg), beta, static_cast<float>(0.5 * 3 * kDeg)};
        const EdgeOp op{mp, ag, coef, coef ? grad : nullptr};
        return run("loss_stencil", op, coef == nullptr, batch, H, W, sums, workspace, workspace_bytes, stream);
    }
    if (kind == MOGE_LOSS_NORMAL) {
        const Angle ag{static_cast<float>(1 * kDeg), static_cast<float>(90 * kDeg), beta, static_cast<float>(0.5 * 3 * kDeg)};
        const NormalOp op{mp, ag, coef, coef ? grad : nullptr};
        return run("loss_stencil", op, coef == nullptr, batch, H, W, sums, workspace, workspace_bytes, stream);
    }
    return set_error("loss_stencil: unknown kind %d", kind);
}

int moge_loss_global(const float* pred, const float* gt, const float* params, float beta, int pass, int64_t batch, int H, int W,
                     float* grad, double* sums, void* workspace, size_t workspace_bytes, void* stream) {
    if (!pred || !gt || !params || (pass == 2 && !grad)) return set_error("null argument");
    if (pass < 0 || pass > 2) return set_error("loss_global: unknown pass %d", pass);
    if (!(beta >= 0.f)) return set_error("loss_global: beta must be >= 0");
    MG_TRY(check_batch_map("loss_global", batch, H, W, kMaxPixels));
    const GlobalOp op{pred, gt, params, beta, pass, static_cast<int64_t>(H) * W, grad};
    return run("loss_global", op, true, batch, H, W, sums, workspace, workspace_bytes, stream);
}

int moge_loss_anchor_weight(const float* points, const uint8_t* mask, const int64_t* di, const int64_t* dj, const float* radius,
                            int64_t batch, int H, int W, int num_test, float* weight, void* stream) {
    if (!points || !mask || !di || !dj || !radius || !weight) return set_error("null argument");
    MG_TRY(check_batch_map("loss_anchor_weight", batch, H, W, kMaxPixels));
    if (num_test < 0) return set_error("loss_anchor_weight: num_test %d < 0", num_test);
    MG_TRY(check_device("loss_anchor_weight"));
    const int64_t n = batch * H * W;
    anchor_weight_kernel<<<static_cast<unsigned>((n + kThreads - 1) / kThreads), kThreads, 0, static_cast<cudaStream_t>(stream)>>>(
        points, mask, di, dj, radius, batch, H, W, num_test, weight);
    CUDA_TRY(cudaGetLastError());
    return 0;
}

static int check_patches(const char* what, int64_t batch, int H, int W, int64_t P, int r) {
    MG_TRY(check_batch_map(what, batch, H, W, kMaxPixels));
    if (P < 1 || P > 65535) return set_error("%s: %lld patches outside [1, 65535]", what, static_cast<long long>(P));
    if (r < 0 || r > 16383) return set_error("%s: patch radius %d outside [0, 16383]", what, r);
    return 0;
}

int moge_loss_patch_mask(const float* gt, const uint8_t* mask, const int64_t* anchor, const float* focal, float half_level,
                         int64_t batch, int H, int W, int64_t P, int r, uint8_t* patch_mask, int* count, float* radius, void* stream) {
    if (!gt || !mask || !anchor || !focal || !patch_mask || !count || !radius) return set_error("null argument");
    MG_TRY(check_patches("loss_patch_mask", batch, H, W, P, r));
    MG_TRY(check_device("loss_patch_mask"));
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const int64_t S2 = static_cast<int64_t>(2 * r + 1) * (2 * r + 1);
    CUDA_TRY(cudaMemsetAsync(count, 0, P * sizeof(int), st));
    patch_mask_kernel<<<dim3(static_cast<unsigned>((S2 + kPatchPx - 1) / kPatchPx), static_cast<unsigned>(P)), kThreads, 0, st>>>(
        gt, mask, anchor, focal, half_level, H, W, r, patch_mask, count, radius);
    CUDA_TRY(cudaGetLastError());
    return 0;
}

int moge_loss_local(const float* pred, const float* gt, const int64_t* anchor, const float* params, const uint8_t* patch_mask,
                    float beta, int pass, int64_t batch, int H, int W, int64_t P, int r, float* grad, double* sums, void* workspace,
                    size_t workspace_bytes, void* stream) {
    if (!gt || (pass > 0 && (!pred || !anchor || !params || !patch_mask))) return set_error("null argument");
    if (pass < 0 || pass > 2) return set_error("loss_local: unknown pass %d", pass);
    if (!(beta >= 0.f)) return set_error("loss_local: beta must be >= 0");
    if (pass == 0) {
        MG_TRY(check_batch_map("loss_local", batch, H, W, kMaxPixels));
        const HarmonicOp op{gt, static_cast<int64_t>(H) * W};
        return run("loss_local", op, true, batch, H, W, sums, workspace, workspace_bytes, stream);
    }
    MG_TRY(check_patches("loss_local", batch, H, W, P, r));
    const LocalArgs a{pred, gt, anchor, params, patch_mask, beta, H, W, r, P};
    const int S = 2 * r + 1;
    MG_TRY(run("loss_local", PatchOp{a, pass}, true, P, S, S, sums, workspace, workspace_bytes, stream));
    if (pass == 2 && grad) {
        const dim3 grid((W + kTile - 1) / kTile, (H + kTile - 1) / kTile, static_cast<unsigned>(batch));
        if (batch > 65535) return set_error("loss_local: batch %lld > 65535", static_cast<long long>(batch));
        local_grad_kernel<<<grid, kThreads, 0, static_cast<cudaStream_t>(stream)>>>(a, grad);
        CUDA_TRY(cudaGetLastError());
    }
    return 0;
}

}  // extern "C"
