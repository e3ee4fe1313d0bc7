// Panorama inference (moge/utils/panorama.py and moge/scripts/infer_panorama.py:83-122 of the reference) on the device.
//
// split: every view pixel's ray (the view camera's unprojection, in fp64 with one rounding per operation, as the utils3d
// restatement in oracle/utils3d_panorama.py writes it), its spherical uv and panorama pixel, rounded to fp32 and sampled as
// cv2.remap(INTER_LINEAR, BORDER_CONSTANT 0) samples a uint8 image: coordinates snapped to 1/32 pixel, 15-bit fixed-point
// weights.  Bitwise equal to cv2 for the same fp32 coordinates.
//
// merge, per pyramid level of h x w: a sample pass projects each panorama direction into every view (fp32 rotation, fp64
// projection) and samples log |p| with cv2's fp32 bilinear (1/32 snapping, replicate border) and the view mask with its nearest
// rule; a right-hand-side pass forms the x / y gradients and the 5-point Laplacians of every view with their masks, sums them over
// the views in view order in fp32 and divides by the counts in fp64.  Rows are dense: h*w x-gradient, (h-1)*(w+1) y-gradient and
// h*w Laplacian rows; a masked-out row has b = 0 and no equation.  The y-gradient rows run over w + 1 columns because the
// reference builds them on the x-wrapped grid: column w repeats column 0, so that equation is in the system twice.
//
// lsmr: SciPy's LSMR (scipy/sparse/linalg/_isolve/lsmr.py) on that stencil system in one cooperative kernel: grid-wide barriers
// between the matrix products, fp64 u, v, h, hbar, x stored in fp64 but rounded to fp32 after each update when the level starts
// from an initial guess (SciPy keeps x0's dtype), and the scalar recurrences and stopping rules evaluated from deterministic
// reductions.  The iteration count and istop are written to the device.  One launch solves the
// systems of a batch of panoramas, each bitwise as alone (see lsmr_kernel); a single merge is a batch of one.
//
// Every stage takes up to MOGE_PANORAMA_MAX_BATCH panoramas, each of its own size, with one set of cameras.  They reach the
// kernels as a table passed by value (__grid_constant__, read in place from the parameter bank), so a launch uploads nothing.
// The per-pixel kernels take the panorama from blockIdx.y and stride over its pixels in x, so each thread does the same work
// at any batch size and mix of sizes; the LSMR finds a virtual block's system by a binary search on the systems' first
// virtual blocks.  A batch of one size is the case where every entry has the same size.
#include "host_api.h"
#include "../../include/moge_b200.h"
#include <cooperative_groups.h>
#include <algorithm>
#include <math.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

namespace cg = cooperative_groups;

namespace mg {
namespace {

constexpr int kThreads = 256;
constexpr int kLsmrThreads = 512;
constexpr int64_t kMaxPixels = int64_t(1) << 28;

struct Cams { moge_panorama_camera_t c[MOGE_PANORAMA_MAX_VIEWS]; int n; };

__device__ __forceinline__ double dmul(double a, double b) { return __dmul_rn(a, b); }
__device__ __forceinline__ double dadd(double a, double b) { return __dadd_rn(a, b); }
__device__ __forceinline__ double dsub(double a, double b) { return __dsub_rn(a, b); }
__device__ __forceinline__ float fmul(float a, float b) { return __fmul_rn(a, b); }
__device__ __forceinline__ float fadd(float a, float b) { return __fadd_rn(a, b); }

// cv2's float map -> fixed point: cvRound(x * 32)
__device__ __forceinline__ int q32(float x) { return __float2int_rn(fmul(x, 32.f)); }

// ---------------------------------------------------------------------------------------------------- split
struct SplitPano { const uint8_t* img; int H, W, view0; };
struct SplitTable { SplitPano p[MOGE_PANORAMA_MAX_BATCH]; };

// panorama blockIdx.y of the table: img (H, W, 3); its views are out (views, 3, res, res) and out_u8 (views, res, res, 3) (or
// null) from view view0 on
__global__ void __launch_bounds__(kThreads) split_kernel(const __grid_constant__ SplitTable tab, const Cams cams,
                                                         const float* __restrict__ grid, int res, float* __restrict__ out,
                                                         uint8_t* __restrict__ out_u8) {
    const SplitPano& pano = tab.p[blockIdx.y];
    const uint8_t* __restrict__ img = pano.img;
    const int H = pano.H, W = pano.W;
    const int64_t total = static_cast<int64_t>(cams.n) * res * res, first = static_cast<int64_t>(pano.view0) * res * res;
    out += first * 3;
    if (out_u8) out_u8 += first * 3;
    for (int64_t idx = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; idx < total; idx += static_cast<int64_t>(gridDim.x) * blockDim.x) {
        const int k = static_cast<int>(idx / (static_cast<int64_t>(res) * res));
        const int pix = static_cast<int>(idx % (static_cast<int64_t>(res) * res)), i = pix / res, j = pix % res;
        const moge_panorama_camera_t& c = cams.c[k];
        // unproject_cv(uv, 1): ((u - cx) / fx, (v - cy) / fy, 1), then R^T (p - t)
        const double p0 = dsub(__ddiv_rn(dsub(static_cast<double>(grid[j]), c.cx), c.fx), static_cast<double>(c.t[0]));
        const double p1 = dsub(__ddiv_rn(dsub(static_cast<double>(grid[i]), c.cy), c.fy), static_cast<double>(c.t[1]));
        const double p2 = dsub(1.0, static_cast<double>(c.t[2]));
        double d[3];
        for (int r = 0; r < 3; ++r)
            d[r] = dadd(dadd(dmul(c.R[r], p0), dmul(c.R[3 + r], p1)), dmul(c.R[6 + r], p2));
        // directions_to_spherical_uv
        const double nrm = sqrt(dadd(dadd(dmul(d[0], d[0]), dmul(d[1], d[1])), dmul(d[2], d[2])));
        const double x = __ddiv_rn(d[0], nrm), y = __ddiv_rn(d[1], nrm), z = __ddiv_rn(d[2], nrm);
        double a = __ddiv_rn(atan2(y, x), 6.283185307179586), m = fmod(a, 1.0);
        if (m != 0.0) { if (m < 0) m = dadd(m, 1.0); } else m = 0.0;         // numpy's floor-mod: sign of the divisor
        const double u = dsub(1.0, m), v = __ddiv_rn(acos(z), 3.141592653589793);
        // uv_to_pixel, fp32, cv2 fixed point
        const int X = q32(__double2float_rn(dsub(dmul(u, static_cast<double>(W)), 0.5)));
        const int Y = q32(__double2float_rn(dsub(dmul(v, static_cast<double>(H)), 0.5)));
        const int ix = X >> 5, iy = Y >> 5, fx = X & 31, fy = Y & 31;
        const int w[4] = {(32 - fx) * (32 - fy) * 32, fx * (32 - fy) * 32, (32 - fx) * fy * 32, fx * fy * 32};
        int acc[3] = {0, 0, 0};
        for (int t = 0; t < 4; ++t) {
            const int yy = iy + (t >> 1), xx = ix + (t & 1);
            if (yy < 0 || yy >= H || xx < 0 || xx >= W) continue;        // BORDER_CONSTANT 0
            const uint8_t* s = img + (static_cast<int64_t>(yy) * W + xx) * 3;
            for (int ch = 0; ch < 3; ++ch) acc[ch] += w[t] * s[ch];
        }
        for (int ch = 0; ch < 3; ++ch) {
            const int val = min(255, max(0, (acc[ch] + (1 << 14)) >> 15));
            out[((static_cast<int64_t>(k) * 3 + ch) * res + i) * res + j] = __double2float_rn(static_cast<double>(val) / 255.0);
            if (out_u8) out_u8[idx * 3 + ch] = static_cast<uint8_t>(val);
        }
    }
}

// ---------------------------------------------------------------------------------------------------- merge right-hand side
__device__ __forceinline__ float log_distance(const float* __restrict__ src, int channels, int64_t e) {
    if (channels == 1) return logf(src[e]);
    const float* p = src + e * 3;
    return logf(sqrtf(fadd(fadd(fmul(p[0], p[0]), fmul(p[1], p[1])), fmul(p[2], p[2]))));
}

// One merge level of each panorama of a call: its size, its first view in the call's views, its ray table, its sampled maps
// in the workspace and its outputs.
struct LevelSys { const float* dirs; float* L; uint8_t* M; double* b; uint8_t* rm; uint8_t* pmask; int h, w, view0; };
struct LevelTable { LevelSys s[MOGE_PANORAMA_MAX_BATCH]; };

// panorama blockIdx.y of the table, per pixel and view: the sampled log-distance (0 outside the view) and mask.  src
// (call views, vh, vw, channels), vmask (call views, vh, vw); the panorama's L and M (views, h, w)
__global__ void __launch_bounds__(kThreads) sample_kernel(const float* __restrict__ src, int channels, const uint8_t* __restrict__ vmask,
                                                          int vh, int vw, const Cams cams, const __grid_constant__ LevelTable tab) {
    const LevelSys& sys = tab.s[blockIdx.y];
    const int h = sys.h, w = sys.w;
    const float* __restrict__ dirs = sys.dirs;
    float* __restrict__ L = sys.L;
    uint8_t* __restrict__ M = sys.M;
    const int64_t n = static_cast<int64_t>(h) * w;
    const int k0 = sys.view0;                      // the panorama's first view in the call
    for (int64_t p = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; p < n; p += static_cast<int64_t>(gridDim.x) * blockDim.x) {
        const float d0 = dirs[p * 3], d1 = dirs[p * 3 + 1], d2 = dirs[p * 3 + 2];
        for (int k = 0; k < cams.n; ++k) {
            const moge_panorama_camera_t& c = cams.c[k];
            float q[3];
            for (int r = 0; r < 3; ++r) q[r] = fadd(fadd(fadd(fmul(c.R[3 * r], d0), fmul(c.R[3 * r + 1], d1)), fmul(c.R[3 * r + 2], d2)), c.t[r]);
            const double X = q[0], Y = q[1], Z = q[2];
            double u = __ddiv_rn(dadd(dmul(c.fx, X), dmul(c.cx, Z)), Z), v = __ddiv_rn(dadd(dmul(c.fy, Y), dmul(c.cy, Z)), Z);
            const bool valid = q[2] > 0.f && u > 0.0 && v > 0.0 && u < 1.0 && v < 1.0;
            u = fmin(fmax(u, 0.0), 1.0);
            v = fmin(fmax(v, 0.0), 1.0);
            const float px = __double2float_rn(dsub(dmul(u, static_cast<double>(vw)), 0.5));
            const float py = __double2float_rn(dsub(dmul(v, static_cast<double>(vh)), 0.5));
            const int64_t base = static_cast<int64_t>(k0 + k) * vh * vw;
            float val = 0.f;
            uint8_t m = 0;
            if (valid) {
                const int Xq = q32(px), Yq = q32(py), ix = Xq >> 5, iy = Yq >> 5;
                const float ax = static_cast<float>(Xq & 31) / 32.f, ay = static_cast<float>(Yq & 31) / 32.f;
                const float wx[2] = {1.f - ax, ax}, wy[2] = {1.f - ay, ay};
                float acc = 0.f;
                for (int t = 0; t < 4; ++t) {
                    const int yy = min(max(iy + (t >> 1), 0), vh - 1), xx = min(max(ix + (t & 1), 0), vw - 1);
                    acc = fadd(acc, fmul(fmul(wy[t >> 1], wx[t & 1]), log_distance(src, channels, base + static_cast<int64_t>(yy) * vw + xx)));
                }
                val = acc;
                const int nx = min(max(__float2int_rn(px), 0), vw - 1), ny = min(max(__float2int_rn(py), 0), vh - 1);
                m = vmask[base + static_cast<int64_t>(ny) * vw + nx] != 0;
            }
            L[k * n + p] = val;
            M[k * n + p] = m;
        }
    }
}

// panorama blockIdx.y of the table, per pixel: its rows of b and row_mask (see the header) and pano_mask.  The panorama's L
// and M (views, h, w), b and rm (rows), pmask (h, w).  Four blocks per SM, as before the table: its fields would otherwise
// take the kernel past 64 registers.
__global__ void __launch_bounds__(kThreads, 4) rhs_kernel(const __grid_constant__ LevelTable tab, int views) {
    const LevelSys& sys = tab.s[blockIdx.y];
    const int h = sys.h, w = sys.w;
    const float* __restrict__ L = sys.L;
    const uint8_t* __restrict__ M = sys.M;
    double* __restrict__ b = sys.b;
    uint8_t* __restrict__ rm = sys.rm;
    uint8_t* __restrict__ pmask = sys.pmask;
    const int64_t n = static_cast<int64_t>(h) * w;
    for (int64_t p = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; p < n; p += static_cast<int64_t>(gridDim.x) * blockDim.x) {
        const int i = static_cast<int>(p / w), j = static_cast<int>(p % w);
        const int64_t pr = i * static_cast<int64_t>(w) + (j + 1) % w, pl = i * static_cast<int64_t>(w) + (j + w - 1) % w;
        const int64_t pu = static_cast<int64_t>(max(i - 1, 0)) * w + j, pd = static_cast<int64_t>(min(i + 1, h - 1)) * w + j;
        float sx = 0.f, sy = 0.f, sl = 0.f;
        int cx = 0, cy = 0, cl = 0, any = 0;
        for (int k = 0; k < views; ++k) {
            const float* Lk = L + k * n;
            const uint8_t* Mk = M + k * n;
            const float c = Lk[p];
            const int mc = Mk[p], mr = Mk[pr];
            any |= mc;
            const int mx = mc & mr;
            const float gx = fmul(__fsub_rn(c, Lk[pr]), static_cast<float>(mx));
            sx = k ? fadd(sx, gx) : gx;
            cx += mx;
            if (i < h - 1) {
                const int my = mc & Mk[p + w];
                const float gy = fmul(__fsub_rn(c, Lk[p + w]), static_cast<float>(my));
                sy = k ? fadd(sy, gy) : gy;
                cy += my;
            }
            // scipy.ndimage.convolve of the edge / wrap padded map: fp64 taps in footprint order, rounded to fp32
            const double lap = dadd(dadd(dadd(dadd(static_cast<double>(Lk[pu]), static_cast<double>(Lk[pl])), -4.0 * static_cast<double>(c)),
                                         static_cast<double>(Lk[pr])), static_cast<double>(Lk[pd]));
            const int ml = mc & Mk[pu] & Mk[pd] & Mk[pl] & mr;
            const float gl = fmul(__double2float_rn(lap), static_cast<float>(ml));
            sl = k ? fadd(sl, gl) : gl;
            cl += ml;
        }
        b[p] = cx ? __ddiv_rn(static_cast<double>(sx), static_cast<double>(cx)) : 0.0;
        rm[p] = cx > 0;
        if (i < h - 1) {
            const double by = cy ? __ddiv_rn(static_cast<double>(sy), static_cast<double>(cy)) : 0.0;
            const int64_t e = n + static_cast<int64_t>(i) * (w + 1) + j;
            b[e] = by;
            rm[e] = cy > 0;
            if (j == 0) { b[e + w] = by; rm[e + w] = cy > 0; }
        }
        const int64_t lo = n + static_cast<int64_t>(h - 1) * (w + 1);
        b[lo + p] = cl ? __ddiv_rn(static_cast<double>(sl), static_cast<double>(cl)) : 0.0;
        rm[lo + p] = cl > 0;
        pmask[p] = any;
    }
}

// ---------------------------------------------------------------------------------------------------- LSMR
__device__ __forceinline__ double sgn(double a) { return a > 0 ? 1.0 : (a < 0 ? -1.0 : 0.0); }
__device__ void sym_ortho(double a, double b, double* c, double* s, double* r) {
    if (b == 0) { *c = sgn(a); *s = 0; *r = fabs(a); }
    else if (a == 0) { *c = 0; *s = sgn(b); *r = fabs(b); }
    else if (fabs(b) > fabs(a)) { const double tau = a / b; *s = sgn(b) / sqrt(1 + tau * tau); *c = *s * tau; *r = b / *s; }
    else { const double tau = b / a; *c = sgn(a) / sqrt(1 + tau * tau); *s = *c * tau; *r = a / *c; }
}

// (A v) at the dense rows of pixel p: x-gradient, y-gradient (i < h - 1), Laplacian (centre, up, down, left, right)
template <typename T>
__device__ __forceinline__ void apply_rows(const T* v, int64_t p, int i, int j, int h, int w, T* ax, T* ay, T* al) {
    const int64_t pr = i * static_cast<int64_t>(w) + (j + 1) % w, pl = i * static_cast<int64_t>(w) + (j + w - 1) % w;
    const int64_t pu = static_cast<int64_t>(max(i - 1, 0)) * w + j, pd = static_cast<int64_t>(min(i + 1, h - 1)) * w + j;
    *ax = v[p] - v[pr];
    *ay = i < h - 1 ? v[p] - v[p + w] : T(0);
    T s = T(-4) * v[p];
    s = s + v[pu]; s = s + v[pd]; s = s + v[pl]; s = s + v[pr];
    *al = s;
}

// (A^T u) at column p, from the dense rows of u (zero at masked-out rows)
__device__ __forceinline__ double apply_cols(const double* u, int64_t p, int i, int j, int h, int w) {
    const int64_t n = static_cast<int64_t>(h) * w;
    const double* ux = u;
    const double* uy = u + n + static_cast<int64_t>(i) * (w + 1);           // row i of the (h-1) x (w+1) y-gradient rows
    const double* ul = u + n + static_cast<int64_t>(h - 1) * (w + 1);
    const int64_t pr = i * static_cast<int64_t>(w) + (j + 1) % w, pl = i * static_cast<int64_t>(w) + (j + w - 1) % w;
    double s = ux[p] - ux[pl];
    if (i < h - 1) { s += uy[j]; if (j == 0) s += uy[w]; }
    if (i > 0) { s -= uy[j - (w + 1)]; if (j == 0) s -= uy[w - (w + 1)]; }
    s += -4.0 * ul[p];
    if (i + 1 < h) s += ul[p + w]; else s += ul[p];        // rows whose down tap is p
    if (i > 0) s += ul[p - w]; else s += ul[p];            // rows whose up tap is p
    s += ul[pr] + ul[pl];                                  // rows whose left / right tap is p
    return s;
}

// the dense rows of pixel (i, j): x-gradient, y-gradient (i < h - 1) and its repeat at column w (j == 0), Laplacian; the kind
// (0 x, 1 y, 2 Laplacian) selects the row's value in apply_rows
__device__ __forceinline__ int pixel_rows(int64_t p, int i, int j, int h, int w, int64_t* e, int* kind) {
    const int64_t n = static_cast<int64_t>(h) * w;
    int c = 0;
    e[c] = p; kind[c++] = 0;
    if (i < h - 1) {
        const int64_t y = n + static_cast<int64_t>(i) * (w + 1) + j;
        e[c] = y; kind[c++] = 1;
        if (j == 0) { e[c] = y + w; kind[c++] = 1; }
    }
    e[c] = n + static_cast<int64_t>(h - 1) * (w + 1) + p; kind[c++] = 2;
    return c;
}

// P independent systems, each of its own level size, in one cooperative launch, sharing each iteration's four grid barriers
// (the single merge is P = 1).  A system's reductions depend on its own size only, not on P nor on the other systems: its
// pixels are split over `vblocks` virtual blocks of 512 threads, one per SM (at most ceil(n / 512)): virtual block k, thread t
// takes pixels k * 512 + t, stepping by vblocks * 512, reduces them with a warp-shuffle and block tree to the block's partial,
// and the partials are summed in virtual-block order.  The systems' virtual blocks are numbered back to back (system s from
// item0) and dealt to the real blocks in contiguous runs of per_block, so a real block serves at most kMaxLocal systems (the
// host checks it) and evaluates each one's scalar recurrences once, in shared memory.  A system that stops keeps its x and
// stats and does no more work; the launch ends when every system has stopped.
constexpr int kMaxLocal = 4;

struct LsmrSys {
    const double* b; const uint8_t* rm; const float* init;     // b, rm (rows); init (n) = log(init) or null
    float* depth; int32_t* stats;                               // depth (n), stats (2)
    double *u, *v, *hv, *hb, *x, *part;                         // u (rows); v, hv, hb, x (n); part: 2 buffers x vblocks x 2
    int h, w, vblocks, item0;                                   // item0: the system's first virtual block
};
struct LsmrTable {
    LsmrSys s[MOGE_PANORAMA_MAX_BATCH];
    int* stop;                                 // (n): the system has stopped
    int n, items, per_block;
};

// a system's LSMR arrays in its workspace piece, in this order, each padded to 32 doubles: u (rows), v, hv, hb, x (n each),
// then the partials (2 buffers x vblocks x 2)
__host__ __device__ __forceinline__ int64_t pad32(int64_t k) { return (k + 31) & ~int64_t(31); }
__host__ __device__ __forceinline__ int64_t lsmr_rows(int h, int w) { return 2 * static_cast<int64_t>(h) * w + static_cast<int64_t>(h - 1) * (w + 1); }

// the system that virtual block `item` belongs to: the last one whose item0 is <= item
__device__ __forceinline__ int find_system(const LsmrTable& a, int item) {
    int lo = 0, hi = a.n - 1;
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (a.s[mid].item0 <= item) lo = mid; else hi = mid - 1;
    }
    return lo;
}

// one system's scalars: SciPy's lsmr locals, and the tests that do not depend on normx
struct LsmrScalars {
    double normb, maxiter, alpha, beta, zetabar, alphabar, rho, rhobar, cbar, sbar, betadd, betad, rhodold, tautildeold, thetatilde;
    double zeta, d, normA2, maxrbar, minrbar, normar, c1, c2, c3, normA, test1, test2, test3;
    int itn, istop;
    bool done, zero_x;
};

// the block tree of one virtual block: its partial sums of (a, c) to P[0], P[1]
__device__ void block_partial(double a, double c, double* P) {
    __shared__ double2 red[kLsmrThreads / 32];
    for (int o = 16; o > 0; o >>= 1) { a += __shfl_xor_sync(0xffffffffu, a, o); c += __shfl_xor_sync(0xffffffffu, c, o); }
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (lane == 0) red[warp] = make_double2(a, c);
    __syncthreads();
    if (threadIdx.x == 0) {
        double s = 0, t = 0;
        for (int k = 0; k < kLsmrThreads / 32; ++k) { s += red[k].x; t += red[k].y; }
        P[0] = s;
        P[1] = t;
    }
    __syncthreads();
}

// after the barrier: the sum of the `count` partials at P in order (lane-strided, then a warp tree), in every lane of the warp
__device__ double2 partial_sum(const double* P, int count) {
    const int lane = threadIdx.x & 31;
    double s = 0, t = 0;
    for (int k = lane; k < count; k += 32) { s += __ldcg(P + k * 2); t += __ldcg(P + k * 2 + 1); }
    for (int o = 16; o > 0; o >>= 1) { s += __shfl_xor_sync(0xffffffffu, s, o); t += __shfl_xor_sync(0xffffffffu, t, o); }
    return make_double2(s, t);
}

__global__ void __launch_bounds__(kLsmrThreads) lsmr_kernel(const __grid_constant__ LsmrTable a) {
    cg::grid_group g = cg::this_grid();
    __shared__ LsmrScalars S[kMaxLocal];
    const int i0 = blockIdx.x * a.per_block, i1 = min(i0 + a.per_block, a.items);
    const int s0 = find_system(a, i0), nloc = find_system(a, i1 - 1) - s0 + 1;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const bool lead = lane == 0 && warp < nloc;                   // evaluates the scalars of local system `warp`
    const bool owner = warp < nloc && a.s[s0 + warp].item0 >= i0; // this block holds that system's virtual block 0
    const double atol = 1e-5, btol = 1e-5, ctol = 1e-8;
    int buf = 0;
    double2 r = make_double2(0, 0);
#define FOR_ITEMS for (int it = i0; it < i1; ++it)
#define ITEM                                                                                                                 \
    const int sy = find_system(a, it);                                                                                       \
    const LsmrSys& ls = a.s[sy];                                                                                             \
    const int h = ls.h, w = ls.w, vb = it - ls.item0;                                                                        \
    const int64_t n = static_cast<int64_t>(h) * w, stride = static_cast<int64_t>(ls.vblocks) * kLsmrThreads;                 \
    [[maybe_unused]] const bool x32 = ls.init != nullptr;                                                                    \
    [[maybe_unused]] const LsmrScalars& q = S[sy - s0];                                                                      \
    [[maybe_unused]] const double* b = ls.b;                                                                                 \
    [[maybe_unused]] const uint8_t* rm = ls.rm;                                                                              \
    [[maybe_unused]] double *u = ls.u, *v = ls.v, *hv = ls.hv, *hb = ls.hb, *x = ls.x
#define FOR_PIXELS for (int64_t p = vb * static_cast<int64_t>(kLsmrThreads) + threadIdx.x; p < n; p += stride)
#define PIXEL_IJ const int i = static_cast<int>(p / w), j = static_cast<int>(p % w)
#define PARTIAL(v0, v1) block_partial(v0, v1, ls.part + (static_cast<int64_t>(buf) * ls.vblocks + vb) * 2)
#define SUM (r = warp < nloc ? partial_sum(a.s[s0 + warp].part + static_cast<int64_t>(buf) * a.s[s0 + warp].vblocks * 2,       \
                                           a.s[s0 + warp].vblocks)                                                           \
                             : make_double2(0, 0), buf ^= 1)
    // u = b - A x0 or u = b; ||b||, rows in use; ||u|| (into the other buffer)
    FOR_ITEMS {
        ITEM;
        const float* init = ls.init;
        double sb = 0, sm = 0, su = 0;
        FOR_PIXELS {
            PIXEL_IJ;
            float ax = 0, ay = 0, al = 0;
            if (x32) apply_rows<float>(init, p, i, j, h, w, &ax, &ay, &al);
            const float av[3] = {ax, ay, al};
            int64_t es[4];
            int ks[4];
            const int nr = pixel_rows(p, i, j, h, w, es, ks);
            for (int k = 0; k < nr; ++k) {
                const int64_t e = es[k];
                const double bb = rm[e] ? b[e] : 0.0;
                const double uu = rm[e] ? bb - static_cast<double>(av[ks[k]]) : 0.0;
                sb += bb * bb; sm += rm[e]; su += uu * uu;
                u[e] = x32 ? uu : bb;
            }
            x[p] = x32 ? static_cast<double>(init[p]) : 0.0;
            hb[p] = 0.0;
        }
        PARTIAL(sb, sm);
        buf ^= 1; PARTIAL(su, 0); buf ^= 1;
    }
    g.sync();
    SUM;
    if (lead) {
        const LsmrSys& ls = a.s[s0 + warp];
        S[warp].normb = sqrt(r.x);
        S[warp].maxiter = fmin(r.y, static_cast<double>(static_cast<int64_t>(ls.h) * ls.w));
        S[warp].beta = S[warp].normb;
    }
    SUM;
    if (lead && a.s[s0 + warp].init != nullptr) S[warp].beta = sqrt(r.x);
    __syncthreads();
    FOR_ITEMS {
        ITEM;
        if (q.beta > 0) {
            const double ib = 1 / q.beta;
            FOR_PIXELS { PIXEL_IJ; int64_t es[4]; int ks[4]; const int nr = pixel_rows(p, i, j, h, w, es, ks); for (int k = 0; k < nr; ++k) u[es[k]] = ib * u[es[k]]; }
        }
    }
    g.sync();
    FOR_ITEMS {
        ITEM;
        double sv = 0;
        if (q.beta > 0) { FOR_PIXELS { PIXEL_IJ; const double vv = apply_cols(u, p, i, j, h, w); v[p] = vv; sv += vv * vv; } }
        else { FOR_PIXELS v[p] = 0; }
        PARTIAL(sv, 0);
    }
    g.sync();
    SUM;
    if (lead) S[warp].alpha = S[warp].beta > 0 ? sqrt(r.x) : 0.0;
    __syncthreads();
    FOR_ITEMS {
        ITEM;
        const double alpha = q.alpha, ia = alpha > 0 ? 1 / alpha : 1.0;
        FOR_PIXELS { const double vv = alpha > 0 ? ia * v[p] : v[p]; v[p] = vv; hv[p] = vv; }
    }
    if (lead) {
        LsmrScalars& q = S[warp];
        const double alpha = q.alpha, beta = q.beta;
        q.itn = 0; q.istop = 0;
        q.zetabar = alpha * beta; q.alphabar = alpha; q.rho = 1; q.rhobar = 1; q.cbar = 1; q.sbar = 0;
        q.betadd = beta; q.betad = 0; q.rhodold = 1; q.tautildeold = 0; q.thetatilde = 0; q.zeta = 0; q.d = 0;
        q.normA2 = alpha * alpha; q.maxrbar = 0; q.minrbar = 1e100;
        q.normar = alpha * beta;
        q.zero_x = q.normar != 0 && q.normb == 0;
        q.done = q.normar == 0 || q.zero_x || !(q.itn < q.maxiter);
        if (owner) a.stop[s0 + warp] = q.done;
    }
    __syncthreads();
    FOR_ITEMS { ITEM; if (q.zero_x) { FOR_PIXELS x[p] = 0; } }
    g.sync();
    for (;;) {
        // u = -alpha u + A v
        FOR_ITEMS {
            ITEM;
            double s = 0;
            if (!q.done) {
                const double alpha = q.alpha;
                FOR_PIXELS {
                    PIXEL_IJ;
                    double ax, ay, al;
                    apply_rows<double>(v, p, i, j, h, w, &ax, &ay, &al);
                    const double av[3] = {ax, ay, al};
                    int64_t es[4];
                    int ks[4];
                    const int nr = pixel_rows(p, i, j, h, w, es, ks);
                    for (int k = 0; k < nr; ++k) {
                        const int64_t e = es[k];
                        const double uu = rm[e] ? dadd(dmul(u[e], -alpha), av[ks[k]]) : 0.0;
                        u[e] = uu;
                        s += uu * uu;
                    }
                }
            }
            PARTIAL(s, 0);
        }
        g.sync();
        SUM;
        // the stop flags were written before this barrier and are next written after two more
        bool all = true;
        for (int k = lane; k < a.n; k += 32) all = all && __ldcg(a.stop + k) != 0;
        if (__all_sync(0xffffffffu, all)) break;
        if (lead && !S[warp].done) { ++S[warp].itn; S[warp].beta = sqrt(r.x); }
        __syncthreads();
        FOR_ITEMS {
            ITEM;
            if (!q.done && q.beta > 0) {
                const double ib = 1 / q.beta;
                FOR_PIXELS { PIXEL_IJ; int64_t es[4]; int ks[4]; const int nr = pixel_rows(p, i, j, h, w, es, ks); for (int k = 0; k < nr; ++k) u[es[k]] = dmul(u[es[k]], ib); }
            }
        }
        g.sync();
        FOR_ITEMS {
            ITEM;
            double sv = 0;
            if (!q.done && q.beta > 0) {
                const double beta = q.beta;
                FOR_PIXELS { PIXEL_IJ; const double vv = dadd(dmul(v[p], -beta), apply_cols(u, p, i, j, h, w)); v[p] = vv; sv += vv * vv; }
            }
            PARTIAL(sv, 0);
        }
        g.sync();
        SUM;
        if (lead && !S[warp].done) {
            LsmrScalars& q = S[warp];
            const double beta = q.beta;
            if (beta > 0) q.alpha = sqrt(r.x);
            const double alpha = q.alpha;
            double chat, shat, alphahat, c, sn;
            sym_ortho(q.alphabar, 0.0, &chat, &shat, &alphahat);
            const double rhoold = q.rho;
            sym_ortho(alphahat, beta, &c, &sn, &q.rho);
            const double rho = q.rho;
            const double thetanew = sn * alpha;
            q.alphabar = c * alpha;
            const double rhobarold = q.rhobar, zetaold = q.zeta, thetabar = q.sbar * rho, rhotemp = q.cbar * rho;
            sym_ortho(q.cbar * rho, thetanew, &q.cbar, &q.sbar, &q.rhobar);
            const double rhobar = q.rhobar;
            q.zeta = q.cbar * q.zetabar;
            q.zetabar = -q.sbar * q.zetabar;
            q.c1 = -(thetabar * rho / (rhoold * rhobarold)); q.c2 = q.zeta / (rho * rhobar); q.c3 = -(thetanew / rho);
            const double betaacute = chat * q.betadd, betacheck = -shat * q.betadd, betahat = c * betaacute;
            q.betadd = -sn * betaacute;
            const double thetatildeold = q.thetatilde;
            double ctildeold, stildeold, rhotildeold;
            sym_ortho(q.rhodold, thetabar, &ctildeold, &stildeold, &rhotildeold);
            q.thetatilde = stildeold * rhobar;
            q.rhodold = ctildeold * rhobar;
            q.betad = -stildeold * q.betad + ctildeold * betahat;
            q.tautildeold = (zetaold - thetatildeold * q.tautildeold) / rhotildeold;
            const double taud = (q.zeta - q.thetatilde * q.tautildeold) / q.rhodold;
            q.d = q.d + betacheck * betacheck;
            const double normr = sqrt(q.d + (q.betad - taud) * (q.betad - taud) + q.betadd * q.betadd);
            q.normA2 = q.normA2 + beta * beta;
            q.normA = sqrt(q.normA2);
            q.normA2 = q.normA2 + alpha * alpha;
            q.maxrbar = fmax(q.maxrbar, rhobarold);
            if (q.itn > 1) q.minrbar = fmin(q.minrbar, rhobarold);
            const double condA = fmax(q.maxrbar, rhotemp) / fmin(q.minrbar, rhotemp);
            q.normar = fabs(q.zetabar);
            q.test1 = normr / q.normb;
            q.test2 = (q.normA * normr) != 0 ? q.normar / (q.normA * normr) : INFINITY;
            q.test3 = 1 / condA;
        }
        __syncthreads();
        FOR_ITEMS {
            ITEM;
            double sx = 0;
            if (!q.done) {
                const bool scale_v = q.beta > 0 && q.alpha > 0;
                const double ia = scale_v ? 1 / q.alpha : 1.0, c1 = q.c1, c2 = q.c2, c3 = q.c3;
                FOR_PIXELS {
                    const double vv = scale_v ? dmul(v[p], ia) : v[p];
                    v[p] = vv;
                    const double hbv = dadd(dmul(hb[p], c1), hv[p]);
                    hb[p] = hbv;
                    double xx = dadd(x[p], dmul(c2, hbv));
                    if (x32) xx = static_cast<double>(__double2float_rn(xx));
                    x[p] = xx;
                    sx += xx * xx;
                    hv[p] = dadd(dmul(hv[p], c3), vv);
                }
            }
            PARTIAL(sx, 0);
        }
        g.sync();
        SUM;
        if (lead && !S[warp].done) {
            LsmrScalars& q = S[warp];
            double normx = sqrt(r.x);
            if (a.s[s0 + warp].init != nullptr) normx = static_cast<double>(static_cast<float>(normx));
            const double t1 = q.test1 / (1 + q.normA * normx / q.normb);
            const double rtol = btol + atol * q.normA * normx / q.normb;
            int istop = 0;
            if (q.itn >= q.maxiter) istop = 7;
            if (1 + q.test3 <= 1) istop = 6;
            if (1 + q.test2 <= 1) istop = 5;
            if (1 + t1 <= 1) istop = 4;
            if (q.test3 <= ctol) istop = 3;
            if (q.test2 <= atol) istop = 2;
            if (q.test1 <= rtol) istop = 1;
            q.istop = istop;
            q.done = istop > 0 || !(q.itn < q.maxiter);
            if (owner) a.stop[s0 + warp] = q.done;
        }
        __syncthreads();
    }
    FOR_ITEMS { ITEM; float* depth = ls.depth; FOR_PIXELS depth[p] = x32 ? expf(static_cast<float>(x[p])) : __double2float_rn(exp(x[p])); }
    if (lead && owner) { a.s[s0 + warp].stats[0] = S[warp].itn; a.s[s0 + warp].stats[1] = S[warp].istop; }
#undef FOR_ITEMS
#undef ITEM
#undef FOR_PIXELS
#undef PIXEL_IJ
#undef PARTIAL
#undef SUM
}

struct LogMap { const float* src; float* dst; int64_t n; };
struct LogTable { LogMap m[MOGE_PANORAMA_MAX_BATCH]; };

// map blockIdx.y of the table: dst = log(src)
__global__ void log_kernel(const __grid_constant__ LogTable tab) {
    const LogMap& m = tab.m[blockIdx.y];
    const float* __restrict__ src = m.src;
    float* __restrict__ dst = m.dst;
    for (int64_t p = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; p < m.n; p += static_cast<int64_t>(gridDim.x) * blockDim.x)
        dst[p] = logf(src[p]);
}

// ---------------------------------------------------------------------------------------------------- resizes and points
// cv2.resize INTER_LINEAR source coordinate of output index d: fp32 (d + 0.5) * in / out - 0.5, clamped at the borders
__device__ __forceinline__ void lin_coef(int d, int in, int out, int* s0, int* s1, float* f) {
    float fx = static_cast<float>((d + 0.5) * (1.0 / (static_cast<double>(out) / in)) - 0.5);
    int sx = static_cast<int>(floorf(fx));
    fx -= static_cast<float>(sx);
    if (sx < 0) { fx = 0.f; sx = 0; }
    if (sx >= in - 1) { fx = 0.f; sx = in - 1; }
    *s0 = sx; *s1 = min(sx + 1, in - 1); *f = fx;
}

struct ResizeMap { const float* src; float* dst; int h, w, H, W; };
struct ResizeTable { ResizeMap m[MOGE_PANORAMA_MAX_BATCH]; };

// map blockIdx.y of the table: src (h, w) -> dst (H, W)
__global__ void __launch_bounds__(kThreads) resize_kernel(const __grid_constant__ ResizeTable tab) {
    const ResizeMap& m = tab.m[blockIdx.y];
    const float* __restrict__ src = m.src;
    float* __restrict__ dst = m.dst;
    const int h = m.h, w = m.w, H = m.H, W = m.W;
    const int64_t n = static_cast<int64_t>(H) * W;
    for (int64_t p = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; p < n; p += static_cast<int64_t>(gridDim.x) * blockDim.x) {
        const int i = static_cast<int>(p / W), j = static_cast<int>(p % W);
        int x0, x1, y0, y1;
        float fx, fy;
        lin_coef(j, w, W, &x0, &x1, &fx);
        lin_coef(i, h, H, &y0, &y1, &fy);
        const float* r0 = src + static_cast<int64_t>(y0) * w;
        const float* r1 = src + static_cast<int64_t>(y1) * w;
        const float a0 = 1.f - fx, b0 = 1.f - fy;
        const float h0 = fadd(fmul(r0[x0], a0), fmul(r0[x1], fx)), h1 = fadd(fmul(r1[x0], a0), fmul(r1[x1], fx));
        dst[p] = fadd(fmul(h0, b0), fmul(h1, fy));
    }
}

// cv2.resize INTER_LINEAR of a 0/1 uint8 mask (11-bit fixed-point coefficients), then > 0; and points = depth * direction.
// Panorama blockIdx.y of the table: depth (H, W) (already resized), mask (h, w), mask_out (H, W), points (H, W, 3)
struct FinishMap { const float* depth; const uint8_t* mask; uint8_t* mask_out; float* points; int h, w, H, W; };
struct FinishTable { FinishMap m[MOGE_PANORAMA_MAX_BATCH]; };

__global__ void __launch_bounds__(kThreads) finish_kernel(const __grid_constant__ FinishTable tab) {
    const FinishMap& m = tab.m[blockIdx.y];
    const float* __restrict__ depth = m.depth;
    const uint8_t* __restrict__ mask = m.mask;
    uint8_t* __restrict__ mask_out = m.mask_out;
    float* __restrict__ points = m.points;
    const int h = m.h, w = m.w, H = m.H, W = m.W;
    const int64_t n = static_cast<int64_t>(H) * W;
    // uv_map's linspace ends and steps
    const double su = 0.5 / W, eu = 1.0 - 0.5 / W, sv = 0.5 / H, ev = 1.0 - 0.5 / H;
    const double stu = W > 1 ? (eu - su) / (W - 1) : 0.0, stv = H > 1 ? (ev - sv) / (H - 1) : 0.0;
    for (int64_t p = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; p < n; p += static_cast<int64_t>(gridDim.x) * blockDim.x) {
        const int i = static_cast<int>(p / W), j = static_cast<int>(p % W);
        int x0, x1, y0, y1;
        float fx, fy;
        lin_coef(j, w, W, &x0, &x1, &fx);
        lin_coef(i, h, H, &y0, &y1, &fy);
        const int a1 = __float2int_rn(fx * 2048.f), a0 = __float2int_rn((1.f - fx) * 2048.f);
        const int b1 = __float2int_rn(fy * 2048.f), b0 = __float2int_rn((1.f - fy) * 2048.f);
        const uint8_t* m0 = mask + static_cast<int64_t>(y0) * w;
        const uint8_t* m1 = mask + static_cast<int64_t>(y1) * w;
        const int r0 = (m0[x0] != 0) * a0 + (m0[x1] != 0) * a1, r1 = (m1[x0] != 0) * a0 + (m1[x1] != 0) * a1;
        const int val = (((b0 * (r0 >> 4)) >> 16) + ((b1 * (r1 >> 4)) >> 16) + 2) >> 2;
        mask_out[p] = val > 0;
        // uv_map(H, W) (np.linspace in fp64, rounded to fp32) and spherical_uv_to_directions in fp32
        const float u = j == W - 1 ? __double2float_rn(eu) : __double2float_rn(dadd(dmul(static_cast<double>(j), stu), su));
        const float v = i == H - 1 ? __double2float_rn(ev) : __double2float_rn(dadd(dmul(static_cast<double>(i), stv), sv));
        const float theta = fmul(1.f - u, 6.28318530717958647692f), phi = fmul(v, 3.14159265358979323846f);
        const float sp = sinf(phi), d = depth[p];
        points[p * 3] = fmul(d, fmul(sp, cosf(theta)));
        points[p * 3 + 1] = fmul(d, fmul(sp, sinf(theta)));
        points[p * 3 + 2] = fmul(d, cosf(phi));
    }
}

// ---------------------------------------------------------------------------------------------------- host side
int check_size(const char* what, int h, int w) {
    if (h < 2 || w < 2) return set_error("%s: a %d x %d map is too small (at least 2 x 2)", what, h, w);
    if (static_cast<int64_t>(h) * w > kMaxPixels) return set_error("%s: a %d x %d map is too large (at most 2^28 pixels)", what, h, w);
    return 0;
}

int load_cams(const char* what, const moge_panorama_camera_t* cams, int views, Cams* out) {
    if (!cams) return set_error("%s: null cameras", what);
    if (views < 1 || views > MOGE_PANORAMA_MAX_VIEWS) return set_error("%s: %d views is outside [1, %d]", what, views, MOGE_PANORAMA_MAX_VIEWS);
    memset(out, 0, sizeof(*out));
    for (int k = 0; k < views; ++k) {
        const moge_panorama_camera_t& c = cams[k];
        if (!(c.fx != 0) || !(c.fy != 0)) return set_error("%s: view %d has a zero focal length", what, k);
        out->c[k] = c;
    }
    out->n = views;
    return 0;
}

unsigned blocks_for(int64_t n, int sms) { return static_cast<unsigned>(std::min<int64_t>((n + kThreads - 1) / kThreads, int64_t(sms) * 16)); }

// an entry's name in messages: the operation's and the entry's index
struct Name {
    char s[96];
    Name(const char* what, int k) { snprintf(s, sizeof(s), "%s: panorama %d", what, k); }
};

int null_argument(const Name& nm) { return set_error("%s: null argument", nm.s); }

int check_batch(const char* what, int batch) {
    if (batch < 1 || batch > MOGE_PANORAMA_MAX_BATCH)
        return set_error("%s: a batch of %d panoramas is outside [1, %d]", what, batch, MOGE_PANORAMA_MAX_BATCH);
    return 0;
}

// the workspace of one call's merges: per system its sampled maps L and M, its LSMR arrays (see LsmrSys) and log(init);
// then the call's stop flags.  Nothing in it outlives a call, and a call whose levels are each no larger fits in the workspace
// of a bigger one, so the workspace of a pyramid's finest levels serves every coarser level.
constexpr int kMaxLsmrBlocks = 132 * 4;            // virtual blocks per system
struct SysLayout { size_t L, M, lsmr, logi; };
struct Layout { SysLayout s[MOGE_PANORAMA_MAX_BATCH]; size_t stop, total; };
int max_vblocks(int64_t n) { return static_cast<int>(std::min<int64_t>((n + kLsmrThreads - 1) / kLsmrThreads, kMaxLsmrBlocks)); }
Layout layout(int views, const moge_panorama_level_t* lv, int count) {
    WsLayout ws;
    Layout l;
    for (int k = 0; k < count; ++k) {
        const int h = lv[k].h, w = lv[k].w;
        const size_t n = static_cast<size_t>(h) * w;
        l.s[k].L = ws.add(views * n * 4);
        l.s[k].M = ws.add(views * n);
        l.s[k].lsmr = ws.add((pad32(lsmr_rows(h, w)) + 4 * pad32(n) + 4 * max_vblocks(n)) * 8);
        l.s[k].logi = ws.add(n * 4);
    }
    l.stop = ws.add(static_cast<size_t>(count) * 4);
    l.total = ws.total;
    return l;
}

int check_levels(const char* what, const moge_panorama_level_t* lv, int count) {
    if (!lv) return set_error("null argument");
    MG_TRY(check_batch(what, count));
    for (int k = 0; k < count; ++k) MG_TRY(check_size(Name(what, k).s, lv[k].h, lv[k].w));
    return 0;
}

int workspace_bytes(const char* what, const moge_panorama_level_t* lv, int count, int views, size_t* bytes) {
    if (!bytes) return set_error("null argument");
    MG_TRY(check_levels(what, lv, count));
    if (views < 1 || views > MOGE_PANORAMA_MAX_VIEWS) return set_error("%s: %d views is outside [1, %d]", what, views, MOGE_PANORAMA_MAX_VIEWS);
    *bytes = layout(views, lv, count).total;
    return 0;
}

int split(const char* what, const moge_panorama_split_t* panos, int count, const moge_panorama_camera_t* cams, int views,
          const float* grid, int res, float* views_f32, uint8_t* views_u8, void* stream) {
    if (!panos || !grid || !views_f32) return set_error("null argument");
    MG_TRY(check_batch(what, count));
    SplitTable tab{};
    for (int k = 0; k < count; ++k) {
        const Name nm(what, k);
        if (!panos[k].image) return null_argument(nm);
        MG_TRY(check_size(nm.s, panos[k].H, panos[k].W));
        if (panos[k].view0 < 0) return set_error("%s: first view %d is negative", nm.s, panos[k].view0);
        tab.p[k] = {panos[k].image, panos[k].H, panos[k].W, panos[k].view0};
    }
    if (res < 1 || res > 8192) return set_error("%s: resolution %d is outside [1, 8192]", what, res);
    Cams cs;
    MG_TRY(load_cams(what, cams, views, &cs));
    int sms;
    MG_TRY(check_device(what, &sms));
    split_kernel<<<dim3(blocks_for(static_cast<int64_t>(views) * res * res, sms), count), kThreads, 0, static_cast<cudaStream_t>(stream)>>>(
        tab, cs, grid, res, views_f32, views_u8);
    CUDA_TRY(cudaGetLastError());
    return 0;
}

int rhs(const char* what, const float* src, int channels, const uint8_t* mask, int views, int vh, int vw,
        const moge_panorama_camera_t* cams, const moge_panorama_level_t* lv, int count, void* workspace, size_t workspace_bytes,
        void* stream) {
    if (!src || !mask) return set_error("null argument");
    if (channels != 1 && channels != 3) return set_error("%s: %d channels (1: distance, 3: points)", what, channels);
    MG_TRY(check_levels(what, lv, count));
    for (int k = 0; k < count; ++k) {
        const Name nm(what, k);
        if (!lv[k].directions || !lv[k].b || !lv[k].row_mask || !lv[k].pano_mask) return null_argument(nm);
        if (lv[k].view0 < 0) return set_error("%s: first view %d is negative", nm.s, lv[k].view0);
    }
    char vname[112];
    snprintf(vname, sizeof(vname), "%s view", what);
    MG_TRY(check_size(vname, vh, vw));
    Cams cs;
    MG_TRY(load_cams(what, cams, views, &cs));
    const Layout l = layout(views, lv, count);
    MG_TRY(check_workspace(l.total, workspace, workspace_bytes, what));
    int sms;
    MG_TRY(check_device(what, &sms));
    char* ws = static_cast<char*>(workspace);
    LevelTable tab{};
    int64_t most = 0;
    for (int k = 0; k < count; ++k) {
        const moge_panorama_level_t& e = lv[k];
        tab.s[k] = {e.directions, reinterpret_cast<float*>(ws + l.s[k].L), reinterpret_cast<uint8_t*>(ws + l.s[k].M), e.b, e.row_mask,
                    e.pano_mask, e.h, e.w, e.view0};
        most = std::max<int64_t>(most, static_cast<int64_t>(e.h) * e.w);
    }
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const dim3 grid(blocks_for(most, sms), count);
    sample_kernel<<<grid, kThreads, 0, st>>>(src, channels, mask, vh, vw, cs, tab);
    CUDA_TRY(cudaGetLastError());
    rhs_kernel<<<grid, kThreads, 0, st>>>(tab, views);
    CUDA_TRY(cudaGetLastError());
    return 0;
}

// the LSMR solves of `count` systems: the virtual partition, the real grid over at most the co-resident blocks, the launch
int lsmr(const char* what, const moge_panorama_level_t* lv, int count, void* workspace, size_t workspace_bytes, void* stream) {
    MG_TRY(check_levels(what, lv, count));
    for (int k = 0; k < count; ++k)
        if (!lv[k].b || !lv[k].row_mask || !lv[k].depth || !lv[k].stats) return null_argument(Name(what, k));
    const Layout l = layout(1, lv, count);
    MG_TRY(check_workspace(l.total, workspace, workspace_bytes, what));
    int sms, dev = 0, coop = 0, per_sm = 0;
    MG_TRY(check_device(what, &sms));
    CUDA_TRY(cudaGetDevice(&dev));
    CUDA_TRY(cudaDeviceGetAttribute(&coop, cudaDevAttrCooperativeLaunch, dev));
    if (!coop) return set_error("%s: the device does not support cooperative launches", what);
    CUDA_TRY(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, lsmr_kernel, kLsmrThreads, 0));
    if (per_sm < 1) return set_error("%s: the solver kernel does not fit on an SM", what);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    char* ws = static_cast<char*>(workspace);
    LsmrTable a{};
    LogTable logs{};
    int items = 0, nlog = 0;
    int64_t most = 0;
    for (int k = 0; k < count; ++k) {
        const moge_panorama_level_t& e = lv[k];
        const int64_t n = static_cast<int64_t>(e.h) * e.w;
        const int vblocks = std::min(sms, max_vblocks(n));
        const float* init = nullptr;
        if (e.init) {                                // x0 = log(init), fp32
            float* logi = reinterpret_cast<float*>(ws + l.s[k].logi);
            logs.m[nlog++] = {e.init, logi, n};
            most = std::max(most, n);
            init = logi;
        }
        double* u = reinterpret_cast<double*>(ws + l.s[k].lsmr);
        double* v = u + pad32(lsmr_rows(e.h, e.w));
        a.s[k] = {e.b, e.row_mask, init, e.depth, e.stats, u, v, v + pad32(n), v + 2 * pad32(n), v + 3 * pad32(n), v + 4 * pad32(n),
                  e.h, e.w, vblocks, items};
        items += vblocks;
    }
    const int resident = sms * per_sm;
    const int per_block = (items + resident - 1) / resident, blocks = (items + per_block - 1) / per_block;
    for (int b = 0, s0 = 0; b < blocks; ++b) {       // the systems of each real block's run of virtual blocks
        const int i0 = b * per_block, i1 = std::min(i0 + per_block, items);
        while (s0 + 1 < count && a.s[s0 + 1].item0 <= i0) ++s0;
        int s1 = s0;
        while (s1 + 1 < count && a.s[s1 + 1].item0 <= i1 - 1) ++s1;
        if (s1 - s0 + 1 > kMaxLocal)
            return set_error("%s: a block would serve more than %d systems (%d virtual blocks per block)", what, kMaxLocal, per_block);
    }
    a.stop = reinterpret_cast<int*>(ws + l.stop);
    a.n = count; a.items = items; a.per_block = per_block;
    if (nlog) {
        log_kernel<<<dim3(blocks_for(most, sms), nlog), kThreads, 0, st>>>(logs);
        CUDA_TRY(cudaGetLastError());
    }
    void* args[] = {&a};
    CUDA_TRY(cudaLaunchCooperativeKernel(reinterpret_cast<void*>(lsmr_kernel), dim3(blocks), dim3(kLsmrThreads), args, 0, st));
    return 0;
}

int resize(const char* what, const moge_panorama_resize_t* maps, int count, void* stream) {
    if (!maps) return set_error("null argument");
    MG_TRY(check_batch(what, count));
    ResizeTable tab{};
    int64_t most = 0;
    for (int k = 0; k < count; ++k) {
        const Name nm(what, k);
        const moge_panorama_resize_t& m = maps[k];
        if (!m.src || !m.dst) return null_argument(nm);
        MG_TRY(check_size(nm.s, m.h, m.w));
        MG_TRY(check_size(nm.s, m.H, m.W));
        tab.m[k] = {m.src, m.dst, m.h, m.w, m.H, m.W};
        most = std::max<int64_t>(most, static_cast<int64_t>(m.H) * m.W);
    }
    int sms;
    MG_TRY(check_device(what, &sms));
    resize_kernel<<<dim3(blocks_for(most, sms), count), kThreads, 0, static_cast<cudaStream_t>(stream)>>>(tab);
    CUDA_TRY(cudaGetLastError());
    return 0;
}

int finish(const char* what, const moge_panorama_finish_t* maps, int count, void* stream) {
    if (!maps) return set_error("null argument");
    MG_TRY(check_batch(what, count));
    ResizeTable rt{};
    FinishTable ft{};
    int64_t most = 0;
    for (int k = 0; k < count; ++k) {
        const Name nm(what, k);
        const moge_panorama_finish_t& m = maps[k];
        if (!m.depth || !m.mask || !m.depth_out || !m.mask_out || !m.points) return null_argument(nm);
        MG_TRY(check_size(nm.s, m.h, m.w));
        MG_TRY(check_size(nm.s, m.H, m.W));
        rt.m[k] = {m.depth, m.depth_out, m.h, m.w, m.H, m.W};
        ft.m[k] = {m.depth_out, m.mask, m.mask_out, m.points, m.h, m.w, m.H, m.W};
        most = std::max<int64_t>(most, static_cast<int64_t>(m.H) * m.W);
    }
    int sms;
    MG_TRY(check_device(what, &sms));
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const dim3 grid(blocks_for(most, sms), count);
    resize_kernel<<<grid, kThreads, 0, st>>>(rt);
    CUDA_TRY(cudaGetLastError());
    finish_kernel<<<grid, kThreads, 0, st>>>(ft);
    CUDA_TRY(cudaGetLastError());
    return 0;
}

}  // namespace
}  // namespace mg

using namespace mg;

extern "C" {

int moge_panorama_split_groups(const moge_panorama_split_t* panos, int n, const moge_panorama_camera_t* cams, int views, const float* grid,
                               int res, float* views_f32, uint8_t* views_u8, void* stream) {
    return split("panorama_split_groups", panos, n, cams, views, grid, res, views_f32, views_u8, stream);
}

int moge_panorama_workspace_bytes_groups(const moge_panorama_level_t* levels, int n, int views, size_t* bytes) {
    return workspace_bytes("panorama_workspace_bytes_groups", levels, n, views, bytes);
}

int moge_panorama_rhs_groups(const float* src, int channels, const uint8_t* mask, int views, int vh, int vw,
                             const moge_panorama_camera_t* cams, const moge_panorama_level_t* levels, int n, void* workspace,
                             size_t workspace_bytes, void* stream) {
    return rhs("panorama_rhs_groups", src, channels, mask, views, vh, vw, cams, levels, n, workspace, workspace_bytes, stream);
}

int moge_panorama_lsmr_groups(const moge_panorama_level_t* levels, int n, void* workspace, size_t workspace_bytes, void* stream) {
    return lsmr("panorama_lsmr_groups", levels, n, workspace, workspace_bytes, stream);
}

int moge_panorama_resize_groups(const moge_panorama_resize_t* maps, int n, void* stream) {
    return resize("panorama_resize_groups", maps, n, stream);
}

int moge_panorama_finish_groups(const moge_panorama_finish_t* maps, int n, void* stream) {
    return finish("panorama_finish_groups", maps, n, stream);
}

}  // extern "C"
