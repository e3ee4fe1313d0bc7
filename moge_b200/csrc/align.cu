// Truncated-L1 alignment solvers (moge/utils/alignment.py:52-214, 233-355, 399-416 of the reference).
//
// One problem is n elements (x, y, w), w >= 0.  After flipping signs so that x >= 0 the candidates are A_i = y_i / max(x_i, 1e-7).
//   untruncated: a = the lower weighted median of A with weights w x (first sorted position with 2 prefix(wx) - sum(wx) >= 0).
//   truncated:   f(a) = sum_i min(t_i, |a wx_i - wy_i|) is piecewise linear with kinks at B_i = (wy - t)/max(wx, 1e-7), A_i and
//                C_i = (wy + t)/max(wx, 1e-7).  With S_X(a) = sums over the breakpoints X_i <= a,
//                    f(a)     = sum t - S_B(t) + S_C(t) + S_B(wy) - 2 S_A(wy) + S_C(wy) + a (2 S_A(wx) - S_B(wx) - S_C(wx)),
//                and the slope just left (right) of a is the last bracket summed over X_i < a (X_i <= a).  The candidates are the A_j with
//                left slope < 0 and right slope >= 0; the answer is the one with the least f (element 0 when there is none).
// Keys are computed in fp32 exactly as the reference computes them (no contraction), so the breakpoints and candidate sets are the
// reference's; prefix sums and objective values are fp64 with exact products w*x, w*y.
//
// A CTA solves one problem at a time: it writes the m keys as order-preserving uint32 packed with the element index into shared
// memory, sorts them with a bitonic network (positions >= m act as +inf and are never stored), and scans in sorted order.  The
// truncated solver sorts A, B and C one after the other; per sorted array it writes the prefix sums to a per-CTA scratch in global
// memory and each candidate accumulates its terms there (the arrays do not fit in shared memory together at m = 12288).
// Anchored problems (alignment.py:163-214, 251-355) form x = src - src_p, y = tgt - tgt_p on the fly from the image, staged once per
// CTA in shared memory; each image keeps the least (loss, anchor, index) through a packed 64-bit atomicMin.
#include "common.cuh"
#include "host_api.h"
#include "../../include/moge_b200.h"
#include <math.h>
#include <stdint.h>
#include <algorithm>

namespace mg {
namespace {

constexpr int kThreads = 512;
constexpr int kWarps = kThreads / 32;
constexpr int kMaxPoints = 4096;              // anchored problems: points per image
constexpr int kMaxElems = 3 * kMaxPoints;     // elements per problem
constexpr float kEps = 1e-7f;
constexpr uint64_t kEmptySlot = ~0ull;
// dynamic shared memory of the largest problem: sort buffer + staged points image (src, tgt: 3 floats per point, w)
constexpr size_t kMaxSmem = static_cast<size_t>(kMaxElems) * 8 + (2 * static_cast<size_t>(kMaxElems) + kMaxPoints) * 4;
// block reduction scratch: kWarps doubles, then kWarps + 1 Prefix (block_scan), then one double
constexpr int kRed = kWarps + 3 * (kWarps + 1) + 1;

struct Prefix { double wx, wy, t; };

// the reference's `sign(x)` flip; x == 0 zeroes y as x * sign(x), y * sign(x) does
struct Elem { float x, y, w, t; };
__device__ __forceinline__ Elem flip(float x, float y, float w, float t) {
    if (x < 0.f) return {-x, -y, w, t};
    if (x > 0.f) return {x, y, w, t};
    return {0.f, 0.f, w, t};
}

// Where the elements of the problem come from: plain rows in global memory, or an image staged in shared memory minus its anchor.
struct Source {
    int mode;                 // MOGE_ALIGN_PLAIN or MOGE_ANCHOR_*
    const float* x;           // plain: this problem's rows; anchored: staged src (n * comps)
    const float* y;           //                              staged tgt
    const float* w;           //                              staged weight (n)
    const float* t;           // plain: per-element trunc row or null
    float ts;                 // scalar trunc
    float ax[3], ay[3];       // anchor offsets per component
    __device__ __forceinline__ Elem get(int e) const {
        if (mode == MOGE_ALIGN_PLAIN) return flip(x[e], y[e], w[e], t ? t[e] : ts);
        if (mode == MOGE_ANCHOR_DEPTH) return flip(__fsub_rn(x[e], ax[0]), __fsub_rn(y[e], ay[0]), w[e], ts);
        const int c = e % 3;
        const float ox = c == 0 ? ax[0] : (c == 1 ? ax[1] : ax[2]), oy = c == 0 ? ay[0] : (c == 1 ? ay[1] : ay[2]);
        return flip(__fsub_rn(x[e], ox), __fsub_rn(y[e], oy), w[e / 3], ts);
    }
};

// breakpoint `which` (0 = A, 1 = B, 2 = C) of an element, in the reference's fp32 arithmetic
__device__ __forceinline__ float breakpoint(const Elem& v, int which) {
    if (which == 0) return __fdiv_rn(v.y, fmaxf(v.x, kEps));
    const float wx = __fmul_rn(v.w, v.x), wy = __fmul_rn(v.w, v.y);
    return __fdiv_rn(which == 1 ? __fsub_rn(wy, v.t) : __fadd_rn(wy, v.t), fmaxf(wx, kEps));
}

// Bitonic sort of buf[0, m) ascending, every stage ascending (the first half-cleaner of a merge compares mirrored positions).
__device__ void sort_keys(uint64_t* buf, int m) {
    int p2 = 1;
    while (p2 < m) p2 <<= 1;
    for (int k = 2; k <= p2; k <<= 1) {
        for (int j = k >> 1; j > 0; j >>= 1) {
            for (int q = threadIdx.x; q < (p2 >> 1); q += blockDim.x) {
                const int i = 2 * j * (q / j) + (q % j);
                const int l = (j == (k >> 1)) ? (i ^ (k - 1)) : (i + j);
                if (l < m) {
                    const uint64_t a = buf[i], b = buf[l];
                    if (a > b) { buf[i] = b; buf[l] = a; }
                }
            }
            __syncthreads();
        }
    }
}

// Exclusive block scan of one Prefix per thread (in thread order); red holds kWarps + 1 entries.
__device__ Prefix block_scan(Prefix v, Prefix* red) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    Prefix inc = v;
    for (int o = 1; o < 32; o <<= 1) {
        const double a = __shfl_up_sync(0xffffffffu, inc.wx, o), b = __shfl_up_sync(0xffffffffu, inc.wy, o),
                     c = __shfl_up_sync(0xffffffffu, inc.t, o);
        if (lane >= o) { inc.wx += a; inc.wy += b; inc.t += c; }
    }
    __syncthreads();
    if (lane == 31) red[warp] = inc;
    __syncthreads();
    Prefix base = {0.0, 0.0, 0.0};
    for (int i = 0; i < warp; ++i) { base.wx += red[i].wx; base.wy += red[i].wy; base.t += red[i].t; }
    return {base.wx + inc.wx - v.wx, base.wy + inc.wy - v.wy, base.t + inc.t - v.t};
}

// count of keys < k (upper = false) or <= k (upper = true) in the sorted buffer
__device__ __forceinline__ int rank_of(const uint64_t* buf, int m, uint32_t k, bool upper) {
    int lo = 0, hi = m;
    while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        const uint32_t km = static_cast<uint32_t>(buf[mid] >> 32);
        if (upper ? (km <= k) : (km < k)) lo = mid + 1; else hi = mid;
    }
    return lo;
}

struct Result { double loss; int index; };

// Untruncated: the lower weighted median of A.  Every thread returns the result.
__device__ __forceinline__ Result solve_median(const Source src, int m, uint64_t* buf, double* red, int* pick) {
    double total = 0.0;
    for (int e = threadIdx.x; e < m; e += blockDim.x) {
        const Elem v = src.get(e);
        buf[e] = (static_cast<uint64_t>(order_key(breakpoint(v, 0))) << 32) | static_cast<uint32_t>(e);
        total += static_cast<double>(v.w) * v.x;
    }
    if (threadIdx.x == 0) *pick = m - 1;
    total = block_sum<kThreads>(total, red);       // its leading __syncthreads also publishes buf
    sort_keys(buf, m);
    // contiguous chunk per thread: local sums, scan of the chunk totals, then the first position with 2 prefix - total >= 0
    const int chunk = (m + blockDim.x - 1) / blockDim.x, c0 = min(m, static_cast<int>(threadIdx.x) * chunk), c1 = min(m, c0 + chunk);
    Prefix mine = {0.0, 0.0, 0.0};
    for (int p = c0; p < c1; ++p) {
        const Elem v = src.get(static_cast<uint32_t>(buf[p]));
        mine.wx += static_cast<double>(v.w) * v.x;
    }
    Prefix* scan_red = reinterpret_cast<Prefix*>(red + kWarps);
    double run = block_scan(mine, scan_red).wx;
    for (int p = c0; p < c1; ++p) {
        const Elem v = src.get(static_cast<uint32_t>(buf[p]));
        run += static_cast<double>(v.w) * v.x;
        if (2.0 * run - total >= 0.0) { atomicMin(pick, p); break; }
    }
    __syncthreads();
    const uint64_t chosen = buf[*pick];
    const float a = key_value(static_cast<uint32_t>(chosen >> 32));
    double loss = 0.0;
    for (int e = threadIdx.x; e < m; e += blockDim.x) {
        const Elem v = src.get(e);
        loss += static_cast<double>(v.w) * fabs(static_cast<double>(a) * v.x - v.y);
    }
    loss = block_sum<kThreads>(loss, red);
    __syncthreads();                     // buf and *pick are rewritten by the next problem
    return {loss, static_cast<int>(static_cast<uint32_t>(chosen))};
}

// Truncated: candidates and objective from three sorted passes.  acc: 3 m doubles (per-candidate slope left/right and constant
// term), pre: 3 (m + 1) doubles (prefix sums of the sorted pass).  Every thread returns the result.
__device__ __forceinline__ Result solve_truncated(const Source src, int m, uint64_t* buf, double* red, double* acc, Prefix* pre) {
    double* sl = acc;
    double* sr = acc + m;
    double* cst = acc + 2 * m;
    double t_total = 0.0;
    for (int pass = 0; pass < 3; ++pass) {
        for (int e = threadIdx.x; e < m; e += blockDim.x) {
            const Elem v = src.get(e);
            buf[e] = (static_cast<uint64_t>(order_key(breakpoint(v, pass))) << 32) | static_cast<uint32_t>(e);
            if (pass == 0) t_total += v.t;
        }
        __syncthreads();
        sort_keys(buf, m);
        const int chunk = (m + blockDim.x - 1) / blockDim.x, c0 = min(m, static_cast<int>(threadIdx.x) * chunk), c1 = min(m, c0 + chunk);
        Prefix mine = {0.0, 0.0, 0.0};
        for (int p = c0; p < c1; ++p) {
            const Elem v = src.get(static_cast<uint32_t>(buf[p]));
            mine.wx += static_cast<double>(v.w) * v.x; mine.wy += static_cast<double>(v.w) * v.y; mine.t += v.t;
        }
        Prefix run = block_scan(mine, reinterpret_cast<Prefix*>(red + kWarps));
        if (threadIdx.x == 0) pre[0] = {0.0, 0.0, 0.0};
        for (int p = c0; p < c1; ++p) {
            const Elem v = src.get(static_cast<uint32_t>(buf[p]));
            run.wx += static_cast<double>(v.w) * v.x; run.wy += static_cast<double>(v.w) * v.y; run.t += v.t;
            pre[p + 1] = run;
        }
        __syncthreads();
        for (int j = threadIdx.x; j < m; j += blockDim.x) {
            const uint32_t k = order_key(breakpoint(src.get(j), 0));
            const Prefix lo = pre[rank_of(buf, m, k, false)], hi = pre[rank_of(buf, m, k, true)];
            if (pass == 0) {
                sl[j] = 2.0 * lo.wx; sr[j] = 2.0 * hi.wx; cst[j] = -2.0 * hi.wy;
            } else {
                sl[j] -= lo.wx; sr[j] -= hi.wx;
                cst[j] += (pass == 1 ? -hi.t : hi.t) + hi.wy;
            }
        }
        __syncthreads();
    }
    t_total = block_sum<kThreads>(t_total, red);
    // least f over the candidates, ties to the smaller element; element 0 when there is no candidate
    double best = INFINITY, f0 = 0.0;
    int best_j = m;
    for (int j = threadIdx.x; j < m; j += blockDim.x) {
        const double a = breakpoint(src.get(j), 0);
        const double f = t_total + cst[j] + a * sr[j];
        if (j == 0) f0 = f;
        if (sl[j] < 0.0 && sr[j] >= 0.0 && (f < best || (f == best && j < best_j))) { best = f; best_j = j; }
    }
    for (int o = 16; o > 0; o >>= 1) {
        const double fb = __shfl_xor_sync(0xffffffffu, best, o);
        const int jb = __shfl_xor_sync(0xffffffffu, best_j, o);
        if (fb < best || (fb == best && jb < best_j)) { best = fb; best_j = jb; }
    }
    __syncthreads();
    double* fr = red;
    int* jr = reinterpret_cast<int*>(red + kWarps);
    if ((threadIdx.x & 31) == 0) { fr[threadIdx.x >> 5] = best; jr[threadIdx.x >> 5] = best_j; }
    if (threadIdx.x == 0) red[kRed - 1] = f0;
    __syncthreads();
    for (int i = 0; i < kWarps; ++i)
        if (fr[i] < best || (fr[i] == best && jr[i] < best_j)) { best = fr[i]; best_j = jr[i]; }
    if (best_j == m) { best = red[kRed - 1]; best_j = 0; }
    __syncthreads();
    return {best, best_j};
}

template <bool TRUNC>
__device__ __forceinline__ Result solve(const Source src, int m, uint64_t* buf, double* red, int* pick, double* acc, Prefix* pre) {
    if constexpr (TRUNC) return solve_truncated(src, m, buf, red, acc, pre);
    else return solve_median(src, m, buf, red, pick);
}

// scratch of one CTA for the truncated solver (doubles)
__host__ __device__ __forceinline__ size_t cta_scratch_doubles(int m) { return 3 * static_cast<size_t>(m) + 3 * (static_cast<size_t>(m) + 1); }

// plain align(): CTA c solves problems c, c + gridDim.x, ...
// (trunc: device pointer to one scalar, or to (batch, n) values when t_per_elem; unused when !TRUNC)
template <bool TRUNC>
__global__ void __launch_bounds__(kThreads) align_plain_kernel(const float* __restrict__ x, const float* __restrict__ y,
                                                                const float* __restrict__ w, const float* __restrict__ trunc, int t_per_elem,
                                                                int64_t batch, int n, float* a_out, float* loss_out, int64_t* index_out,
                                                                double* scratch) {
    extern __shared__ uint64_t buf[];
    __shared__ double red[kRed];
    __shared__ int pick;
    double* acc = scratch + blockIdx.x * cta_scratch_doubles(n);
    Prefix* pre = reinterpret_cast<Prefix*>(acc + 3 * static_cast<size_t>(n));
    const float ts = (TRUNC && !t_per_elem) ? trunc[0] : 0.f;
    for (int64_t b = blockIdx.x; b < batch; b += gridDim.x) {
        const size_t off = static_cast<size_t>(b) * n;
        const float* t = (TRUNC && t_per_elem) ? trunc + off : nullptr;
        Source src{MOGE_ALIGN_PLAIN, x + off, y + off, w + off, t, ts, {0.f, 0.f, 0.f}, {0.f, 0.f, 0.f}};
        const Result r = solve<TRUNC>(src, n, buf, red, &pick, acc, pre);
        if (threadIdx.x == 0) {
            a_out[b] = breakpoint(src.get(r.index), 0);
            loss_out[b] = static_cast<float>(fmax(r.loss, 0.0));       // fp64 prefix differences can leave -0 or -1e-17 at an exact fit
            index_out[b] = r.index;
        }
    }
}

// anchored solvers: grid (anchor ranges, images); the CTA stages its image, then solves every positive-weight anchor of its range
template <bool TRUNC>
__global__ void __launch_bounds__(kThreads) align_anchored_kernel(const float* __restrict__ src_g, const float* __restrict__ tgt_g,
                                                                   const float* __restrict__ w_g, int mode, float trunc, int n,
                                                                   unsigned long long* slots, double* scratch) {
    extern __shared__ uint64_t smem[];
    __shared__ double red[kRed];
    __shared__ int pick;
    const int comps = mode == MOGE_ANCHOR_DEPTH ? 1 : 3, m = n * comps;
    const int64_t img = blockIdx.y;
    uint64_t* buf = smem;
    float* s_src = reinterpret_cast<float*>(smem + m);
    float* s_tgt = s_src + m;
    float* s_w = s_tgt + m;
    for (int i = threadIdx.x; i < m; i += blockDim.x) { s_src[i] = src_g[img * m + i]; s_tgt[i] = tgt_g[img * m + i]; }
    for (int i = threadIdx.x; i < n; i += blockDim.x) s_w[i] = w_g[img * n + i];
    __syncthreads();
    const size_t cta = static_cast<size_t>(blockIdx.y) * gridDim.x + blockIdx.x;
    double* acc = scratch + cta * cta_scratch_doubles(m);
    Prefix* pre = reinterpret_cast<Prefix*>(acc + 3 * static_cast<size_t>(m));
    const int per = (n + gridDim.x - 1) / gridDim.x, p0 = blockIdx.x * per, p1 = min(n, p0 + per);
    for (int p = p0; p < p1; ++p) {
        if (!(s_w[p] > 0.f)) continue;
        Source src{mode, s_src, s_tgt, s_w, nullptr, trunc, {0.f, 0.f, 0.f}, {0.f, 0.f, 0.f}};
        if (mode == MOGE_ANCHOR_DEPTH) { src.ax[0] = s_src[p]; src.ay[0] = s_tgt[p]; }
        else {
            const bool xy = mode == MOGE_ANCHOR_POINTS_XYZ;      // POINTS_Z anchors z only
            src.ax[0] = xy ? s_src[3 * p] : 0.f;     src.ay[0] = xy ? s_tgt[3 * p] : 0.f;
            src.ax[1] = xy ? s_src[3 * p + 1] : 0.f; src.ay[1] = xy ? s_tgt[3 * p + 1] : 0.f;
            src.ax[2] = s_src[3 * p + 2];            src.ay[2] = s_tgt[3 * p + 2];
        }
        const Result r = solve<TRUNC>(src, m, buf, red, &pick, acc, pre);
        if (threadIdx.x == 0) {
            // >= 0 (prefix differences can round an exact fit below zero): a set sign bit would sort the key after every positive loss
            const float loss = __fadd_rn(static_cast<float>(fmax(r.loss, 0.0)), 0.f);
            // (loss, anchor, index) packed so that the unsigned order is the lexicographic one: loss >= 0 (or NaN, which sorts last)
            const unsigned long long packed = (static_cast<unsigned long long>(__float_as_uint(loss)) << 26) |
                                              (static_cast<unsigned long long>(p) << 14) | static_cast<unsigned long long>(r.index);
            atomicMin(slots + img, packed);
        }
    }
}

__global__ void anchored_finish_kernel(const unsigned long long* slots, int64_t batch, float* loss, int64_t* anchor, int64_t* index) {
    const int64_t b = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
    if (b >= batch) return;
    const unsigned long long s = slots[b];
    if (s == kEmptySlot) { loss[b] = INFINITY; anchor[b] = -1; index[b] = -1; return; }
    loss[b] = __uint_as_float(static_cast<uint32_t>(s >> 26));
    anchor[b] = static_cast<int64_t>((s >> 14) & 0xfffu);
    index[b] = static_cast<int64_t>(s & 0x3fffu);
}

// align_affine_lstsq (alignment.py:399-416): lstsq of [sqrt(w) x, 1] a|b = sqrt(w) y, i.e. the 2x2 normal equations with
// u = sqrt(w) x, v = sqrt(w) y:  [Su2 Su; Su n] [a; b] = [Suv; Sv]
__global__ void __launch_bounds__(kThreads) lstsq_kernel(const float* __restrict__ x, const float* __restrict__ y, const float* __restrict__ w,
                                                         int64_t n, float* a_out, float* b_out) {
    __shared__ double red[kWarps];
    const size_t off = static_cast<size_t>(blockIdx.x) * n;
    double su = 0.0, su2 = 0.0, suv = 0.0, sv = 0.0;
    for (int64_t i = threadIdx.x; i < n; i += blockDim.x) {
        const float r = w ? sqrtf(w[off + i]) : 1.f;
        const double u = static_cast<double>(__fmul_rn(r, x[off + i])), v = static_cast<double>(__fmul_rn(r, y[off + i]));
        su += u; su2 += u * u; suv += u * v; sv += v;
    }
    su = block_sum<kThreads>(su, red); su2 = block_sum<kThreads>(su2, red);
    suv = block_sum<kThreads>(suv, red); sv = block_sum<kThreads>(sv, red);
    if (threadIdx.x == 0) {
        const double nn = static_cast<double>(n), det = su2 * nn - su * su;
        a_out[blockIdx.x] = static_cast<float>((nn * suv - su * sv) / det);
        b_out[blockIdx.x] = static_cast<float>((su2 * sv - su * suv) / det);
    }
}

// launch geometry shared by the workspace query and the launches
struct Plan { dim3 grid; size_t smem; size_t scratch_bytes; size_t slot_bytes; };

int plan(int mode, int truncated, int64_t batch, int n, Plan* pl) {
    if (batch <= 0) return set_error("align: batch must be positive (got %lld)", static_cast<long long>(batch));
    if (mode < MOGE_ALIGN_PLAIN || mode > MOGE_ANCHOR_POINTS_XYZ) return set_error("align: unknown mode %d", mode);
    if (mode == MOGE_ALIGN_PLAIN) {
        if (n <= 0 || n > kMaxElems) return set_error("align: n = %d elements is outside [1, %d] (4096 points x 3 components)", n, kMaxElems);
    } else if (n <= 0 || n > kMaxPoints) {
        return set_error("align: n = %d points is outside [1, %d]", n, kMaxPoints);
    }
    int sms = 0, dev = 0, smem_per_sm = 0;
    MG_TRY(check_device("align", &sms));
    CUDA_TRY(cudaGetDevice(&dev));
    CUDA_TRY(cudaDeviceGetAttribute(&smem_per_sm, cudaDevAttrMaxSharedMemoryPerMultiprocessor, dev));
    const int comps = mode == MOGE_ANCHOR_DEPTH || mode == MOGE_ALIGN_PLAIN ? 1 : 3, m = n * comps;
    int64_t ctas;
    if (mode == MOGE_ALIGN_PLAIN) {
        ctas = batch < 2 * sms ? batch : 2 * sms;          // 2 CTAs of <= 97 KB fit an SM
        pl->grid = dim3(static_cast<unsigned>(ctas));
        pl->smem = static_cast<size_t>(m) * 8;
        pl->slot_bytes = 0;
    } else {
        if (batch > 65535) return set_error("align: at most 65535 images per call (got %lld)", static_cast<long long>(batch));
        pl->smem = static_cast<size_t>(m) * 8 + (2 * static_cast<size_t>(m) + n) * 4;
        // One wave: as many anchor ranges per image as fit the resident CTAs of the device (rounded down, so that a batch never
        // spills a partial second wave).  Residency is bounded by shared memory (the CTA's own plus ~2 KB of static smem and
        // per-block reserve) and by registers: <= 64 per thread at 512 threads leaves room for two CTAs per SM.
        const int per_sm = static_cast<int>(std::max<size_t>(1, std::min<size_t>(2, smem_per_sm / (pl->smem + 2048))));
        const int ranges = static_cast<int>(std::min<int64_t>(n, std::max<int64_t>(1, static_cast<int64_t>(sms) * per_sm / batch)));
        ctas = static_cast<int64_t>(ranges) * batch;
        pl->grid = dim3(ranges, static_cast<unsigned>(batch));
        pl->slot_bytes = WsLayout::up(static_cast<size_t>(batch) * 8);
    }
    pl->scratch_bytes = truncated ? static_cast<size_t>(ctas) * cta_scratch_doubles(m) * 8 : 0;
    return 0;
}

// one instantiation (and one once-per-device flag) per kernel
template <auto Kern, typename... Args>
int launch(const Plan& pl, cudaStream_t st, Args... args) {
    MG_SET_SMEM_ONCE(Kern, static_cast<int>(kMaxSmem));      // the largest any call of this kernel uses
    Kern<<<pl.grid, kThreads, pl.smem, st>>>(args...);
    CUDA_TRY(cudaGetLastError());
    return 0;
}

}  // namespace
}  // namespace mg

using namespace mg;

extern "C" {

int moge_align_workspace_bytes(int mode, int truncated, int64_t batch, int n, size_t* bytes) {
    if (!bytes) return set_error("null argument");
    Plan pl;
    MG_TRY(plan(mode, truncated, batch, n, &pl));
    *bytes = pl.slot_bytes + pl.scratch_bytes;
    return 0;
}

int moge_align(const float* x, const float* y, const float* w, const float* trunc, int trunc_per_elem, int64_t batch, int n, float* a,
               float* loss, int64_t* index, void* workspace, size_t workspace_bytes, void* stream) {
    if (!x || !y || !w || !a || !loss || !index) return set_error("null argument");
    Plan pl;
    MG_TRY(plan(MOGE_ALIGN_PLAIN, trunc != nullptr, batch, n, &pl));
    MG_TRY(check_workspace(pl.slot_bytes + pl.scratch_bytes, workspace, workspace_bytes, "align"));
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    double* scratch = static_cast<double*>(workspace);
    if (!trunc) return launch<align_plain_kernel<false>>(pl, st, x, y, w, trunc, 0, batch, n, a, loss, index, scratch);
    return launch<align_plain_kernel<true>>(pl, st, x, y, w, trunc, trunc_per_elem, batch, n, a, loss, index, scratch);
}

int moge_align_anchored(const float* src, const float* tgt, const float* w, int mode, float trunc, int64_t batch, int n, float* loss,
                        int64_t* anchor, int64_t* index, void* workspace, size_t workspace_bytes, void* stream) {
    if (!src || !tgt || !w || !loss || !anchor || !index) return set_error("null argument");
    if (mode == MOGE_ALIGN_PLAIN) return set_error("align_anchored: mode must be one of MOGE_ANCHOR_*");
    Plan pl;
    MG_TRY(plan(mode, trunc >= 0.f, batch, n, &pl));
    MG_TRY(check_workspace(pl.slot_bytes + pl.scratch_bytes, workspace, workspace_bytes, "align"));
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    unsigned long long* slots = static_cast<unsigned long long*>(workspace);
    double* scratch = reinterpret_cast<double*>(static_cast<char*>(workspace) + pl.slot_bytes);
    CUDA_TRY(cudaMemsetAsync(slots, 0xff, static_cast<size_t>(batch) * 8, st));
    if (trunc >= 0.f) MG_TRY(launch<align_anchored_kernel<true>>(pl, st, src, tgt, w, mode, trunc, n, slots, scratch));
    else MG_TRY(launch<align_anchored_kernel<false>>(pl, st, src, tgt, w, mode, trunc, n, slots, scratch));
    anchored_finish_kernel<<<static_cast<unsigned>((batch + 255) / 256), 256, 0, st>>>(slots, batch, loss, anchor, index);
    CUDA_TRY(cudaGetLastError());
    return 0;
}

int moge_align_affine_lstsq(const float* x, const float* y, const float* w, int64_t batch, int64_t n, float* a, float* b, void* stream) {
    if (!x || !y || !a || !b) return set_error("null argument");
    if (batch <= 0 || n <= 0) return set_error("align_affine_lstsq: bad shape batch=%lld n=%lld", static_cast<long long>(batch),
                                               static_cast<long long>(n));
    if (batch > 0x7fffffff) return set_error("align_affine_lstsq: batch too large");
    MG_TRY(check_device("align_affine_lstsq"));
    lstsq_kernel<<<static_cast<unsigned>(batch), kThreads, 0, static_cast<cudaStream_t>(stream)>>>(x, y, w, n, a, b);
    CUDA_TRY(cudaGetLastError());
    return 0;
}

}  // extern "C"
