// Map colourisation (moge/utils/vis.py of the reference): colorize_depth, colorize_depth_affine, colorize_disparity and
// colorize_normal, restated in oracle/vis_port.py, which these kernels match bit for bit.  No fast-math: every fp32 operation
// of the reference is one IEEE-rounded intrinsic here.
//
// Masked quantiles (np.nanquantile, linear method, fp32): an MSD radix select over order_key(value) in four 8-bit digit passes.
// Every rank one call needs (floor and ceil of each q's virtual index) is selected in the same passes.  A pass counts the digit
// of every valid value whose higher digits equal that rank's prefix into a per-CTA shared histogram (warp-aggregated with
// __match_any_sync), then adds the nonzero bins to the image's global histogram with integer atomics; one small kernel per pass
// turns the histograms into the next prefix and the rank left inside it.  Integer sums do not depend on the order of the
// additions, so the selected keys and the quantiles are the same bits on every run and for every batch composition.  The
// finishing kernel applies numpy's index arithmetic and _lerp (including its t >= 0.5 branch) and writes (batch, nq) fp32.
//
// Colouring: value -> (v - lo) / (hi - lo) -> optionally 1 - x -> x * 256 -> the 256-entry uint8 table with matplotlib's
// Colormap.__call__ rules (256 -> 255, < 0 -> first colour, >= 256 -> last colour, NaN -> black, truncation).
#include "common.cuh"
#include "host_api.h"
#include "../../include/moge_b200.h"
#include <math.h>
#include <stdint.h>

namespace mg {
namespace {

constexpr int kThreads = 256;
constexpr int kPxPerThread = 64;
constexpr int kPxPerCta = kThreads * kPxPerThread;   // pixels per CTA of a histogram pass
constexpr int kDigits = 4;                          // 8-bit digits of a 32-bit key, most significant first
constexpr int kBins = 256;
constexpr int kMaxRanks = 2 * MOGE_VIS_MAX_QUANTILES;
constexpr int64_t kMaxPixels = int64_t(1) << 30;    // per image: histogram counts stay int32

// the q values, fp32 as nanquantile casts a Python float to the array's dtype
struct Quantiles { float q[MOGE_VIS_MAX_QUANTILES]; };
// per image: the valid count, and per rank the rank left inside its current prefix and that prefix
struct State {
    long long n;
    long long left[kMaxRanks];
    uint32_t prefix[kMaxRanks];
};

// The value the reference colours at pixel p, NaN where it is excluded: 1 / depth where depth > 0 (DEPTH, infinities kept: 1 /
// inf = 0), the value itself (VALUE); NaN off the mask.
__device__ __forceinline__ float vis_value(const float* __restrict__ src, int kind, const uint8_t* __restrict__ mask, int64_t e) {
    const float v = src[e];
    const float nan = __int_as_float(0x7fc00000);
    if (mask && !mask[e]) return nan;
    if (kind == MOGE_VIS_DEPTH) return v > 0.f ? __fdiv_rn(1.f, v) : nan;
    return v;
}

// grid (CTAs per image, images).  digit 0 counts every valid value into histogram slot 0; later digits count, per rank, the
// values whose higher digits equal the rank's prefix.
__global__ void __launch_bounds__(kThreads) hist_kernel(const float* __restrict__ src, int kind, const uint8_t* __restrict__ mask,
                                                        int64_t hw, int ranks, int digit, const State* __restrict__ state,
                                                        int* __restrict__ hist) {
    __shared__ int h[kMaxRanks * kBins];
    __shared__ uint32_t pre[kMaxRanks];
    const int64_t b = blockIdx.y;
    const int slots = digit == 0 ? 1 : ranks;
    for (int i = threadIdx.x; i < slots * kBins; i += kThreads) h[i] = 0;
    if (threadIdx.x < ranks) pre[threadIdx.x] = state[b].prefix[threadIdx.x];
    __syncthreads();
    const int shift = 24 - 8 * digit;
    const int64_t p0 = static_cast<int64_t>(blockIdx.x) * kPxPerCta;
    for (int r = 0; r < kPxPerThread; ++r) {
        const int64_t p = p0 + static_cast<int64_t>(r) * kThreads + threadIdx.x;
        if (p0 + static_cast<int64_t>(r) * kThreads >= hw) break;       // uniform over the CTA
        bool ok = p < hw;
        float v = 0.f;
        if (ok) { v = vis_value(src, kind, mask, b * hw + p); ok = !(v != v); }
        const uint32_t key = order_key(v);
        const int bin = static_cast<int>((key >> shift) & 0xffu);
        for (int s = 0; s < slots; ++s) {
            const bool hit = ok && (digit == 0 || (key >> (shift + 8)) == pre[s]);
            const int slot = hit ? s * kBins + bin : -1;
            const unsigned peers = __match_any_sync(0xffffffffu, slot);
            if (hit && (threadIdx.x & 31) == __ffs(peers) - 1) atomicAdd(&h[slot], __popc(peers));
        }
    }
    __syncthreads();
    int* g = hist + (b * kDigits + digit) * kMaxRanks * kBins;
    for (int i = threadIdx.x; i < slots * kBins; i += kThreads)
        if (h[i]) atomicAdd(&g[i], h[i]);
}

// numpy's linear-method index arithmetic on fp32 (nanquantile casts a Python-float q to the array's dtype): virtual index
// v = fp32(n - 1) * q, previous = floor(v), next = previous + 1, both n - 1 when v >= n - 1; gamma = fp32(v - previous) with
// previous as an integer (-1 above the bounds).
struct Virtual { long long prev, next; float gamma; };
__device__ __forceinline__ Virtual virtual_index(long long n, float q) {
    const float last = __ll2float_rn(n - 1);
    const float v = __fmul_rn(last, q);
    Virtual r;
    if (v >= last) {
        r.prev = r.next = n - 1;
        r.gamma = __double2float_rn(__dadd_rn(static_cast<double>(v), 1.0));
    } else {
        const float f = floorf(v);
        r.prev = static_cast<long long>(f);
        r.next = static_cast<long long>(__fadd_rn(f, 1.f));
        r.gamma = __double2float_rn(__dsub_rn(static_cast<double>(v), static_cast<double>(r.prev)));
    }
    return r;
}

// grid (images), one warp: after digit `digit`'s histograms, each rank's next prefix and the rank left inside it
__global__ void select_kernel(const int* __restrict__ hist, const Quantiles q, int nq, int digit, State* __restrict__ state) {
    const int64_t b = blockIdx.x;
    State& s = state[b];
    const int* g = hist + (b * kDigits + digit) * kMaxRanks * kBins;
    const int r = threadIdx.x;
    long long n = 0;
    if (digit == 0) {
        for (int i = 0; i < kBins; ++i) n += g[i];
        if (r == 0) s.n = n;
        if (r < 2 * nq && n > 0) {
            const Virtual v = virtual_index(n, q.q[r / 2]);
            s.left[r] = (r & 1) ? v.next : v.prev;
        }
    } else {
        n = s.n;
    }
    if (r >= 2 * nq || n == 0) return;
    const int* h = g + (digit == 0 ? 0 : r * kBins);
    long long left = s.left[r], cum = 0;
    int bin = 0;
    for (; bin < kBins - 1; ++bin) {
        if (cum + h[bin] > left) break;
        cum += h[bin];
    }
    s.left[r] = left - cum;
    s.prefix[r] = (s.prefix[r] << 8) | static_cast<uint32_t>(bin);
}

// grid (images), one thread per q: numpy's _lerp(previous, next, gamma) in fp32; NaN for an image without a valid value
__global__ void finish_kernel(const Quantiles q, int nq, const State* __restrict__ state, float* __restrict__ out) {
    const int64_t b = blockIdx.x;
    const int i = threadIdx.x;
    if (i >= nq) return;
    const State& s = state[b];
    float res = __int_as_float(0x7fc00000);
    if (s.n > 0) {
        const float t = virtual_index(s.n, q.q[i]).gamma;
        const float a = key_value(s.prefix[2 * i]), c = key_value(s.prefix[2 * i + 1]);
        const float diff = __fsub_rn(c, a);
        res = t >= 0.5f ? __fsub_rn(c, __fmul_rn(diff, __fsub_rn(1.f, t))) : __fadd_rn(a, __fmul_rn(diff, t));
    }
    out[b * nq + i] = res;
}

// grid (pixel blocks, images), one thread per pixel
__global__ void __launch_bounds__(kThreads) colorize_kernel(const float* __restrict__ src, int kind, int invert, const uint8_t* __restrict__ mask,
                                                            int64_t hw, const float* __restrict__ range, const uint8_t* __restrict__ lut,
                                                            int bgr, uint8_t* __restrict__ out) {
    __shared__ uint8_t s_lut[kBins * 3];
    for (int i = threadIdx.x; i < kBins * 3; i += kThreads) s_lut[i] = lut[i];
    __syncthreads();
    const int64_t b = blockIdx.y, p = static_cast<int64_t>(blockIdx.x) * kThreads + threadIdx.x;
    if (p >= hw) return;
    const int64_t e = b * hw + p;
    float x = vis_value(src, kind, mask, e);
    if (range) {
        const float lo = range[b * 2], hi = range[b * 2 + 1];
        x = __fdiv_rn(__fsub_rn(x, lo), __fsub_rn(hi, lo));
    }
    if (invert) x = __fsub_rn(1.f, x);
    x = __fmul_rn(x, static_cast<float>(kBins));
    if (x == static_cast<float>(kBins)) x = static_cast<float>(kBins - 1);
    uint8_t c0 = 0, c1 = 0, c2 = 0;
    if (!(x != x)) {
        const int i = x < 0.f ? 0 : x >= static_cast<float>(kBins) ? kBins - 1 : static_cast<int>(x);
        c0 = s_lut[i * 3]; c1 = s_lut[i * 3 + 1]; c2 = s_lut[i * 3 + 2];
    }
    uint8_t* o = out + e * 3;
    o[0] = bgr ? c2 : c0;
    o[1] = c1;
    o[2] = bgr ? c0 : c2;
}

// colorize_normal in fp64: trunc(clip(n * (0.5, -0.5, -0.5) + 0.5, 0, 1) * 255), 0 (-> 127) off the mask, NaN -> 0 (numpy's cast)
__device__ __forceinline__ uint8_t normal_byte(float n, double s) {
    double x = __dadd_rn(__dmul_rn(static_cast<double>(n), s), 0.5);
    if (x != x) return 0;
    x = fmin(fmax(x, 0.0), 1.0);
    return static_cast<uint8_t>(__dmul_rn(x, 255.0));
}
__global__ void __launch_bounds__(kThreads) normal_kernel(const float* __restrict__ normal, const uint8_t* __restrict__ mask, int64_t hw,
                                                          int bgr, uint8_t* __restrict__ out) {
    const int64_t b = blockIdx.y, p = static_cast<int64_t>(blockIdx.x) * kThreads + threadIdx.x;
    if (p >= hw) return;
    const int64_t e = b * hw + p;
    const bool in = !mask || mask[e];
    const uint8_t c0 = normal_byte(in ? normal[e * 3] : 0.f, 0.5), c1 = normal_byte(in ? normal[e * 3 + 1] : 0.f, -0.5),
                  c2 = normal_byte(in ? normal[e * 3 + 2] : 0.f, -0.5);
    uint8_t* o = out + e * 3;
    o[0] = bgr ? c2 : c0;
    o[1] = c1;
    o[2] = bgr ? c0 : c2;
}

// workspace layout: per-image state, the (batch, digits, ranks, bins) histograms
struct Layout { size_t state, hist, total; };
Layout layout(int64_t batch) {
    const size_t B = static_cast<size_t>(batch);
    WsLayout ws;
    Layout l;
    l.state = ws.add(B * sizeof(State));
    l.hist = ws.add(B * kDigits * kMaxRanks * kBins * sizeof(int));
    l.total = ws.total;
    return l;
}

int check_kind(const char* what, int kind) {
    if (kind != MOGE_VIS_DEPTH && kind != MOGE_VIS_VALUE) return set_error("%s: unknown value kind %d", what, kind);
    return 0;
}

}  // namespace
}  // namespace mg

using namespace mg;

extern "C" {

int moge_vis_workspace_bytes(int64_t batch, int H, int W, size_t* bytes) {
    if (!bytes) return set_error("null argument");
    MG_TRY(check_batch_map("vis", batch, H, W, kMaxPixels));
    *bytes = layout(batch).total;
    return 0;
}

int moge_vis_quantiles(const float* src, int kind, const uint8_t* mask, int64_t batch, int H, int W, const float* q, int nq, float* out,
                       void* workspace, size_t workspace_bytes, void* stream) {
    if (!src || !q || !out) return set_error("null argument");
    MG_TRY(check_batch_map("vis_quantiles", batch, H, W, kMaxPixels));
    MG_TRY(check_kind("vis_quantiles", kind));
    if (nq < 1 || nq > MOGE_VIS_MAX_QUANTILES) return set_error("vis_quantiles: %d quantiles is outside [1, %d]", nq, MOGE_VIS_MAX_QUANTILES);
    for (int i = 0; i < nq; ++i)
        if (!(q[i] >= 0.f && q[i] <= 1.f)) return set_error("vis_quantiles: quantile %g is outside [0, 1]", static_cast<double>(q[i]));
    const Layout l = layout(batch);
    MG_TRY(check_workspace(l.total, workspace, workspace_bytes, "vis_quantiles"));
    MG_TRY(check_device("vis_quantiles"));
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    char* ws = static_cast<char*>(workspace);
    State* state = reinterpret_cast<State*>(ws + l.state);
    int* hist = reinterpret_cast<int*>(ws + l.hist);
    Quantiles dq = {};
    for (int i = 0; i < nq; ++i) dq.q[i] = q[i];
    CUDA_TRY(cudaMemsetAsync(ws, 0, l.total, st));
    const int64_t hw = static_cast<int64_t>(H) * W;
    const dim3 grid(static_cast<unsigned>((hw + kPxPerCta - 1) / kPxPerCta), static_cast<unsigned>(batch));
    for (int d = 0; d < kDigits; ++d) {
        hist_kernel<<<grid, kThreads, 0, st>>>(src, kind, mask, hw, 2 * nq, d, state, hist);
        CUDA_TRY(cudaGetLastError());
        select_kernel<<<static_cast<unsigned>(batch), 32, 0, st>>>(hist, dq, nq, d, state);
        CUDA_TRY(cudaGetLastError());
    }
    finish_kernel<<<static_cast<unsigned>(batch), 32, 0, st>>>(dq, nq, state, out);
    CUDA_TRY(cudaGetLastError());
    return 0;
}

int moge_vis_colorize(const float* src, int kind, int invert, const uint8_t* mask, int64_t batch, int H, int W, const float* range,
                      const uint8_t* lut, int bgr, uint8_t* out, void* stream) {
    if (!src || !lut || !out) return set_error("null argument");
    MG_TRY(check_batch_map("vis_colorize", batch, H, W, kMaxPixels));
    MG_TRY(check_kind("vis_colorize", kind));
    MG_TRY(check_device("vis_colorize"));
    const int64_t hw = static_cast<int64_t>(H) * W;
    const dim3 grid(static_cast<unsigned>((hw + kThreads - 1) / kThreads), static_cast<unsigned>(batch));
    colorize_kernel<<<grid, kThreads, 0, static_cast<cudaStream_t>(stream)>>>(src, kind, invert ? 1 : 0, mask, hw, range, lut, bgr ? 1 : 0, out);
    CUDA_TRY(cudaGetLastError());
    return 0;
}

int moge_vis_normal(const float* normal, const uint8_t* mask, int64_t batch, int H, int W, int bgr, uint8_t* out, void* stream) {
    if (!normal || !out) return set_error("null argument");
    MG_TRY(check_batch_map("vis_normal", batch, H, W, kMaxPixels));
    MG_TRY(check_device("vis_normal"));
    const int64_t hw = static_cast<int64_t>(H) * W;
    const dim3 grid(static_cast<unsigned>((hw + kThreads - 1) / kThreads), static_cast<unsigned>(batch));
    normal_kernel<<<grid, kThreads, 0, static_cast<cudaStream_t>(stream)>>>(normal, mask, hw, bgr ? 1 : 0, out);
    CUDA_TRY(cudaGetLastError());
    return 0;
}

}  // extern "C"
