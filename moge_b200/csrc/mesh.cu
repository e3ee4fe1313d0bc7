// Mesh export (moge/scripts/infer.py:124-150 of the reference): utils3d's depth_map_edge and build_mesh_from_map, restated in
// oracle/utils3d_mesh.py, which these kernels match bit for bit.  The panorama export (moge/scripts/infer_panorama.py:136-150)
// adds point_map_to_normal_map and normal_map_edge, restated in oracle/utils3d_normals.py: the normals match it bit for bit, the
// normal edges up to acosf's rounding (at most 2 ulp, as numpy's arccos) at angles within a few ulp of the threshold.
//
// depth_map_edge: one CTA per 32 x 32 output tile with a halo of kernel_size / 2, a separable NaN-propagating window max of the
// depth and of its negation (masked-out and out-of-image pixels are -inf), then diff = max(d) + max(-d) and the two tolerance
// tests in fp32 with one rounding per operation (__fadd_rn / __fdiv_rn: the contract is bitwise).
//
// build_mesh_from_map: the pixels of an image are cut into fixed tiles of kTilePx in row-major order.  A quad is named by its
// top-left pixel, so row-major pixel order is both the vertex order and the quad order of the reference's np.unique compaction.
// A count pass writes per-tile vertex and quad counts, one CTA scans them image by image in a fixed order (integers only), and
// the emit passes re-derive the flags, rank them inside the tile with ballots and write the vertex-index map, the gathered
// attributes and the faces.  Nothing depends on the other images of a batch except where an image's rows land.
#include "common.cuh"
#include "host_api.h"
#include "../../include/moge_b200.h"
#include <math.h>
#include <stdint.h>
#include <string.h>

namespace mg {
namespace {

constexpr int kThreads = 256;
constexpr int kWarps = kThreads / 32;
constexpr int kRounds = 16;
constexpr int kTilePx = kThreads * kRounds;       // pixels per count / emit tile
constexpr int kScanThreads = 1024;
constexpr int kEdgeT = 32;                        // edge tile: kEdgeT x kEdgeT outputs
constexpr int kMaxR = 3;                          // kernel_size <= 7
constexpr int kEdgeS = kEdgeT + 2 * kMaxR;
constexpr int64_t kMaxPixels = int64_t(1) << 30;  // per image: vertex ids and triangle counts stay below 2^31

struct Maps { moge_mesh_map_t m[MOGE_MESH_MAX_MAPS]; int n; };

// ---------------------------------------------------------------------------------------------------- depth edge
__global__ void __launch_bounds__(kThreads) edge_kernel(const float* __restrict__ depth, const uint8_t* __restrict__ mask,
                                                        const uint8_t* __restrict__ keep, int H, int W, int r, float atol, int has_atol,
                                                        float rtol, int has_rtol, uint8_t* __restrict__ out) {
    __shared__ float s_hi[kEdgeS][kEdgeS], s_lo[kEdgeS][kEdgeS];   // d and -d; -inf outside the image and off the mask
    __shared__ float h_hi[kEdgeS][kEdgeT], h_lo[kEdgeS][kEdgeT];   // row-pass maxima
    const int64_t b = blockIdx.z, hw = static_cast<int64_t>(H) * W;
    const int i0 = blockIdx.y * kEdgeT, j0 = blockIdx.x * kEdgeT, S = kEdgeT + 2 * r, k2 = 2 * r;
    for (int k = threadIdx.x; k < S * S; k += kThreads) {
        const int li = k / S, lj = k % S, i = i0 - r + li, j = j0 - r + lj;
        float hi = -INFINITY, lo = -INFINITY;
        if (i >= 0 && i < H && j >= 0 && j < W) {
            const int64_t p = b * hw + static_cast<int64_t>(i) * W + j;
            if (!mask || mask[p]) { const float d = depth[p]; hi = d; lo = -d; }
        }
        s_hi[li][lj] = hi;
        s_lo[li][lj] = lo;
    }
    __syncthreads();
    for (int k = threadIdx.x; k < S * kEdgeT; k += kThreads) {
        const int li = k / kEdgeT, oj = k % kEdgeT;
        float hi = s_hi[li][oj], lo = s_lo[li][oj];
        for (int t = 1; t <= k2; ++t) { hi = nan_max(hi, s_hi[li][oj + t]); lo = nan_max(lo, s_lo[li][oj + t]); }
        h_hi[li][oj] = hi;
        h_lo[li][oj] = lo;
    }
    __syncthreads();
    for (int k = threadIdx.x; k < kEdgeT * kEdgeT; k += kThreads) {
        const int oi = k / kEdgeT, oj = k % kEdgeT, i = i0 + oi, j = j0 + oj;
        if (i >= H || j >= W) continue;
        float hi = h_hi[oi][oj], lo = h_lo[oi][oj];
        for (int t = 1; t <= k2; ++t) { hi = nan_max(hi, h_hi[oi + t][oj]); lo = nan_max(lo, h_lo[oi + t][oj]); }
        const int64_t p = b * hw + static_cast<int64_t>(i) * W + j;
        const float diff = __fadd_rn(hi, lo);
        bool edge = false;
        if (has_atol) edge |= diff > atol;
        if (has_rtol) edge |= __fdiv_rn(diff, depth[p]) > rtol;
        out[p] = keep ? static_cast<uint8_t>(keep[p] && !edge) : static_cast<uint8_t>(edge);
    }
}

// ---------------------------------------------------------------------------------------------------- normals
// Vector helpers with one fp32 rounding per operation, in numpy's order (oracle/utils3d_normals.py): no contraction into FMAs.
struct F3 { float x, y, z; };
__device__ __forceinline__ F3 load3(const float* __restrict__ p, int64_t e) { return {p[e * 3], p[e * 3 + 1], p[e * 3 + 2]}; }
__device__ __forceinline__ F3 sub3(F3 a, F3 b) { return {__fsub_rn(a.x, b.x), __fsub_rn(a.y, b.y), __fsub_rn(a.z, b.z)}; }
__device__ __forceinline__ F3 add3(F3 a, F3 b) { return {__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y), __fadd_rn(a.z, b.z)}; }
__device__ __forceinline__ F3 scale3(F3 a, float s) { return {__fmul_rn(a.x, s), __fmul_rn(a.y, s), __fmul_rn(a.z, s)}; }
// np.cross: component a1 * b2 - a2 * b1, both products rounded
__device__ __forceinline__ F3 cross3(F3 a, F3 b) {
    return {__fsub_rn(__fmul_rn(a.y, b.z), __fmul_rn(a.z, b.y)), __fsub_rn(__fmul_rn(a.z, b.x), __fmul_rn(a.x, b.z)),
            __fsub_rn(__fmul_rn(a.x, b.y), __fmul_rn(a.y, b.x))};
}
// (a0 * b0 + a1 * b1) + a2 * b2
__device__ __forceinline__ float dot3(F3 a, F3 b) { return __fadd_rn(__fadd_rn(__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y)), __fmul_rn(a.z, b.z)); }
// n / (sqrt((x^2 + y^2) + z^2) + 1e-12)
__device__ __forceinline__ F3 normalize3(F3 n) {
    const float d = __fadd_rn(__fsqrt_rn(dot3(n, n)), 1e-12f);
    return {__fdiv_rn(n.x, d), __fdiv_rn(n.y, d), __fdiv_rn(n.z, d)};
}

// point_map_to_normal_map: grid (pixel blocks, images), one thread per pixel.  Neighbours outside the image are zero points off
// the mask; without a mask every product counts.  normal_mask (may be NULL) = any product valid.
__global__ void __launch_bounds__(kThreads) normal_map_kernel(const float* __restrict__ pts, const uint8_t* __restrict__ mask, int H, int W,
                                                              float* __restrict__ normal, uint8_t* __restrict__ normal_mask) {
    const int64_t hw = static_cast<int64_t>(H) * W, p = static_cast<int64_t>(blockIdx.x) * kThreads + threadIdx.x;
    if (p >= hw) return;
    const int64_t e = static_cast<int64_t>(blockIdx.y) * hw + p;
    const int i = static_cast<int>(p / W), j = static_cast<int>(p % W);
    const bool hu = i > 0, hl = j > 0, hd = i + 1 < H, hr = j + 1 < W;
    const F3 zero = {0.f, 0.f, 0.f}, c = load3(pts, e);
    const F3 up = sub3(hu ? load3(pts, e - W) : zero, c), left = sub3(hl ? load3(pts, e - 1) : zero, c);
    const F3 down = sub3(hd ? load3(pts, e + W) : zero, c), right = sub3(hr ? load3(pts, e + 1) : zero, c);
    bool v0 = true, v1 = true, v2 = true, v3 = true;
    if (mask) {
        const bool mc = mask[e], mu = hu && mask[e - W], ml = hl && mask[e - 1], md = hd && mask[e + W], mr = hr && mask[e + 1];
        v0 = mc && mu && ml; v1 = mc && ml && md; v2 = mc && md && mr; v3 = mc && mr && mu;
    }
    // (n * valid).sum(0): multiplied by 0.0 / 1.0, not selected, so a NaN in an invalid product still propagates
    F3 s = scale3(normalize3(cross3(up, left)), v0 ? 1.f : 0.f);
    s = add3(s, scale3(normalize3(cross3(left, down)), v1 ? 1.f : 0.f));
    s = add3(s, scale3(normalize3(cross3(down, right)), v2 ? 1.f : 0.f));
    s = add3(s, scale3(normalize3(cross3(right, up)), v3 ? 1.f : 0.f));
    s = normalize3(s);
    const bool any = v0 || v1 || v2 || v3;
    if (mask && !any) s = zero;
    normal[e * 3] = s.x;
    normal[e * 3 + 1] = s.y;
    normal[e * 3 + 2] = s.z;
    if (normal_mask) normal_mask[e] = any;
}

// normal_map_edge: one CTA per 32 x 32 output tile.  The normals (normalised, edge-padded by clamping) and the edge-padded mask
// of the tile with a 2r halo go to shared memory; the window-max angle map is formed on the tile with an r halo (-inf outside
// the image: the pool's padding), then pooled separably.  NaN propagates through both maxima and is never an edge.  The edge
// is angle > tol compared in fp64; with and_edge it is ANDed with that map, and with keep the output is keep & ~edge.
constexpr int kNrmS = kEdgeT + 4 * kMaxR;
__global__ void __launch_bounds__(kThreads) normal_edge_kernel(const float* __restrict__ normals, const uint8_t* __restrict__ mask,
                                                               const uint8_t* __restrict__ and_edge, const uint8_t* __restrict__ keep, int H,
                                                               int W, int r, double tol, uint8_t* __restrict__ out, float* __restrict__ angle) {
    __shared__ float s_n[3][kNrmS][kNrmS];
    __shared__ uint8_t s_m[kNrmS][kNrmS];
    __shared__ float s_a[kEdgeS][kEdgeS];      // window-max angles
    __shared__ float s_h[kEdgeS][kEdgeT];      // row-pass maxima
    const int64_t b = blockIdx.z, hw = static_cast<int64_t>(H) * W;
    const int i0 = blockIdx.y * kEdgeT, j0 = blockIdx.x * kEdgeT, SN = kEdgeT + 4 * r, SA = kEdgeT + 2 * r, k = 2 * r + 1;
    for (int t = threadIdx.x; t < SN * SN; t += kThreads) {
        const int li = t / SN, lj = t % SN;
        const int i = min(max(i0 - 2 * r + li, 0), H - 1), j = min(max(j0 - 2 * r + lj, 0), W - 1);
        const int64_t p = b * hw + static_cast<int64_t>(i) * W + j;
        const F3 n = normalize3(load3(normals, p));
        s_n[0][li][lj] = n.x;
        s_n[1][li][lj] = n.y;
        s_n[2][li][lj] = n.z;
        s_m[li][lj] = mask ? mask[p] != 0 : 1;
    }
    __syncthreads();
    for (int t = threadIdx.x; t < SA * SA; t += kThreads) {
        const int ai = t / SA, aj = t % SA, i = i0 - r + ai, j = j0 - r + aj;
        float a = -INFINITY;
        if (i >= 0 && i < H && j >= 0 && j < W) {
            const F3 c = {s_n[0][ai + r][aj + r], s_n[1][ai + r][aj + r], s_n[2][ai + r][aj + r]};
            for (int di = 0; di < k; ++di)
                for (int dj = 0; dj < k; ++dj) {
                    const int li = ai + di, lj = aj + dj;
                    const float x = s_m[li][lj] ? acosf(dot3(c, {s_n[0][li][lj], s_n[1][li][lj], s_n[2][li][lj]})) : 0.f;
                    a = nan_max(a, x);
                }
        }
        s_a[ai][aj] = a;
    }
    __syncthreads();
    for (int t = threadIdx.x; t < SA * kEdgeT; t += kThreads) {
        const int li = t / kEdgeT, oj = t % kEdgeT;
        float a = s_a[li][oj];
        for (int d = 1; d < k; ++d) a = nan_max(a, s_a[li][oj + d]);
        s_h[li][oj] = a;
    }
    __syncthreads();
    for (int t = threadIdx.x; t < kEdgeT * kEdgeT; t += kThreads) {
        const int oi = t / kEdgeT, oj = t % kEdgeT, i = i0 + oi, j = j0 + oj;
        if (i >= H || j >= W) continue;
        float a = s_h[oi][oj];
        for (int d = 1; d < k; ++d) a = nan_max(a, s_h[oi + d][oj]);
        const int64_t p = b * hw + static_cast<int64_t>(i) * W + j;
        bool edge = static_cast<double>(a) > tol;
        if (and_edge) edge = edge && and_edge[p];
        out[p] = keep ? static_cast<uint8_t>(keep[p] && !edge) : static_cast<uint8_t>(edge);
        if (angle) angle[p] = a;
    }
}

// ---------------------------------------------------------------------------------------------------- mesh flags
// quad (i, j) has corners (i, j), (i + 1, j), (i + 1, j + 1), (i, j + 1); m == NULL keeps every quad
__device__ __forceinline__ bool quad_kept(const uint8_t* m, int H, int W, int i, int j) {
    if (i < 0 || j < 0 || i >= H - 1 || j >= W - 1) return false;
    if (!m) return true;
    const uint8_t* r0 = m + static_cast<int64_t>(i) * W + j;
    const uint8_t* r1 = r0 + W;
    return r0[0] && r1[0] && r1[1] && r0[1];
}
__device__ __forceinline__ bool vertex_kept(const uint8_t* m, int H, int W, int i, int j) {
    return quad_kept(m, H, W, i - 1, j - 1) || quad_kept(m, H, W, i - 1, j) || quad_kept(m, H, W, i, j - 1) || quad_kept(m, H, W, i, j);
}

__device__ __forceinline__ int block_sum_int(int v, int* red) {
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    __syncthreads();
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
    __syncthreads();
    int s = 0;
    for (int w = 0; w < kWarps; ++w) s += red[w];
    return s;
}

// Rank of this thread's flag among the set flags of the CTA's current round (thread order), and the round's total.  warp_tot is
// double-buffered by round parity, so one barrier per round suffices.
__device__ __forceinline__ int round_rank(bool flag, int (*warp_tot)[kWarps], int round, int* total) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const unsigned bal = __ballot_sync(0xffffffffu, flag);
    int* wt = warp_tot[round & 1];
    if (lane == 0) wt[warp] = __popc(bal);
    __syncthreads();
    int before = 0, tot = 0;
    for (int w = 0; w < kWarps; ++w) { const int c = wt[w]; before += w < warp ? c : 0; tot += c; }
    *total = tot;
    return before + __popc(bal & ((1u << lane) - 1u));
}

// grid (tiles, images): per tile (kept vertices, kept quads)
__global__ void __launch_bounds__(kThreads) count_kernel(const uint8_t* __restrict__ mask, int H, int W, int tiles, int32_t* __restrict__ counts) {
    __shared__ int red[kWarps];
    const int64_t b = blockIdx.y, hw = static_cast<int64_t>(H) * W;
    const uint8_t* m = mask ? mask + b * hw : nullptr;
    const int64_t p0 = static_cast<int64_t>(blockIdx.x) * kTilePx;
    int nv = 0, nq = 0;
    for (int r = 0; r < kRounds; ++r) {
        const int64_t p = p0 + r * kThreads + threadIdx.x;
        if (p >= hw) break;
        const int i = static_cast<int>(p / W), j = static_cast<int>(p % W);
        nv += vertex_kept(m, H, W, i, j);
        nq += quad_kept(m, H, W, i, j);
    }
    nv = block_sum_int(nv, red);
    nq = block_sum_int(nq, red);
    if (threadIdx.x == 0) {
        counts[(b * tiles + blockIdx.x) * 2] = nv;
        counts[(b * tiles + blockIdx.x) * 2 + 1] = nq;
    }
}

// one CTA: image by image, the exclusive scan of the tile counts (offsets inside the image), then per image (vertices, quads,
// first vertex row, first quad) in the batch-wide outputs
__global__ void __launch_bounds__(kScanThreads) scan_kernel(const int32_t* __restrict__ counts, int64_t batch, int tiles,
                                                            int32_t* __restrict__ offsets, int64_t* __restrict__ totals) {
    __shared__ int2 warp_tot[kScanThreads / 32];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    int64_t voff = 0, qoff = 0;
    for (int64_t b = 0; b < batch; ++b) {
        int run_v = 0, run_q = 0;
        for (int t0 = 0; t0 < tiles; t0 += kScanThreads) {
            const int t = t0 + threadIdx.x;
            const int cv = t < tiles ? counts[(b * tiles + t) * 2] : 0, cq = t < tiles ? counts[(b * tiles + t) * 2 + 1] : 0;
            int iv = cv, iq = cq;
            for (int o = 1; o < 32; o <<= 1) {
                const int v = __shfl_up_sync(0xffffffffu, iv, o), q = __shfl_up_sync(0xffffffffu, iq, o);
                if (lane >= o) { iv += v; iq += q; }
            }
            if (lane == 31) warp_tot[warp] = make_int2(iv, iq);
            __syncthreads();
            int bv = 0, bq = 0, tv = 0, tq = 0;
            for (int w = 0; w < kScanThreads / 32; ++w) {
                const int2 c = warp_tot[w];
                if (w < warp) { bv += c.x; bq += c.y; }
                tv += c.x; tq += c.y;
            }
            if (t < tiles) {
                offsets[(b * tiles + t) * 2] = run_v + bv + iv - cv;
                offsets[(b * tiles + t) * 2 + 1] = run_q + bq + iq - cq;
            }
            run_v += tv;
            run_q += tq;
            __syncthreads();
        }
        if (threadIdx.x == 0) {
            totals[b * 4] = run_v;
            totals[b * 4 + 1] = run_q;
            totals[b * 4 + 2] = voff;
            totals[b * 4 + 3] = qoff;
        }
        voff += run_v;
        qoff += run_q;
    }
}

// grid (tiles, images): the vertex-index map (-1 where not kept) and every map's row at each kept vertex
__global__ void __launch_bounds__(kThreads) vertices_kernel(const uint8_t* __restrict__ mask, int H, int W, int tiles,
                                                            const int32_t* __restrict__ offsets, const int64_t* __restrict__ totals,
                                                            const Maps maps, int32_t* __restrict__ vmap) {
    __shared__ int warp_tot[2][kWarps];
    const int64_t b = blockIdx.y, hw = static_cast<int64_t>(H) * W;
    const uint8_t* m = mask ? mask + b * hw : nullptr;
    const int64_t p0 = static_cast<int64_t>(blockIdx.x) * kTilePx, row0 = totals[b * 4 + 2];
    int run = offsets[(b * tiles + blockIdx.x) * 2];
    for (int r = 0; r < kRounds; ++r) {
        const int64_t p = p0 + r * kThreads + threadIdx.x;
        if (p0 + r * kThreads >= hw) break;                          // uniform over the CTA
        const bool in = p < hw;
        const int i = in ? static_cast<int>(p / W) : 0, j = in ? static_cast<int>(p % W) : 0;
        const bool kept = in && vertex_kept(m, H, W, i, j);
        int total;
        const int id = run + round_rank(kept, warp_tot, r, &total);
        run += total;
        if (!in) continue;
        vmap[b * hw + p] = kept ? id : -1;
        if (!kept) continue;
        const int64_t row = row0 + id;
        for (int k = 0; k < maps.n; ++k) {
            const moge_mesh_map_t& d = maps.m[k];
            const int C = d.channels;
            for (int c = 0; c < C; ++c) {
                float x;
                if (d.kind == MOGE_MESH_UV) {
                    x = c == 0 ? __fdiv_rn(static_cast<float>(j) + 0.5f, static_cast<float>(W)) : __fdiv_rn(static_cast<float>(i) + 0.5f, static_cast<float>(H));
                } else {
                    const int64_t e = d.layout == MOGE_MESH_HWC ? (b * hw + p) * C + c : (b * C + c) * hw + p;
                    x = d.kind == MOGE_MESH_U8_UNIT ? __fdiv_rn(static_cast<float>(static_cast<const uint8_t*>(d.src)[e]), 255.f)
                                                    : static_cast<const float*>(d.src)[e];
                }
                x = __fmul_rn(x, d.sign[c]);
                if (d.offset[c] != 0.f) x = __fadd_rn(x, d.offset[c]);
                d.dst[row * C + c] = x;
            }
        }
    }
}

// grid (tiles, images): each kept quad's corners from the vertex-index map, as one quad or two triangles [a, b, c], [a, c, d]
__global__ void __launch_bounds__(kThreads) faces_kernel(const uint8_t* __restrict__ mask, int H, int W, int tiles, int tri,
                                                         const int32_t* __restrict__ offsets, const int64_t* __restrict__ totals,
                                                         const int32_t* __restrict__ vmap, int32_t* __restrict__ faces) {
    __shared__ int warp_tot[2][kWarps];
    const int64_t b = blockIdx.y, hw = static_cast<int64_t>(H) * W;
    const uint8_t* m = mask ? mask + b * hw : nullptr;
    const int32_t* v = vmap + b * hw;
    const int64_t p0 = static_cast<int64_t>(blockIdx.x) * kTilePx, quad0 = totals[b * 4 + 3];
    int run = offsets[(b * tiles + blockIdx.x) * 2 + 1];
    for (int r = 0; r < kRounds; ++r) {
        const int64_t p = p0 + r * kThreads + threadIdx.x;
        if (p0 + r * kThreads >= hw) break;
        const bool in = p < hw;
        const bool kept = in && quad_kept(m, H, W, static_cast<int>(p / W), static_cast<int>(p % W));
        int total;
        const int id = run + round_rank(kept, warp_tot, r, &total);
        run += total;
        if (!kept) continue;
        const int32_t a = v[p], bb = v[p + W], c = v[p + W + 1], d = v[p + 1];
        if (tri) {
            int32_t* f = faces + (quad0 + id) * 6;
            f[0] = a; f[1] = bb; f[2] = c; f[3] = a; f[4] = c; f[5] = d;
        } else {
            int32_t* f = faces + (quad0 + id) * 4;
            f[0] = a; f[1] = bb; f[2] = c; f[3] = d;
        }
    }
}

int num_tiles(int H, int W) { return static_cast<int>((static_cast<int64_t>(H) * W + kTilePx - 1) / kTilePx); }

// workspace layout: tile counts, tile offsets, vertex-index map
struct Layout { size_t counts, offsets, vmap, total; };
Layout layout(int64_t batch, int H, int W) {
    const size_t t = static_cast<size_t>(num_tiles(H, W)), B = static_cast<size_t>(batch);
    WsLayout ws;
    Layout l;
    l.counts = ws.add(B * t * 2 * 4);
    l.offsets = ws.add(B * t * 2 * 4);
    l.vmap = ws.add(B * static_cast<size_t>(H) * W * 4);
    l.total = ws.total;
    return l;
}

}  // namespace
}  // namespace mg

using namespace mg;

extern "C" {

int moge_mesh_workspace_bytes(int64_t batch, int H, int W, size_t* bytes) {
    if (!bytes) return set_error("null argument");
    MG_TRY(check_batch_map("mesh", batch, H, W, kMaxPixels));
    *bytes = layout(batch, H, W).total;
    return 0;
}

int moge_depth_edge(const float* depth, const uint8_t* mask, const uint8_t* keep, int64_t batch, int H, int W, int kernel_size,
                    const float* atol, const float* rtol, uint8_t* out, void* stream) {
    if (!depth || !out) return set_error("null argument");
    MG_TRY(check_batch_map("depth_map_edge", batch, H, W, kMaxPixels));
    if (kernel_size < 3 || kernel_size > 2 * kMaxR + 1 || kernel_size % 2 == 0)
        return set_error("depth_map_edge: kernel_size %d is not one of 3, 5, 7", kernel_size);
    MG_TRY(check_device("depth_map_edge"));
    const dim3 grid((W + kEdgeT - 1) / kEdgeT, (H + kEdgeT - 1) / kEdgeT, static_cast<unsigned>(batch));
    edge_kernel<<<grid, kThreads, 0, static_cast<cudaStream_t>(stream)>>>(depth, mask, keep, H, W, kernel_size / 2, atol ? *atol : 0.f,
                                                                          atol != nullptr, rtol ? *rtol : 0.f, rtol != nullptr, out);
    CUDA_TRY(cudaGetLastError());
    return 0;
}

int moge_normal_map(const float* points, const uint8_t* mask, int64_t batch, int H, int W, float* normal, uint8_t* normal_mask, void* stream) {
    if (!points || !normal) return set_error("null argument");
    MG_TRY(check_batch_map("point_map_to_normal_map", batch, H, W, kMaxPixels));
    MG_TRY(check_device("point_map_to_normal_map"));
    const int64_t blocks = (static_cast<int64_t>(H) * W + kThreads - 1) / kThreads;
    normal_map_kernel<<<dim3(static_cast<unsigned>(blocks), static_cast<unsigned>(batch)), kThreads, 0, static_cast<cudaStream_t>(stream)>>>(
        points, mask, H, W, normal, normal_mask);
    CUDA_TRY(cudaGetLastError());
    return 0;
}

int moge_normal_edge(const float* normals, const uint8_t* mask, const uint8_t* and_edge, const uint8_t* keep, int64_t batch, int H, int W,
                     int kernel_size, double tol, uint8_t* out, float* angle, void* stream) {
    if (!normals || !out) return set_error("null argument");
    MG_TRY(check_batch_map("normal_map_edge", batch, H, W, kMaxPixels));
    if (kernel_size < 3 || kernel_size > 2 * kMaxR + 1 || kernel_size % 2 == 0)
        return set_error("normal_map_edge: kernel_size %d is not one of 3, 5, 7", kernel_size);
    if ((H + kEdgeT - 1) / kEdgeT > 65535) return set_error("normal_map_edge: %d rows is more than %d", H, 65535 * kEdgeT);
    MG_TRY(check_device("normal_map_edge"));
    const dim3 grid((W + kEdgeT - 1) / kEdgeT, (H + kEdgeT - 1) / kEdgeT, static_cast<unsigned>(batch));
    normal_edge_kernel<<<grid, kThreads, 0, static_cast<cudaStream_t>(stream)>>>(normals, mask, and_edge, keep, H, W, kernel_size / 2, tol,
                                                                                out, angle);
    CUDA_TRY(cudaGetLastError());
    return 0;
}

int moge_mesh_count(const uint8_t* mask, int64_t batch, int H, int W, int64_t* totals, void* workspace, size_t workspace_bytes, void* stream) {
    if (!totals) return set_error("null argument");
    MG_TRY(check_batch_map("mesh_count", batch, H, W, kMaxPixels));
    const Layout l = layout(batch, H, W);
    MG_TRY(check_workspace(l.total, workspace, workspace_bytes, "mesh_count"));
    MG_TRY(check_device("mesh_count"));
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    char* ws = static_cast<char*>(workspace);
    const int tiles = num_tiles(H, W);
    int32_t* counts = reinterpret_cast<int32_t*>(ws + l.counts);
    count_kernel<<<dim3(tiles, static_cast<unsigned>(batch)), kThreads, 0, st>>>(mask, H, W, tiles, counts);
    CUDA_TRY(cudaGetLastError());
    scan_kernel<<<1, kScanThreads, 0, st>>>(counts, batch, tiles, reinterpret_cast<int32_t*>(ws + l.offsets), totals);
    CUDA_TRY(cudaGetLastError());
    return 0;
}

int moge_mesh_build(const uint8_t* mask, int64_t batch, int H, int W, int tri, const moge_mesh_map_t* maps, int num_maps,
                    const int64_t* totals, int32_t* faces, void* workspace, size_t workspace_bytes, void* stream) {
    if (!totals || !faces || (num_maps && !maps)) return set_error("null argument");
    MG_TRY(check_batch_map("mesh_build", batch, H, W, kMaxPixels));
    if (num_maps < 0 || num_maps > MOGE_MESH_MAX_MAPS) return set_error("mesh_build: %d maps is outside [0, %d]", num_maps, MOGE_MESH_MAX_MAPS);
    Maps ms;
    memset(&ms, 0, sizeof(ms));
    ms.n = num_maps;
    for (int k = 0; k < num_maps; ++k) {
        const moge_mesh_map_t& d = maps[k];
        if (d.kind < MOGE_MESH_F32 || d.kind > MOGE_MESH_UV) return set_error("mesh_build: map %d has unknown kind %d", k, d.kind);
        if (d.channels < 1 || d.channels > MOGE_MESH_MAX_CHANNELS) return set_error("mesh_build: map %d has %d channels", k, d.channels);
        if (d.kind == MOGE_MESH_UV ? d.channels != 2 : !d.src) return set_error("mesh_build: map %d: a UV map has 2 channels, other maps a source", k);
        if (d.layout != MOGE_MESH_HWC && d.layout != MOGE_MESH_CHW) return set_error("mesh_build: map %d has unknown layout %d", k, d.layout);
        if (!d.dst) return set_error("mesh_build: map %d has no destination", k);
        ms.m[k] = d;
    }
    const Layout l = layout(batch, H, W);
    MG_TRY(check_workspace(l.total, workspace, workspace_bytes, "mesh_build"));
    MG_TRY(check_device("mesh_build"));
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    char* ws = static_cast<char*>(workspace);
    const int tiles = num_tiles(H, W);
    const int32_t* offsets = reinterpret_cast<const int32_t*>(ws + l.offsets);
    int32_t* vmap = reinterpret_cast<int32_t*>(ws + l.vmap);
    const dim3 grid(tiles, static_cast<unsigned>(batch));
    vertices_kernel<<<grid, kThreads, 0, st>>>(mask, H, W, tiles, offsets, totals, ms, vmap);
    CUDA_TRY(cudaGetLastError());
    faces_kernel<<<grid, kThreads, 0, st>>>(mask, H, W, tiles, tri ? 1 : 0, offsets, totals, vmap, faces);
    CUDA_TRY(cudaGetLastError());
    return 0;
}

}  // extern "C"
