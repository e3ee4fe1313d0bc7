// The two ends of the DINOv2 backbone run on its own (moge_dino_*): the front end for an input that is already normalised, and
// the export of the residual stream after a requested block, with or without the final LayerNorm, in the caller's layout.
// Everything in between is the MoGe encoder's launch list (engine.cu).
#include "common.cuh"
#include "host_api.h"
#include "moge_b200.h"
#include <algorithm>

namespace mg {

// A call's shape groups, as the kernels see them: a table passed by value (__grid_constant__, read in place from the parameter
// bank), so a launch needs no upload and the phase-0 / phase-2 launches bind fresh pointers without touching a captured graph.
// The table holds MOGE_DINO_MAX_GROUPS entries.  A thread finds its group from its packed index: the last group whose first
// index is <= it (a binary search, 6 steps at most).
template <class First>
__device__ __forceinline__ int group_of(int n, First first, long key) {
    int lo = 0, hi = n - 1;
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (first(mid) <= key) lo = mid;
        else hi = mid - 1;
    }
    return lo;
}

// ------------------------------------------------------------------------------------------ front end
// dinov2/layers/patch_embed.py:68-81 as the patch-embed GEMM reads it: image (B,3,H,W), H = 14h, W = 14w, taken as it is (the
// backbone does no resize or normalisation of its own) -> A[B*T, 592] 16-bit, column c*196 + py*14 + px, columns 588..591 zero.
// One thread per (patch row, segment) over the patch rows of every group: segments 0..41 are the 14-pixel image rows (c, py) of
// the patch, read contiguously in the group's own dtype and stored as 7 packed pairs; segment 42 writes the 4 zero columns.
constexpr int kPatchSegs = 43;

struct PatchGroup {
    const void* image;
    int dtype, H, W, w, T;
    long row0;                     // first patch row of the group
};
struct PatchTable {
    PatchGroup g[MOGE_DINO_MAX_GROUPS];
    int n;
};

template <bool BF16>
__global__ void dino_patchify_kernel(const __grid_constant__ PatchTable tab, long rows, typename H16<BF16>::T* __restrict__ patches) {
    pdl_prologue();
    using Hx = H16<BF16>;
    const size_t total = static_cast<size_t>(rows) * kPatchSegs;
    for (size_t idx = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; idx < total;
         idx += static_cast<size_t>(gridDim.x) * blockDim.x) {
        const size_t row = idx / kPatchSegs;
        const int seg = static_cast<int>(idx - row * kPatchSegs);
        typename Hx::T* dst = patches + row * 592;
        if (seg == kPatchSegs - 1) {
            *reinterpret_cast<uint2*>(dst + 588) = make_uint2(0u, 0u);
            continue;
        }
        const PatchGroup& g = tab.g[group_of(tab.n, [&](int i) { return tab.g[i].row0; }, static_cast<long>(row))];
        const long r = static_cast<long>(row) - g.row0;
        const int b = static_cast<int>(r / g.T), t = static_cast<int>(r % g.T);
        const int c = seg / 14, py = seg % 14;
        const size_t src = (static_cast<size_t>(b) * 3 + c) * g.H * g.W + static_cast<size_t>((t / g.w) * 14 + py) * g.W + (t % g.w) * 14;
        uint32_t* out = reinterpret_cast<uint32_t*>(dst + c * 196 + py * 14);
#pragma unroll
        for (int px = 0; px < 14; px += 2) {
            float a, v;
            if (g.dtype == MOGE_F32) {
                const float* s = static_cast<const float*>(g.image) + src + px;
                a = s[0]; v = s[1];
            } else if (g.dtype == MOGE_F16) {
                const __half* s = static_cast<const __half*>(g.image) + src + px;
                a = __half2float(s[0]); v = __half2float(s[1]);
            } else {
                const __nv_bfloat16* s = static_cast<const __nv_bfloat16*>(g.image) + src + px;
                a = __bfloat162float(s[0]); v = __bfloat162float(s[1]);
            }
            out[px / 2] = Hx::pack(a, v);
        }
    }
}

int launch_dino_patchify(const DinoPatchIn* groups, int n, void* patches, bool bf16, cudaStream_t st) {
    if (n < 1 || n > MOGE_DINO_MAX_GROUPS) return set_error("dino patchify: %d groups out of range (1..%d)", n, MOGE_DINO_MAX_GROUPS);
    PatchTable tab{};
    tab.n = n;
    long rows = 0;
    for (int i = 0; i < n; ++i) {
        const DinoPatchIn& in = groups[i];
        if (in.H % 14 || in.W % 14)
            return set_error("dino patchify: group %d: %d x %d is not a multiple of the 14-pixel patch", i, in.H, in.W);
        PatchGroup& g = tab.g[i];
        g.image = in.image; g.dtype = in.image_dtype; g.H = in.H; g.W = in.W; g.w = in.W / 14; g.T = (in.H / 14) * g.w;
        g.row0 = rows;
        rows += static_cast<long>(in.B) * g.T;
    }
    const size_t total = static_cast<size_t>(rows) * kPatchSegs;
    const int threads = 256;
    const int blocks = static_cast<int>(std::min<size_t>((total + threads - 1) / threads, 132 * 16));
    if (bf16) CUDA_TRY(launch_pdl(dino_patchify_kernel<true>, dim3(blocks), dim3(threads), 0, st, tab, rows, static_cast<__nv_bfloat16*>(patches)));
    else CUDA_TRY(launch_pdl(dino_patchify_kernel<false>, dim3(blocks), dim3(threads), 0, st, tab, rows, static_cast<__half*>(patches)));
    CUDA_TRY(cudaGetLastError());
    return 0;
}

// ------------------------------------------------------------------------------------------ export
// vision_transformer.py:321-333 (get_intermediate_layers) and 274-281 (forward_features): the residual stream after a block, through
// the final LayerNorm (eps 1e-6, biased variance; gamma null: the raw rows), fp32.  A row's statistics come from one warp in a fixed
// order (each lane sums its float4s in order, then a butterfly), as layernorm_kernel computes them, and every element is formed with
// explicitly rounded operations, so both layouts give the same bits for the same row, whatever else is in the call.
template <int VEC>
__device__ __forceinline__ void row_stats(const float* __restrict__ xr, int D, int lane, float* mean, float* rstd) {
    const float4* x4 = reinterpret_cast<const float4*>(xr);
    float4 v[VEC];
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < VEC; ++i) {
        v[i] = x4[lane + 32 * i];
        s += v[i].x + v[i].y + v[i].z + v[i].w;
    }
    const float m = warp_sum(s) / D;
    float q = 0.f;
#pragma unroll
    for (int i = 0; i < VEC; ++i) {
        const float a = v[i].x - m, b = v[i].y - m, c = v[i].z - m, d = v[i].w - m;
        q += a * a + b * b + c * c + d * d;
    }
    *mean = m;
    *rstd = rsqrtf(warp_sum(q) / D + 1e-6f);
}

__device__ __forceinline__ float norm_elem(float v, float mean, float rstd, float g, float b) {
    return __fadd_rn(__fmul_rn(__fmul_rn(__fsub_rn(v, mean), rstd), g), b);
}

// one row by one warp: src row -> dst (D floats)
template <int VEC>
__device__ __forceinline__ void export_row(const float* __restrict__ xr, int D, const float* __restrict__ gamma,
                                           const float* __restrict__ beta, int lane, float* __restrict__ dst) {
    const float4* x4 = reinterpret_cast<const float4*>(xr);
    float4* d4 = reinterpret_cast<float4*>(dst);
    if (!gamma) {
#pragma unroll
        for (int i = 0; i < VEC; ++i) d4[lane + 32 * i] = x4[lane + 32 * i];
        return;
    }
    float mean, rstd;
    row_stats<VEC>(xr, D, lane, &mean, &rstd);
#pragma unroll
    for (int i = 0; i < VEC; ++i) {
        const int c4 = lane + 32 * i;
        const float4 v = x4[c4];
        const float4 g = reinterpret_cast<const float4*>(gamma)[c4];
        const float4 b = reinterpret_cast<const float4*>(beta)[c4];
        d4[c4] = make_float4(norm_elem(v.x, mean, rstd, g.x, b.x), norm_elem(v.y, mean, rstd, g.y, b.y),
                             norm_elem(v.z, mean, rstd, g.z, b.z), norm_elem(v.w, mean, rstd, g.w, b.w));
    }
}

constexpr int kExportTile = 32;

struct ExportGroup {
    float* tokens; float* cls;
    long row0;                     // first row of the group in x
    int N;
    int tiles;                     // channel-major: 32-token tiles per image (the class row's block comes after them)
    int blk0;                      // channel-major: the group's first block
};
struct ExportTable {
    ExportGroup g[MOGE_DINO_MAX_GROUPS];
    int n;
};

// Token-major: one warp per packed row of x (the groups' B*N rows back to back, each image's class token first); patch row (b, t)
// of a group -> its tokens[(b*T + t)*D], class row of image b -> its cls[b*D].  Either output may be null.
template <int VEC>
__global__ void dino_export_rows_kernel(const __grid_constant__ ExportTable tab, const float* __restrict__ x, long rows, int D,
                                        const float* __restrict__ gamma, const float* __restrict__ beta) {
    pdl_prologue();
    const long r = (blockIdx.x * static_cast<long>(blockDim.x) + threadIdx.x) >> 5;
    if (r >= rows) return;
    const ExportGroup& g = tab.g[group_of(tab.n, [&](int i) { return tab.g[i].row0; }, r)];
    const long lr = r - g.row0;
    const int b = static_cast<int>(lr / g.N), n = static_cast<int>(lr % g.N);
    float* dst = n == 0 ? (g.cls ? g.cls + static_cast<size_t>(b) * D : nullptr)
                        : (g.tokens ? g.tokens + (static_cast<size_t>(b) * (g.N - 1) + n - 1) * D : nullptr);
    if (dst) export_row<VEC>(x + static_cast<size_t>(r) * D, D, gamma, beta, threadIdx.x & 31, dst);
}

// Channel-major: per image of every group, `tiles` blocks of 32 patch tokens, then one block for the class row.  A tile block's
// warps first compute the tile's row statistics, then the block walks the channels 32 at a time: a 32 x 32 tile is read along the
// channels, normalised into shared memory and written along the tokens to tokens[(b*D + d)*T + t], both sides coalesced.  The
// tile's 32 rows (128 KB at D = 1024) are read from HBM by the statistics and again, right after, by the transpose, which finds
// them in L2: no second pass over HBM.  The class block writes the class row of image b (cls may be null; tokens too, then only
// that block works).
template <int VEC>
__global__ void __launch_bounds__(256) dino_export_chw_kernel(const __grid_constant__ ExportTable tab, const float* __restrict__ x, int D,
                                                             const float* __restrict__ gamma, const float* __restrict__ beta) {
    pdl_prologue();
    __shared__ float tile[kExportTile][kExportTile + 1];
    __shared__ float s_mean[kExportTile], s_rstd[kExportTile];
    const ExportGroup& g = tab.g[group_of(tab.n, [&](int i) { return static_cast<long>(tab.g[i].blk0); }, blockIdx.x)];
    const int local = blockIdx.x - g.blk0;
    const int b = local / (g.tiles + 1), tb = local % (g.tiles + 1);
    const int T = g.N - 1;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nwarps = blockDim.x >> 5;
    const float* xb = x + (g.row0 + static_cast<size_t>(b) * g.N) * D;
    if (tb == g.tiles) {
        if (g.cls && warp == 0) export_row<VEC>(xb, D, gamma, beta, lane, g.cls + static_cast<size_t>(b) * D);
        return;
    }
    float* tokens = g.tokens;
    if (!tokens) return;
    const int t0 = tb * kExportTile;
    if (gamma) {
        for (int r = warp; r < kExportTile; r += nwarps) {
            const int t = min(t0 + r, T - 1);          // rows past the image's end: any valid row, never stored
            float mean, rstd;
            row_stats<VEC>(xb + static_cast<size_t>(1 + t) * D, D, lane, &mean, &rstd);
            if (lane == 0) { s_mean[r] = mean; s_rstd[r] = rstd; }
        }
        __syncthreads();
    }
    for (int d0 = 0; d0 < D; d0 += kExportTile) {
        const int d = d0 + lane;
        for (int r = warp; r < kExportTile; r += nwarps) {
            const int t = t0 + r;
            if (t < T) {
                const float v = xb[static_cast<size_t>(1 + t) * D + d];
                tile[r][lane] = gamma ? norm_elem(v, s_mean[r], s_rstd[r], gamma[d], beta[d]) : v;
            }
        }
        __syncthreads();
        const int t = t0 + lane;
        if (t < T)
            for (int c = warp; c < kExportTile; c += nwarps) tokens[(static_cast<size_t>(b) * D + d0 + c) * T + t] = tile[lane][c];
        __syncthreads();
    }
}

int launch_dino_export(const float* x, const DinoExportOut* groups, int n, int D, const float* gamma, const float* beta,
                       bool channel_major, cudaStream_t st) {
    if (D % 128 || D > 1024) return set_error("dino export: D=%d unsupported (a multiple of 128, <= 1024)", D);
    if (n < 1 || n > MOGE_DINO_MAX_GROUPS) return set_error("dino export: %d groups out of range (1..%d)", n, MOGE_DINO_MAX_GROUPS);
    ExportTable tab{};
    tab.n = n;
    long rows = 0, blocks = 0;
    bool any = false;
    for (int i = 0; i < n; ++i) {
        const DinoExportOut& o = groups[i];
        ExportGroup& g = tab.g[i];
        g.tokens = o.tokens; g.cls = o.cls; g.row0 = rows; g.N = o.N;
        g.tiles = (o.N - 1 + kExportTile - 1) / kExportTile;
        g.blk0 = static_cast<int>(blocks);
        rows += static_cast<long>(o.B) * o.N;
        blocks += static_cast<long>(o.B) * (g.tiles + 1);
        any = any || o.tokens || o.cls;
    }
    if (!any) return 0;
    if (blocks > 0x7fffffffL) return set_error("dino export: %ld blocks exceed one grid", blocks);
    const int threads = 256;
    cudaError_t ce = cudaSuccess;
#define DINO_EXPORT_CASE(V)                                                                                                       \
    case V:                                                                                                                       \
        if (channel_major)                                                                                                        \
            ce = launch_pdl(dino_export_chw_kernel<V>, dim3(static_cast<unsigned>(blocks)), dim3(threads), 0, st, tab, x, D,      \
                            gamma, beta);                                                                                         \
        else                                                                                                                      \
            ce = launch_pdl(dino_export_rows_kernel<V>, dim3(static_cast<unsigned>((rows + threads / 32 - 1) / (threads / 32))),  \
                            dim3(threads), 0, st, tab, x, rows, D, gamma, beta);                                                  \
        break;
    switch (D / 128) {
        DINO_EXPORT_CASE(1) DINO_EXPORT_CASE(2) DINO_EXPORT_CASE(3) DINO_EXPORT_CASE(4)
        DINO_EXPORT_CASE(5) DINO_EXPORT_CASE(6) DINO_EXPORT_CASE(7) DINO_EXPORT_CASE(8)
    }
#undef DINO_EXPORT_CASE
    if (ce != cudaSuccess) return set_error("dino export launch failed: %s", cudaGetErrorString(ce));
    CUDA_TRY(cudaGetLastError());
    return 0;
}

}  // namespace mg
