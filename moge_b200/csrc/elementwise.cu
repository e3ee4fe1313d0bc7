// HBM-bound kernels around the tensor-core path: input resize/normalise/patchify, pos-embed resampling, LayerNorm,
// scale-head MLP, fused output resize + remap, focal/shift recovery, post-processing.
// Each kernel cites the reference lines it restates (paths relative to /root/reference).
#include "common.cuh"
#include "host_api.h"
#include <math.h>
#include <algorithm>

namespace mg {

// ------------------------------------------------------------------------------------------ K1 preprocess
// moge/model/modules.py:121-122 (F.interpolate bilinear antialias=True to (14h,14w); (x-mean)/std) and the im2col of
// dinov2/layers/patch_embed.py:68-81.  Triangle-filter weights as ATen _upsample_bilinear2d_aa (SURVEY.md app. B-2).
__device__ __forceinline__ float load_img(const void* img, int dtype, size_t idx) {
    if (dtype == 0) return static_cast<const float*>(img)[idx];
    if (dtype == 1) return __half2float(static_cast<const __half*>(img)[idx]);
    return __bfloat162float(static_cast<const __nv_bfloat16*>(img)[idx]);
}

struct AAFilter { int lo, n; float scale, support, inv; };
__device__ __forceinline__ AAFilter aa_setup(int in, int out, int i, float& center) {
    AAFilter f;
    f.scale = static_cast<float>(in) / static_cast<float>(out);
    f.support = (f.scale >= 1.0f) ? f.scale : 1.0f;
    f.inv = (f.scale >= 1.0f) ? 1.0f / f.scale : 1.0f;
    center = f.scale * (i + 0.5f);
    f.lo = max(static_cast<int>(center - f.support + 0.5f), 0);
    const int hi = min(static_cast<int>(center + f.support + 0.5f), in);
    f.n = hi - f.lo;
    return f;
}
__device__ __forceinline__ float aa_w(const AAFilter& f, float center, int j) {
    const float w = 1.0f - fabsf((j + f.lo - center + 0.5f) * f.inv);
    return w > 0.f ? w : 0.f;
}

template <bool BF16>
__global__ void preprocess_kernel(const void* __restrict__ image, int dtype, int B, int H, int W, int h, int w,
                                  typename H16<BF16>::T* __restrict__ patches, int Kp) {
    pdl_prologue();
    const int T = h * w;
    const size_t total = static_cast<size_t>(B) * T * Kp;
    const float mean[3] = {0.485f, 0.456f, 0.406f};
    const float stdv[3] = {0.229f, 0.224f, 0.225f};
    for (size_t idx = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; idx < total;
         idx += static_cast<size_t>(gridDim.x) * blockDim.x) {
        const int k = static_cast<int>(idx % Kp);
        const size_t row = idx / Kp;
        float val = 0.f;
        if (k < 588) {
            const int b = static_cast<int>(row / T), t = static_cast<int>(row % T);
            const int c = k / 196, py = (k % 196) / 14, px = k % 14;
            const int Y = (t / w) * 14 + py, X = (t % w) * 14 + px;
            const int OH = h * 14, OW = w * 14;
            const size_t plane0 = (static_cast<size_t>(b) * 3 + c) * H * W;
            if (H == OH && W == OW) {                         // native grid (e.g. 518 px @ 37x37): the resize is the identity
                patches[idx] = H16<BF16>::from_float((load_img(image, dtype, plane0 + static_cast<size_t>(Y) * W + X) - mean[c]) / stdv[c]);
                continue;
            }
            float cy, cx;
            const AAFilter fy = aa_setup(H, OH, Y, cy);
            const AAFilter fx = aa_setup(W, OW, X, cx);
            float wys = 0.f, wxs = 0.f;
            for (int j = 0; j < fy.n; ++j) wys += aa_w(fy, cy, j);
            for (int i = 0; i < fx.n; ++i) wxs += aa_w(fx, cx, i);
            const size_t plane = (static_cast<size_t>(b) * 3 + c) * H * W;
            float acc = 0.f;
            for (int j = 0; j < fy.n; ++j) {
                const float wy = aa_w(fy, cy, j) / wys;
                float rowacc = 0.f;
                for (int i = 0; i < fx.n; ++i)
                    rowacc += (aa_w(fx, cx, i) / wxs) * load_img(image, dtype, plane + static_cast<size_t>(fy.lo + j) * W + fx.lo + i);
                acc += wy * rowacc;
            }
            val = (acc - mean[c]) / stdv[c];
        }
        patches[idx] = H16<BF16>::from_float(val);
    }
}

int launch_preprocess(const void* image, int image_dtype, int B, int H, int W, int h, int w, void* patches, int Kp,
                      bool bf16, cudaStream_t st) {
    const size_t total = static_cast<size_t>(B) * h * w * Kp;
    const int threads = 256;
    const int blocks = static_cast<int>(std::min<size_t>((total + threads - 1) / threads, 132 * 16));
    if (bf16) CUDA_TRY(launch_pdl(preprocess_kernel<true>, dim3(blocks), dim3(threads), 0, st, image, image_dtype, B, H, W, h, w, static_cast<__nv_bfloat16*>(patches), Kp));
    else CUDA_TRY(launch_pdl(preprocess_kernel<false>, dim3(blocks), dim3(threads), 0, st, image, image_dtype, B, H, W, h, w, static_cast<__half*>(patches), Kp));
    CUDA_TRY(cudaGetLastError());
    return 0;
}

// ------------------------------------------------------------------------------------------ K3 pos table
// dinov2/models/vision_transformer.py:187-221: bicubic (A=-0.75, align_corners=False) resampling of the 37x37
// pos-embed grid with scale_factor=((h+0.1)/37,(w+0.1)/37)  => source = (dst+0.5)*37/(h+0.1) - 0.5, taps clamped;
// returned unchanged when h == w == 37.  The patch-embed bias is folded into the table.
__device__ __forceinline__ void cubic_coeffs(float t, float* c) {
    const float A = -0.75f;
    float x = t + 1.0f;
    c[0] = ((A * x - 5.0f * A) * x + 8.0f * A) * x - 4.0f * A;
    x = t;
    c[1] = ((A + 2.0f) * x - (A + 3.0f)) * x * x + 1.0f;
    x = 1.0f - t;
    c[2] = ((A + 2.0f) * x - (A + 3.0f)) * x * x + 1.0f;
    x = 2.0f - t;
    c[3] = ((A * x - 5.0f * A) * x + 8.0f * A) * x - 4.0f * A;
}

__global__ void pos_table_kernel(const float* __restrict__ pos, const float* __restrict__ cls, const float* __restrict__ pbias,
                                 int D, int h, int w, float* __restrict__ table, float* __restrict__ cls_row) {
    const int M = 37;
    const int t = blockIdx.x;           // 0..h*w  (last block: the cls row)
    if (t == h * w) {
        for (int d = threadIdx.x; d < D; d += blockDim.x) cls_row[d] = cls[d] + pos[d];
        return;
    }
    const int oy = t / w, ox = t % w;
    const float* grid = pos + D;        // skip the cls position
    if (h == M && w == M) {
        for (int d = threadIdx.x; d < D; d += blockDim.x) table[static_cast<size_t>(t) * D + d] = grid[static_cast<size_t>(t) * D + d] + pbias[d];
        return;
    }
    const float ry = static_cast<float>(1.0 / ((h + 0.1) / static_cast<double>(M)));   // ATen: float(1 / scale_factor)
    const float rx = static_cast<float>(1.0 / ((w + 0.1) / static_cast<double>(M)));
    const float sy = ry * (oy + 0.5f) - 0.5f, sx = rx * (ox + 0.5f) - 0.5f;
    const int iy = static_cast<int>(floorf(sy)), ix = static_cast<int>(floorf(sx));
    float cy[4], cx[4];
    cubic_coeffs(sy - iy, cy);
    cubic_coeffs(sx - ix, cx);
    for (int d = threadIdx.x; d < D; d += blockDim.x) {
        float acc = 0.f;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int yy = min(max(iy - 1 + j, 0), M - 1);
            float r = 0.f;
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const int xx = min(max(ix - 1 + i, 0), M - 1);
                r += cx[i] * grid[(static_cast<size_t>(yy) * M + xx) * D + d];
            }
            acc += cy[j] * r;
        }
        table[static_cast<size_t>(t) * D + d] = acc + pbias[d];
    }
}

int launch_pos_table(const float* pos_embed, const float* cls_token, const float* patch_bias, int D, int h, int w,
                     float* table, float* cls_row, cudaStream_t st) {
    pos_table_kernel<<<h * w + 1, 128, 0, st>>>(pos_embed, cls_token, patch_bias, D, h, w, table, cls_row);
    CUDA_TRY(cudaGetLastError());
    return 0;
}

__global__ void init_cls_kernel(float* __restrict__ x, const float* __restrict__ cls_row, int B, int N, int D) {
    pdl_prologue();
    const int b = blockIdx.x;
    for (int d = threadIdx.x; d < D; d += blockDim.x) x[static_cast<size_t>(b) * N * D + d] = cls_row[d];
}
int launch_init_cls(float* x, const float* cls_row, int B, int N, int D, cudaStream_t st) {
    CUDA_TRY(launch_pdl(init_cls_kernel, dim3(B), dim3(256), 0, st, x, cls_row, B, N, D));
    CUDA_TRY(cudaGetLastError());
    return 0;
}

// ------------------------------------------------------------------------------------------ LayerNorm folded into the next GEMM
// LN(x) W^T + b = rstd * ((x - mu 1) W'^T) + b' = rstd * (x W''^T) + b'
//   with  W' = W diag(gamma),  W'' = W' (I - 1 1^T / D)  (every row of W' centred: the mean removal is a linear map and lives
//   in the weight),  b' = b + W beta.
// The GEMM consumes the ROUNDED residual rows x16 directly and its epilogue only scales by rstd[row] and adds b' -- the same
// instruction count as a plain bias epilogue (an explicit rank-1 mean correction would add work to every output element of the
// qkv / fc1 GEMMs).  rstd comes from per-row partial sums (sum, sum of squares
// of the rounded values) that the producing epilogue (patch embed, proj, fc2) writes next to x16, reduced by ln_rstd_kernel.
// Rounding W'' to 16 bit leaves a column-sum residual of ~sqrt(D) * 2^-11 * |W''|: the mean is removed to that relative
// precision, which is below the 16-bit rounding of the activations for |mu| <~ 10 sigma.
template <bool BF16>
__global__ void ln_prepare_kernel(const float* __restrict__ x, long row_stride, int D, typename H16<BF16>::T* __restrict__ x16,
                                  long row_stride16, float2* __restrict__ stats, long stats_stride, int parts) {
    pdl_prologue();
    using H = H16<BF16>;
    const long r = blockIdx.x;
    const float* xr = x + r * row_stride;
    float s1 = 0.f, s2 = 0.f;
    for (int d = 2 * threadIdx.x; d < D; d += 2 * blockDim.x) {
        const uint32_t pk = H::pack(xr[d], xr[d + 1]);
        *reinterpret_cast<uint32_t*>(x16 + r * row_stride16 + d) = pk;
        const float2 f = H::unpack(pk);
        s1 += f.x + f.y; s2 += f.x * f.x + f.y * f.y;
    }
    __shared__ float red[2][32];
    for (int o = 16; o > 0; o >>= 1) { s1 += __shfl_xor_sync(0xffffffffu, s1, o); s2 += __shfl_xor_sync(0xffffffffu, s2, o); }
    if ((threadIdx.x & 31) == 0) { red[0][threadIdx.x >> 5] = s1; red[1][threadIdx.x >> 5] = s2; }
    __syncthreads();
    if (threadIdx.x == 0) {
        float a = 0.f, b = 0.f;
        for (int w = 0; w < (blockDim.x >> 5); ++w) { a += red[0][w]; b += red[1][w]; }
        stats[r * stats_stride] = make_float2(a, b);
        for (int pp = 1; pp < parts; ++pp) stats[r * stats_stride + pp] = make_float2(0.f, 0.f);
    }
}
int launch_ln_prepare(const float* x, int rows, long row_stride, int D, void* x16, long row_stride16, float2* stats, long stats_stride,
                      int parts, bool bf16, cudaStream_t st) {
    if (D % 2) return set_error("ln_prepare: D must be even");
    if (rows <= 0) return 0;
    if (bf16) CUDA_TRY(launch_pdl(ln_prepare_kernel<true>, dim3(rows), dim3(128), 0, st, x, row_stride, D, static_cast<__nv_bfloat16*>(x16), row_stride16, stats, stats_stride, parts));
    else CUDA_TRY(launch_pdl(ln_prepare_kernel<false>, dim3(rows), dim3(128), 0, st, x, row_stride, D, static_cast<__half*>(x16), row_stride16, stats, stats_stride, parts));
    CUDA_TRY(cudaGetLastError());
    return 0;
}

// per-row rstd from the partial sums: rstd[r] = 1 / sqrt(E[x^2] - E[x]^2 + 1e-6)
__global__ void ln_rstd_kernel(const float2* __restrict__ stats, int ld, int parts, int rows, float inv_d, float* __restrict__ rstd) {
    pdl_prologue();
    const int r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= rows) return;
    float a = 0.f, b = 0.f;
    for (int pp = 0; pp < parts; ++pp) { const float2 t = stats[static_cast<size_t>(r) * ld + pp]; a += t.x; b += t.y; }
    const float mean = a * inv_d;
    rstd[r] = rsqrtf(fmaxf(b * inv_d - mean * mean, 0.f) + 1e-6f);
}
int launch_ln_rstd(const float2* stats, int ld, int parts, int rows, int D, float* rstd, cudaStream_t st) {
    if (rows <= 0) return 0;
    CUDA_TRY(launch_pdl(ln_rstd_kernel, dim3((rows + 255) / 256), dim3(256), 0, st, stats, ld, parts, rows, 1.0f / static_cast<float>(D), rstd));
    CUDA_TRY(cudaGetLastError());
    return 0;
}

// one block per output feature n: c = mean_k(W[n,k] gamma[k]);  w16[n,k] = T(W[n,k] gamma[k] - c);  b2[n] = b[n] + sum_k W[n,k] beta[k]
template <bool BF16>
__global__ void ln_fold_kernel(const float* __restrict__ W, const float* __restrict__ gamma, const float* __restrict__ beta,
                               const float* __restrict__ bias, int K, int ldw, typename H16<BF16>::T* __restrict__ w16,
                               float* __restrict__ b2) {
    using H = H16<BF16>;
    const int n = blockIdx.x;
    float s = 0.f, t = 0.f;
    for (int k = threadIdx.x; k < K; k += blockDim.x) {
        const float w = W[static_cast<size_t>(n) * K + k];
        s += w * gamma[k];
        t += w * beta[k];
    }
    __shared__ float red[2][32];
    __shared__ float centre;
    for (int o = 16; o > 0; o >>= 1) { s += __shfl_xor_sync(0xffffffffu, s, o); t += __shfl_xor_sync(0xffffffffu, t, o); }
    if ((threadIdx.x & 31) == 0) { red[0][threadIdx.x >> 5] = s; red[1][threadIdx.x >> 5] = t; }
    __syncthreads();
    if (threadIdx.x == 0) {
        float a = 0.f, b = 0.f;
        for (int w = 0; w < (blockDim.x >> 5); ++w) { a += red[0][w]; b += red[1][w]; }
        centre = a / static_cast<float>(K);
        b2[n] = (bias ? bias[n] : 0.f) + b;
    }
    __syncthreads();
    const float c = centre;
    for (int k = 2 * threadIdx.x; k < K; k += 2 * blockDim.x) {
        const float w0 = W[static_cast<size_t>(n) * K + k], w1 = W[static_cast<size_t>(n) * K + k + 1];
        *reinterpret_cast<uint32_t*>(w16 + static_cast<size_t>(n) * ldw + k) = H::pack(w0 * gamma[k] - c, w1 * gamma[k + 1] - c);
    }
}
int launch_ln_fold(const float* W, const float* gamma, const float* beta, const float* bias, int N, int K, int ldw, void* w16,
                   float* b2, bool bf16, cudaStream_t st) {
    if (K % 2) return set_error("ln_fold: K must be even");
    if (bf16) ln_fold_kernel<true><<<N, 128, 0, st>>>(W, gamma, beta, bias, K, ldw, static_cast<__nv_bfloat16*>(w16), b2);
    else ln_fold_kernel<false><<<N, 128, 0, st>>>(W, gamma, beta, bias, K, ldw, static_cast<__half*>(w16), b2);
    CUDA_TRY(cudaGetLastError());
    return 0;
}

// ------------------------------------------------------------------------------------------ LayerNorm
// torch LayerNorm (biased variance, eps 1e-6; vision_transformer.py:95) on the fp32 residual stream -> 16-bit GEMM
// operand.  One warp per row, row held in registers (D <= 1024), two-pass statistics by warp shuffles.
template <bool BF16, int VEC>   // VEC = D / 128 float4 per lane
__global__ void layernorm_kernel(const float* __restrict__ x, const float* __restrict__ gamma, const float* __restrict__ beta,
                                 typename H16<BF16>::T* __restrict__ out, int rows, int D, int ld_out, int col_off, int mode,
                                 int N, float* __restrict__ cls_out) {
    pdl_prologue();
    const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (warp >= rows) return;
    const float4* xr = reinterpret_cast<const float4*>(x + static_cast<size_t>(warp) * D);
    float4 v[VEC];
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < VEC; ++i) {
        v[i] = xr[lane + 32 * i];
        s += v[i].x + v[i].y + v[i].z + v[i].w;
    }
    const float mean = warp_sum(s) / D;
    float q = 0.f;
#pragma unroll
    for (int i = 0; i < VEC; ++i) {
        const float a = v[i].x - mean, b = v[i].y - mean, c = v[i].z - mean, d = v[i].w - mean;
        q += a * a + b * b + c * c + d * d;
    }
    const float rstd = rsqrtf(warp_sum(q) / D + 1e-6f);
    size_t orow = warp;
    bool is_cls = false;
    if (mode == 1) {
        const int b = warp / N, n = warp % N;
        is_cls = (n == 0);
        orow = static_cast<size_t>(b) * (N - 1) + (n - 1);
        if (is_cls && cls_out == nullptr) return;
        if (is_cls) orow = b;
    }
#pragma unroll
    for (int i = 0; i < VEC; ++i) {
        const int c4 = lane + 32 * i;
        const float4 g = reinterpret_cast<const float4*>(gamma)[c4];
        const float4 bt = reinterpret_cast<const float4*>(beta)[c4];
        const float a = (v[i].x - mean) * rstd * g.x + bt.x, b = (v[i].y - mean) * rstd * g.y + bt.y;
        const float c = (v[i].z - mean) * rstd * g.z + bt.z, d = (v[i].w - mean) * rstd * g.w + bt.w;
        if (is_cls) {
            reinterpret_cast<float4*>(cls_out + orow * D)[c4] = make_float4(a, b, c, d);
        } else {
            uint2 pk;
            pk.x = H16<BF16>::pack(a, b);
            pk.y = H16<BF16>::pack(c, d);
            *reinterpret_cast<uint2*>(out + orow * ld_out + col_off + 4 * c4) = pk;
        }
    }
}

int launch_layernorm(const float* x, const float* gamma, const float* beta, void* out, int rows, int D, int ld_out,
                     int col_off, int mode, int tokens_per_image, float* cls_out, bool bf16, cudaStream_t st) {
    if (D % 128 != 0 || D > 1024) return set_error("layernorm: D=%d unsupported (need D %% 128 == 0, D <= 1024)", D);
    const int threads = 256, wpb = threads / 32;
    const int blocks = (rows + wpb - 1) / wpb;
#define LN_CASE(V)                                                                                                        \
    case V:                                                                                                               \
        if (bf16) { if (launch_pdl(layernorm_kernel<true, V>, dim3(blocks), dim3(threads), 0, st, x, gamma, beta, static_cast<__nv_bfloat16*>(out), rows, D, ld_out, col_off, mode, tokens_per_image, cls_out) != cudaSuccess) return set_error("layernorm launch failed"); } \
        else { if (launch_pdl(layernorm_kernel<false, V>, dim3(blocks), dim3(threads), 0, st, x, gamma, beta, static_cast<__half*>(out), rows, D, ld_out, col_off, mode, tokens_per_image, cls_out) != cudaSuccess) return set_error("layernorm launch failed"); }       \
        break;
    switch (D / 128) {
        LN_CASE(1) LN_CASE(2) LN_CASE(3) LN_CASE(4) LN_CASE(5) LN_CASE(6) LN_CASE(7) LN_CASE(8)
    }
#undef LN_CASE
    CUDA_TRY(cudaGetLastError());
    return 0;
}

// ------------------------------------------------------------------------------------------ scale head
// moge/model/modules.py:184-192 + v2.py:167,182: exp(W3 relu(W2 relu(W1 cls + b1) + b2) + b3).  Warp per output row.
__global__ void mlp_layer_kernel(const float* __restrict__ in, const float* __restrict__ W, const float* __restrict__ bias,
                                 float* __restrict__ out, int din, int dout, int relu, int do_exp) {
    pdl_prologue();
    const int b = blockIdx.y;
    const int j = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (j >= dout) return;
    const float* xr = in + static_cast<size_t>(b) * din;
    const float* wr = W + static_cast<size_t>(j) * din;
    float s = 0.f;
    for (int i = lane; i < din; i += 32) s += wr[i] * xr[i];
    s = warp_sum(s);
    if (lane == 0) {
        s += bias[j];
        if (relu) s = fmaxf(s, 0.f);
        if (do_exp) s = expf(s);
        out[static_cast<size_t>(b) * dout + j] = s;
    }
}
int launch_scale_head(const float* cls, const float* const* w, const float* const* bias, const int* dims, int nlayers,
                      int B, float* out, float* scratch, cudaStream_t st) {
    const float* cur = cls;
    int maxd = 0;
    for (int i = 0; i <= nlayers; ++i) maxd = dims[i] > maxd ? dims[i] : maxd;
    for (int l = 0; l < nlayers; ++l) {
        const bool last = (l == nlayers - 1);
        float* dst = last ? out : scratch + static_cast<size_t>(l & 1) * B * maxd;
        dim3 grid((dims[l + 1] + 7) / 8, B);
        CUDA_TRY(launch_pdl(mlp_layer_kernel, grid, dim3(256), 0, st, cur, w[l], bias[l], dst, dims[l], dims[l + 1], last ? 0 : 1, last ? 1 : 0));
        cur = dst;
    }
    CUDA_TRY(cudaGetLastError());
    return 0;
}

// ------------------------------------------------------------------------------------------ K17 head output
// v2.py:170-182: bilinear resize (align_corners=False, antialias=False) of the 16x-grid head maps to (H,W), then
// points remap (v2.py:122-136), F.normalize(eps=1e-12) of the normals, sigmoid of the mask logit.
__global__ void head_output_kernel(const float4* __restrict__ pts, const float4* __restrict__ nrm, const float* __restrict__ msk,
                                   int B, int Hl, int Wl, int H, int W, int remap, float* __restrict__ points,
                                   float* __restrict__ normal, float* __restrict__ mask) {
    pdl_prologue();
    const size_t total = static_cast<size_t>(B) * H * W;
    const float rh = static_cast<float>(Hl) / H, rw = static_cast<float>(Wl) / W;
    for (size_t idx = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; idx < total;
         idx += static_cast<size_t>(gridDim.x) * blockDim.x) {
        const int X = static_cast<int>(idx % W);
        const int Y = static_cast<int>((idx / W) % H);
        const int b = static_cast<int>(idx / (static_cast<size_t>(W) * H));
        const float sy = fmaxf(rh * (Y + 0.5f) - 0.5f, 0.f), sx = fmaxf(rw * (X + 0.5f) - 0.5f, 0.f);
        const int y0 = min(static_cast<int>(sy), Hl - 1), x0 = min(static_cast<int>(sx), Wl - 1);
        const int y1 = min(y0 + 1, Hl - 1), x1 = min(x0 + 1, Wl - 1);
        const float ly = sy - y0, lx = sx - x0;
        const float w00 = (1.f - ly) * (1.f - lx), w01 = (1.f - ly) * lx, w10 = ly * (1.f - lx), w11 = ly * lx;
        const size_t base = static_cast<size_t>(b) * Hl * Wl;
        const size_t i00 = base + static_cast<size_t>(y0) * Wl + x0, i01 = base + static_cast<size_t>(y0) * Wl + x1;
        const size_t i10 = base + static_cast<size_t>(y1) * Wl + x0, i11 = base + static_cast<size_t>(y1) * Wl + x1;
        if (pts != nullptr) {
            const float4 a = pts[i00], bq = pts[i01], c = pts[i10], d = pts[i11];
            float x = w00 * a.x + w01 * bq.x + w10 * c.x + w11 * d.x;
            float y = w00 * a.y + w01 * bq.y + w10 * c.y + w11 * d.y;
            float z = w00 * a.z + w01 * bq.z + w10 * c.z + w11 * d.z;
            if (remap == 1) { x = sinhf(x); y = sinhf(y); z = sinhf(z); }
            else if (remap == 2) { z = expf(z); x *= z; y *= z; }
            else if (remap == 3) { x = sinhf(x); y = sinhf(y); z = expf(z); }
            points[idx * 3] = x; points[idx * 3 + 1] = y; points[idx * 3 + 2] = z;
        }
        if (nrm != nullptr) {
            const float4 a = nrm[i00], bq = nrm[i01], c = nrm[i10], d = nrm[i11];
            const float x = w00 * a.x + w01 * bq.x + w10 * c.x + w11 * d.x;
            const float y = w00 * a.y + w01 * bq.y + w10 * c.y + w11 * d.y;
            const float z = w00 * a.z + w01 * bq.z + w10 * c.z + w11 * d.z;
            const float inv = 1.0f / fmaxf(sqrtf(x * x + y * y + z * z), 1e-12f);
            normal[idx * 3] = x * inv; normal[idx * 3 + 1] = y * inv; normal[idx * 3 + 2] = z * inv;
        }
        if (msk != nullptr) {
            const float m = w00 * msk[i00] + w01 * msk[i01] + w10 * msk[i10] + w11 * msk[i11];
            mask[idx] = 1.0f / (1.0f + expf(-m));
        }
    }
}
int launch_head_output(const float4* pts_lr, const float4* nrm_lr, const float* msk_lr, int B, int Hl, int Wl, int H, int W,
                       int remap_mode, float* points, float* normal, float* mask, cudaStream_t st) {
    const size_t total = static_cast<size_t>(B) * H * W;
    const int threads = 256;
    const int blocks = static_cast<int>(std::min<size_t>((total + threads - 1) / threads, 132 * 16));
    CUDA_TRY(launch_pdl(head_output_kernel, dim3(blocks), dim3(threads), 0, st, pts_lr, nrm_lr, msk_lr, B, Hl, Wl, H, W, remap_mode, points, normal, mask));
    CUDA_TRY(cudaGetLastError());
    return 0;
}

// ------------------------------------------------------------------------------------------ K18 focal / shift
// moge/utils/geometry_torch.py:115-170 + geometry_numpy.py:79-112.  The reference syncs to the host and runs SciPy
// MINPACK-LM per image; here one CTA per image gathers the 64x64 nearest samples and runs a damped Gauss-Newton on
// the 1-D shift (focal in closed form inside the residual), all reductions on chip, fp64 accumulation like SciPy.
constexpr int FS_THREADS = 256;
constexpr int FS_PER_THREAD = 4096 / FS_THREADS;

__device__ __forceinline__ double block_sum(double v, double* red) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    __syncthreads();
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
    __syncthreads();
    double t = 0.0;
#pragma unroll
    for (int i = 0; i < FS_THREADS / 32; ++i) t += red[i];
    return t;
}

struct FsEval { double cost, jtr, jtj, focal; };

// Residuals r(s) = f(s) q - uv with q = xy/(z+s) (f in closed form or given).  Returns cost = |r(s)|^2 and, when
// `with_jac`, J^T r and J^T J for the forward-difference Jacobian J = (r(s+h) - r(s)) / h the reference's solver uses
// (SciPy's 2-point step): near the poles z + s = 0 of ill-posed maps the analytic and
// the finite-difference Jacobians differ a lot, and parity with the reference means following ITS iterates.
__device__ FsEval fs_eval(double s, bool with_jac, const float* x, const float* y, const float* z, const float* u, const float* v,
                          unsigned valid, bool fixed_focal, double focal_given, double* red) {
    // SciPy >= 1.x drives MINPACK lmder with its own 2-point Jacobian: h = sqrt(eps) * sign(s) * max(1, |s|)
    const double h = 1.4901161193847656e-08 * (s < 0.0 ? -1.0 : 1.0) * fmax(1.0, fabs(s));
    const double s2 = s + h;
    double a = 0, bq = 0, a2 = 0, bq2 = 0;
#pragma unroll
    for (int i = 0; i < FS_PER_THREAD; ++i)
        if (valid >> i & 1) {
            const double inv = 1.0 / (static_cast<double>(z[i]) + s);
            const double qx = x[i] * inv, qy = y[i] * inv;
            a += qx * u[i] + qy * v[i];
            bq += qx * qx + qy * qy;
            if (with_jac) {
                const double inv2 = 1.0 / (static_cast<double>(z[i]) + s2);
                const double px = x[i] * inv2, py = y[i] * inv2;
                a2 += px * u[i] + py * v[i];
                bq2 += px * px + py * py;
            }
        }
    a = block_sum(a, red); bq = block_sum(bq, red);
    if (with_jac) { a2 = block_sum(a2, red); bq2 = block_sum(bq2, red); }
    const double f = fixed_focal ? focal_given : a / bq;
    const double f2 = fixed_focal ? focal_given : (with_jac ? a2 / bq2 : 0.0);
    double cost = 0, jtr = 0, jtj = 0;
#pragma unroll
    for (int i = 0; i < FS_PER_THREAD; ++i)
        if (valid >> i & 1) {
            const double inv = 1.0 / (static_cast<double>(z[i]) + s);
            const double rx = f * x[i] * inv - u[i], ry = f * y[i] * inv - v[i];
            cost += rx * rx + ry * ry;
            if (with_jac) {
                const double inv2 = 1.0 / (static_cast<double>(z[i]) + s2);
                const double jx = ((f2 * x[i] * inv2 - u[i]) - rx) / h, jy = ((f2 * y[i] * inv2 - v[i]) - ry) / h;
                jtr += jx * rx + jy * ry;
                jtj += jx * jx + jy * jy;
            }
        }
    FsEval e;
    e.cost = block_sum(cost, red); e.focal = f; e.jtr = 0; e.jtj = 0;
    if (with_jac) { e.jtr = block_sum(jtr, red); e.jtj = block_sum(jtj, red); }
    return e;
}

__global__ void __launch_bounds__(FS_THREADS)
focal_shift_kernel(const float* __restrict__ points, const float* __restrict__ mask_prob, const uint8_t* __restrict__ mask_u8,
                   int H, int W, const float* __restrict__ focal_in, float* __restrict__ focal_out, float* __restrict__ shift_out) {
    pdl_prologue();
    __shared__ double red[FS_THREADS / 32];
    __shared__ int count_sh;
    const int b = blockIdx.x;
    const float aspect = static_cast<float>(W) / H;
    const float su = aspect / sqrtf(1.f + aspect * aspect), sv = 1.f / sqrtf(1.f + aspect * aspect);
    const float sh = static_cast<float>(H) / 64.0f, sw = static_cast<float>(W) / 64.0f;   // legacy 'nearest' scales
    float x[FS_PER_THREAD], y[FS_PER_THREAD], z[FS_PER_THREAD], u[FS_PER_THREAD], v[FS_PER_THREAD];
    unsigned valid = 0;
    int cnt = 0;
#pragma unroll
    for (int i = 0; i < FS_PER_THREAD; ++i) {
        const int sidx = threadIdx.x + i * FS_THREADS;
        const int oy = sidx >> 6, ox = sidx & 63;
        const int iy = min(static_cast<int>(floorf(oy * sh)), H - 1), ix = min(static_cast<int>(floorf(ox * sw)), W - 1);
        const size_t pix = (static_cast<size_t>(b) * H + iy) * W + ix;
        x[i] = points[pix * 3]; y[i] = points[pix * 3 + 1]; z[i] = points[pix * 3 + 2];
        u[i] = su * ((2 * ix + 1) / static_cast<float>(W) - 1.0f);
        v[i] = sv * ((2 * iy + 1) / static_cast<float>(H) - 1.0f);
        bool m = true;
        if (mask_u8 != nullptr) m = mask_u8[pix] != 0;
        else if (mask_prob != nullptr) m = mask_prob[pix] > 0.5f;
        if (m) { valid |= 1u << i; ++cnt; }
    }
    if (threadIdx.x == 0) count_sh = 0;
    __syncthreads();
    atomicAdd(&count_sh, cnt);
    __syncthreads();
    const bool fixed = focal_in != nullptr;
    const double fgiven = fixed ? static_cast<double>(focal_in[b]) : 0.0;
    if (count_sh < 2) {      // geometry_torch.py:153-156
        if (threadIdx.x == 0) { focal_out[b] = fixed ? focal_in[b] : 1.0f; shift_out[b] = 0.0f; }
        return;
    }
    // ---- MINPACK lmder restated for one unknown: what scipy.optimize.least_squares(method='lm', x0=0, ftol=1e-3, xtol=gtol=1e-8,
    // factor=100) executes in the reference (geometry_numpy.py:90,109) with SciPy >= 1.16, whose default x_scale is 'jac' ->
    // diag=None -> MINPACK MODE 1: the variable is scaled by d = the running maximum of the Jacobian column norm, and the trust
    // region bounds |d * step| (SciPy < 1.16 used x_scale=1, mode 2: set d = 1 below).  The solver stops on ftol = 1e-3, i.e. long
    // before its fixed point, so the reference's answer IS its iterate sequence: reproducing the trust-region updates, the
    // 2-point Jacobian and the stopping rule -- not just the optimum -- is what keeps depth / intrinsics within 1e-3 of it.
    const double ftol = 1e-3, xtol = 1e-8, gtol = 1e-8, epsmch = 2.220446049250313e-16, dwarf = 2.2250738585072014e-308;
    double s = 0.0;
    FsEval cur = fs_eval(s, true, x, y, z, u, v, valid, fixed, fgiven, red);
    double fnorm = sqrt(cur.cost);
    double par = 0.0, delta = 0.0, xnorm = 0.0, d = 1.0;
    int nfev = 1;
    bool stop = false;
    bool jac_stale = false;
    for (int iter = 1; !stop && nfev < 200; ++iter) {
        if (jac_stale) {                                  // lmdif: Jacobian re-evaluated at the start of every outer iteration
            cur = fs_eval(s, true, x, y, z, u, v, valid, fixed, fgiven, red);
            jac_stale = false;
        }
        const double jtj = cur.jtj, jtr = cur.jtr;
        const double jnorm = sqrt(jtj);
        if (iter == 1) {
            d = (jnorm != 0.0) ? jnorm : 1.0;                           // mode 1: diag = column norm of the first Jacobian
            xnorm = d * fabs(s);
            delta = 100.0 * xnorm;
            if (delta == 0.0) delta = 100.0;
        }
        double gnorm = 0.0;
        if (fnorm != 0.0 && jnorm != 0.0) gnorm = fabs(jtr / jnorm) / fnorm;
        if (gnorm <= gtol) break;                                   // info = 4
        if (!(jnorm > 0.0) || !isfinite(jnorm)) break;
        d = fmax(d, jnorm);                                         // mode 1: diag = max(diag, column norm)
        const double d2 = d * d;
        double ratio = 0.0;
        do {
            // ---- lmpar (n = 1, R = jnorm, Q^T f = jtr / jnorm, scale d): step xs solves (jtj + par d^2) xs = jtr, p = -xs,
            //      trust region on |d xs|
            const double qtb = jtr / jnorm;
            double xs = qtb / jnorm;
            double dxnorm = d * fabs(xs);
            double fp = dxnorm - delta;
            if (fp <= 0.1 * delta) {
                par = 0.0;
            } else {
                double parl = (fp / delta) * jtj / d2;
                const double gn = fabs(jtr) / d;
                double paru = gn / delta;
                if (paru == 0.0) paru = dwarf / fmin(delta, 0.1);
                par = fmax(par, parl);
                par = fmin(par, paru);
                if (par == 0.0) par = gn / dxnorm;
                for (int k = 1;; ++k) {
                    if (par == 0.0) par = fmax(dwarf, 0.001 * paru);
                    xs = jtr / (jtj + par * d2);
                    dxnorm = d * fabs(xs);
                    const double temp = fp;
                    fp = dxnorm - delta;
                    if (fabs(fp) <= 0.1 * delta || (parl == 0.0 && fp <= temp && temp < 0.0) || k == 10) break;
                    const double parc = (fp / delta) * (jtj + par * d2) / d2;
                    if (fp > 0.0) parl = fmax(parl, par);
                    if (fp < 0.0) paru = fmin(paru, par);
                    par = fmax(parl, par + parc);
                }
            }
            const double pstep = -xs;
            const double pnorm = d * fabs(pstep);
            if (iter == 1) delta = fmin(delta, pnorm);
            FsEval nxt = fs_eval(s + pstep, false, x, y, z, u, v, valid, fixed, fgiven, red);
            ++nfev;
            const double fnorm1 = sqrt(nxt.cost);
            double actred = -1.0;
            if (0.1 * fnorm1 < fnorm) actred = 1.0 - (fnorm1 / fnorm) * (fnorm1 / fnorm);
            const double temp1 = jnorm * fabs(pstep) / fnorm, temp2 = sqrt(par) * pnorm / fnorm;
            const double prered = temp1 * temp1 + 2.0 * temp2 * temp2;
            const double dirder = -(temp1 * temp1 + temp2 * temp2);
            ratio = (prered != 0.0) ? actred / prered : 0.0;
            if (ratio <= 0.25) {
                double temp = (actred >= 0.0) ? 0.5 : 0.5 * dirder / (dirder + 0.5 * actred);
                if (0.1 * fnorm1 >= fnorm || temp < 0.1) temp = 0.1;
                delta = temp * fmin(delta, pnorm / 0.1);
                par /= temp;
            } else if (par == 0.0 || ratio >= 0.75) {
                delta = pnorm / 0.5;
                par *= 0.5;
            }
            if (ratio >= 1e-4) {                                    // successful iteration
                s += pstep;
                cur = nxt;
                jac_stale = true;
                xnorm = d * fabs(s);
                fnorm = fnorm1;
            }
            if (fabs(actred) <= ftol && prered <= ftol && 0.5 * ratio <= 1.0) stop = true;      // info = 1 (scipy status 2)
            if (delta <= xtol * xnorm) stop = true;                                              // info = 2
            if (fabs(actred) <= epsmch && prered <= epsmch && 0.5 * ratio <= 1.0) stop = true;  // info = 6
            if (delta <= epsmch * xnorm) stop = true;                                            // info = 7
            if (nfev >= 200 || !isfinite(fnorm1)) stop = true;
        } while (!stop && ratio < 1e-4);
    }
    if (threadIdx.x == 0) {
        const float sf = static_cast<float>(s);                          // geometry_numpy.py:91 casts the shift to float32 ...
        shift_out[b] = sf;
        focal_out[b] = fixed ? focal_in[b] : static_cast<float>(cur.focal);
    }
    // ... and recomputes the focal with the float32 shift (geometry_numpy.py:93-94)
    if (!fixed) {
        const FsEval fin = fs_eval(static_cast<double>(static_cast<float>(s)), false, x, y, z, u, v, valid, false, 0.0, red);
        if (threadIdx.x == 0) focal_out[b] = static_cast<float>(fin.focal);
    }
}
int launch_focal_shift(const float* points, const float* mask_prob, const uint8_t* mask_u8, int B, int H, int W,
                       const float* focal_in, float* focal_out, float* shift_out, cudaStream_t st) {
    CUDA_TRY(launch_pdl(focal_shift_kernel, dim3(B), dim3(FS_THREADS), 0, st, points, mask_prob, mask_u8, H, W, focal_in, focal_out, shift_out));
    CUDA_TRY(cudaGetLastError());
    return 0;
}

// ------------------------------------------------------------------------------------------ K19 post-processing
// v2.py:265-289 (+ utils3d intrinsics_from_focal_center / depth_map_to_point_map): intrinsics, z += shift,
// mask &= z > 0, re-projection, metric scale, masking (points/depth -> +inf, normal -> 0).
__global__ void postprocess_kernel(float* __restrict__ points, const float* __restrict__ normal_in, const float* __restrict__ mask_prob,
                                   const float* __restrict__ metric_scale, const float* __restrict__ focal,
                                   const float* __restrict__ shift, int H, int W, int force_projection, int apply_mask,
                                   float* __restrict__ depth, float* __restrict__ normal_out, uint8_t* __restrict__ mask_out,
                                   float* __restrict__ intrinsics) {
    pdl_prologue();
    const int b = blockIdx.y;
    const float aspect = static_cast<float>(W) / H;
    const float diag = sqrtf(1.f + aspect * aspect);
    const float f = focal[b];
    const float fx = f / 2.f * diag / aspect, fy = f / 2.f * diag;
    const float sft = shift[b];
    const float ms = metric_scale ? metric_scale[b] : 1.0f;
    if (blockIdx.x == 0 && threadIdx.x < 9) {
        const float K[9] = {fx, 0.f, 0.5f, 0.f, fy, 0.5f, 0.f, 0.f, 1.f};
        intrinsics[b * 9 + threadIdx.x] = K[threadIdx.x];
    }
    const size_t npix = static_cast<size_t>(H) * W;
    for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < npix; i += static_cast<size_t>(gridDim.x) * blockDim.x) {
        const size_t pix = static_cast<size_t>(b) * npix + i;
        const int X = static_cast<int>(i % W), Y = static_cast<int>(i / W);
        float px = points[pix * 3], py = points[pix * 3 + 1];
        const float z = points[pix * 3 + 2] + sft;
        bool m = true;
        if (mask_prob != nullptr) m = (mask_prob[pix] > 0.5f) && (z > 0.f);
        if (force_projection) {
            px = ((X + 0.5f) / W - 0.5f) / fx * z;
            py = ((Y + 0.5f) / H - 0.5f) / fy * z;
        }
        float ox = px * ms, oy = py * ms, oz = z * ms;
        const bool kill = apply_mask && mask_prob != nullptr && !m;
        if (kill) { ox = oy = oz = INFINITY; }
        points[pix * 3] = ox; points[pix * 3 + 1] = oy; points[pix * 3 + 2] = oz;
        depth[pix] = oz;
        if (mask_out != nullptr) mask_out[pix] = m ? 1 : 0;
        if (normal_in != nullptr) {
            const float nx = normal_in[pix * 3], ny = normal_in[pix * 3 + 1], nz = normal_in[pix * 3 + 2];
            normal_out[pix * 3] = kill ? 0.f : nx; normal_out[pix * 3 + 1] = kill ? 0.f : ny; normal_out[pix * 3 + 2] = kill ? 0.f : nz;
        }
    }
}
int launch_postprocess(float* points, const float* normal_in, const float* mask_prob, const float* metric_scale,
                       const float* focal, const float* shift, int B, int H, int W, int force_projection, int apply_mask,
                       float* depth, float* normal_out, uint8_t* mask_out, float* intrinsics, cudaStream_t st) {
    const size_t npix = static_cast<size_t>(H) * W;
    dim3 grid(static_cast<unsigned>(std::min<size_t>((npix + 255) / 256, 132 * 8)), B);
    CUDA_TRY(launch_pdl(postprocess_kernel, grid, dim3(256), 0, st, points, normal_in, mask_prob, metric_scale, focal, shift, H, W, force_projection,
                        apply_mask, depth, normal_out, mask_out, intrinsics));
    return 0;
}

}  // namespace mg
