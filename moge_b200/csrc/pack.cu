// Load-time weight repacking: PyTorch state-dict layouts -> the engine's K-major 16-bit GEMM operands, plus a small
// fp32 SIMT GEMM used only to fold consecutive linear maps at load time (never on the inference path).
#include "common.cuh"
#include "host_api.h"
#include <algorithm>

namespace mg {

__device__ __forceinline__ float load_any(const void* p, int dtype, size_t i) {
    if (dtype == 0) return static_cast<const float*>(p)[i];
    if (dtype == 1) return __half2float(static_cast<const __half*>(p)[i]);
    return __bfloat162float(static_cast<const __nv_bfloat16*>(p)[i]);
}
template <bool BF16> __device__ __forceinline__ void store16(void* p, size_t i, float v) {
    static_cast<typename H16<BF16>::T*>(p)[i] = H16<BF16>::from_float(v);
}

template <bool BF16>
__global__ void cast_2d_kernel(const void* src, int sdt, void* dst, int rows, int cols, int sld, int dld) {
    const size_t total = static_cast<size_t>(rows) * dld;
    for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < total; i += static_cast<size_t>(gridDim.x) * blockDim.x) {
        const int c = static_cast<int>(i % dld);
        const size_t r = i / dld;
        store16<BF16>(dst, i, c < cols ? load_any(src, sdt, r * sld + c) : 0.f);     // zero-fills the K padding
    }
}
int launch_cast_2d(const void* src, int src_dtype, void* dst, bool bf16, int rows, int cols, int src_ld, int dst_ld, cudaStream_t st) {
    const size_t total = static_cast<size_t>(rows) * dst_ld;
    const int blocks = static_cast<int>(std::min<size_t>((total + 255) / 256, 132 * 16));
    if (bf16) cast_2d_kernel<true><<<blocks, 256, 0, st>>>(src, src_dtype, dst, rows, cols, src_ld, dst_ld);
    else cast_2d_kernel<false><<<blocks, 256, 0, st>>>(src, src_dtype, dst, rows, cols, src_ld, dst_ld);
    CUDA_TRY(cudaGetLastError());
    return 0;
}

// Conv2d weight (Cout, Cin, kh, kw) -> B[co, k_off + tap*Cin + ci], tap = ky*kw + kx  (taps = kh*kw)
template <bool BF16>
__global__ void pack_conv_kernel(const float* w, void* dst, int Cout, int Cin, int taps, int dld, int koff) {
    const size_t total = static_cast<size_t>(Cout) * taps * Cin;
    for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < total; i += static_cast<size_t>(gridDim.x) * blockDim.x) {
        const int ci = static_cast<int>(i % Cin);
        const int tap = static_cast<int>((i / Cin) % taps);
        const int co = static_cast<int>(i / (static_cast<size_t>(Cin) * taps));
        store16<BF16>(dst, static_cast<size_t>(co) * dld + koff + static_cast<size_t>(tap) * Cin + ci,
                      w[(static_cast<size_t>(co) * Cin + ci) * taps + tap]);
    }
}
int launch_pack_conv(const float* w, void* dst, bool bf16, int Cout, int Cin, int taps, int dst_ld, int k_off, cudaStream_t st) {
    const size_t total = static_cast<size_t>(Cout) * taps * Cin;
    const int blocks = static_cast<int>(std::min<size_t>((total + 255) / 256, 132 * 16));
    if (bf16) pack_conv_kernel<true><<<blocks, 256, 0, st>>>(w, dst, Cout, Cin, taps, dst_ld, k_off);
    else pack_conv_kernel<false><<<blocks, 256, 0, st>>>(w, dst, Cout, Cin, taps, dst_ld, k_off);
    CUDA_TRY(cudaGetLastError());
    return 0;
}

// ConvTranspose2d weight (Cin, Cout, 2, 2) -> B[(q*Cout + co), ci], q = di*2 + dj
template <bool BF16>
__global__ void pack_convT_kernel(const float* w, void* dst, int Cin, int Cout) {
    const size_t total = static_cast<size_t>(4) * Cout * Cin;
    for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < total; i += static_cast<size_t>(gridDim.x) * blockDim.x) {
        const int ci = static_cast<int>(i % Cin);
        const int co = static_cast<int>((i / Cin) % Cout);
        const int q = static_cast<int>(i / (static_cast<size_t>(Cin) * Cout));
        store16<BF16>(dst, i, w[(static_cast<size_t>(ci) * Cout + co) * 4 + q]);
    }
}
int launch_pack_convT(const float* w, void* dst, bool bf16, int Cin, int Cout, cudaStream_t st) {
    const size_t total = static_cast<size_t>(4) * Cout * Cin;
    const int blocks = static_cast<int>(std::min<size_t>((total + 255) / 256, 132 * 16));
    if (bf16) pack_convT_kernel<true><<<blocks, 256, 0, st>>>(w, dst, Cin, Cout);
    else pack_convT_kernel<false><<<blocks, 256, 0, st>>>(w, dst, Cin, Cout);
    CUDA_TRY(cudaGetLastError());
    return 0;
}

// Bilinear x2 upsample (align_corners=False) followed by a 3x3 replicate-padded conv == four phase-specific 3x3
// convs on the LOW-resolution map (exact, incl. the borders, when that map carries a replicated 1-pixel border):
//   out[2i+py, 2j+px] = sum_{a,b} Weff[py,px][a,b] . in[i-1+a, j-1+b],   Weff = sum_{ky,kx} Uy[py][ky][a] Ux[px][kx][b] W[ky,kx]
// src (Cout,Cin,3,3) fp32 -> dst (4*Cout,Cin,3,3) fp32 with row n = (py*2+px)*Cout + co.
__global__ void up2_expand_kernel(const float* w, float* dst, int Cout, int Cin) {
    // U[p][k][a]: weight of low-res tap a (offsets -1,0,+1) in upsampled row 2i+p-1+k
    const float U[2][3][3] = {{{0.75f, 0.25f, 0.f}, {0.25f, 0.75f, 0.f}, {0.f, 0.75f, 0.25f}},
                              {{0.25f, 0.75f, 0.f}, {0.f, 0.75f, 0.25f}, {0.f, 0.25f, 0.75f}}};
    const size_t total = static_cast<size_t>(4) * Cout * Cin * 9;
    for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < total; i += static_cast<size_t>(gridDim.x) * blockDim.x) {
        const int b = static_cast<int>(i % 3), a = static_cast<int>((i / 3) % 3);
        const int ci = static_cast<int>((i / 9) % Cin);
        const int n = static_cast<int>(i / (static_cast<size_t>(9) * Cin));
        const int ph = n / Cout, co = n % Cout, py = ph >> 1, px = ph & 1;
        const float* ws = w + (static_cast<size_t>(co) * Cin + ci) * 9;
        float acc = 0.f;
        for (int ky = 0; ky < 3; ++ky)
            for (int kx = 0; kx < 3; ++kx) acc += U[py][ky][a] * U[px][kx][b] * ws[ky * 3 + kx];
        dst[i] = acc;
    }
}
int launch_up2_expand(const float* w, float* dst, int Cout, int Cin, cudaStream_t st) {
    const size_t total = static_cast<size_t>(4) * Cout * Cin * 9;
    up2_expand_kernel<<<static_cast<int>(std::min<size_t>((total + 255) / 256, 132 * 16)), 256, 0, st>>>(w, dst, Cout, Cin);
    CUDA_TRY(cudaGetLastError());
    return 0;
}

// C[M,N] = A[M,K] * B[K,N] (+C): 16x16 tiled fp32 SIMT, load time only.
__global__ void sgemm_kernel(const float* A, int lda, const float* B, int ldb, float* C, int ldc, int M, int N, int K, int acc) {
    __shared__ float sa[16][17], sb[16][17];
    const int row = blockIdx.y * 16 + threadIdx.y, col = blockIdx.x * 16 + threadIdx.x;
    float s = 0.f;
    for (int k0 = 0; k0 < K; k0 += 16) {
        sa[threadIdx.y][threadIdx.x] = (row < M && k0 + threadIdx.x < K) ? A[static_cast<size_t>(row) * lda + k0 + threadIdx.x] : 0.f;
        sb[threadIdx.y][threadIdx.x] = (k0 + threadIdx.y < K && col < N) ? B[static_cast<size_t>(k0 + threadIdx.y) * ldb + col] : 0.f;
        __syncthreads();
#pragma unroll
        for (int k = 0; k < 16; ++k) s += sa[threadIdx.y][k] * sb[k][threadIdx.x];
        __syncthreads();
    }
    if (row < M && col < N) {
        float* c = C + static_cast<size_t>(row) * ldc + col;
        *c = acc ? *c + s : s;
    }
}
int launch_sgemm(const float* A, int lda, const float* B, int ldb, float* C, int ldc, int M, int N, int K, int accumulate, cudaStream_t st) {
    dim3 grid((N + 15) / 16, (M + 15) / 16), block(16, 16);
    sgemm_kernel<<<grid, block, 0, st>>>(A, lda, B, ldb, C, ldc, M, N, K, accumulate);
    CUDA_TRY(cudaGetLastError());
    return 0;
}

}  // namespace mg
