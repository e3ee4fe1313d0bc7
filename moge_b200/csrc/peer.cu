// Output gather over NVLink peer memory (BASELINE.json configs[3]: "all outputs resident on rank 0") without a single SM:
// every rank exposes a staging buffer through CUDA IPC, rank 0 maps them and PULLS with copy-engine DMAs
// (cudaMemcpyAsync, peer to peer), ordered by device-side flags in peer memory instead of host barriers.
// A NCCL send/recv gather runs copy KERNELS on both ends; next to persistent one-CTA-per-SM kernels that use the whole register
// file an SM that hosts a NCCL block cannot host ours, and the step stretches by the duration of the transfer (at N = 8 rank 0
// receives 1.74 GB per step of the ViT-L 518 px batch of 32).
// NCCL stays what it is used for elsewhere (weight broadcast, barriers); this file has no dependency on it.
#include "moge_b200.h"
#include "host_api.h"
#include <string.h>

namespace mg {

__global__ void flag_set_kernel(int* flag, int value) {
    __threadfence_system();                                        // everything earlier on this stream is visible system-wide first
    asm volatile("st.release.sys.global.s32 [%0], %1;" ::"l"(flag), "r"(value) : "memory");
}

// One thread polls a flag that another GPU writes over NVLink.  ~20 s of polling without progress traps (a dead peer must not
// hang the stream forever).  32 threads x < 32 registers: fits next to a resident CTA that owns almost the whole register file.
__global__ void __launch_bounds__(32, 1) flag_wait_kernel(const int* flag, int value) {
    if (threadIdx.x != 0) return;
    const long long t0 = clock64();
    for (;;) {
        int v;
        asm volatile("ld.acquire.sys.global.s32 %0, [%1];" : "=r"(v) : "l"(flag) : "memory");
        if (v >= value) break;
        __nanosleep(200);
        if (clock64() - t0 > 40000000000LL) __trap();
    }
}

}  // namespace mg

using namespace mg;

extern "C" {

int moge_peer_alloc(size_t bytes, void** dev_ptr, unsigned char* handle64) {
    if (!dev_ptr || !handle64 || bytes == 0) return set_error("peer_alloc: bad argument");
    static_assert(sizeof(cudaIpcMemHandle_t) == 64, "cudaIpcMemHandle_t is expected to be 64 bytes");
    void* p = nullptr;
    CUDA_TRY(cudaMalloc(&p, bytes));
    CUDA_TRY(cudaMemset(p, 0, bytes));
    cudaIpcMemHandle_t h;
    cudaError_t e = cudaIpcGetMemHandle(&h, p);
    if (e != cudaSuccess) { cudaFree(p); return set_error("cudaIpcGetMemHandle failed: %s", cudaGetErrorString(e)); }
    memcpy(handle64, &h, 64);
    *dev_ptr = p;
    return 0;
}

int moge_peer_free(void* dev_ptr) {
    if (dev_ptr) CUDA_TRY(cudaFree(dev_ptr));
    return 0;
}

int moge_peer_open(const unsigned char* handle64, void** dev_ptr) {
    if (!handle64 || !dev_ptr) return set_error("peer_open: null argument");
    cudaIpcMemHandle_t h;
    memcpy(&h, handle64, 64);
    CUDA_TRY(cudaIpcOpenMemHandle(dev_ptr, h, cudaIpcMemLazyEnablePeerAccess));
    return 0;
}

int moge_peer_close(void* dev_ptr) {
    if (dev_ptr) CUDA_TRY(cudaIpcCloseMemHandle(dev_ptr));
    return 0;
}

int moge_peer_copy(void* dst, const void* src, size_t bytes, void* stream) {
    if (bytes == 0) return 0;
    if (!dst || !src) return set_error("peer_copy: null argument");
    CUDA_TRY(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDefault, static_cast<cudaStream_t>(stream)));
    return 0;
}

int moge_peer_flag_set(int* flag, int value, void* stream) {
    if (!flag) return set_error("peer_flag_set: null argument");
    flag_set_kernel<<<1, 1, 0, static_cast<cudaStream_t>(stream)>>>(flag, value);
    CUDA_TRY(cudaGetLastError());
    return 0;
}

int moge_peer_flag_wait(const int* flag, int value, void* stream) {
    if (!flag) return set_error("peer_flag_wait: null argument");
    flag_wait_kernel<<<1, 32, 0, static_cast<cudaStream_t>(stream)>>>(flag, value);
    CUDA_TRY(cudaGetLastError());
    return 0;
}

}  // extern "C"
