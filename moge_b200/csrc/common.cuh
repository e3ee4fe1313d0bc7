// moge_b200 device-side primitives for sm_90a: mbarrier, TMA (cp.async.bulk.tensor), wgmma.
// Hand-written inline PTX; no CUTLASS/CuTe.  The bit layout of the wgmma shared-memory descriptor follows the PTX ISA
// "Matrix Descriptor Format" of the asynchronous warpgroup MMA section.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <cuda_fp16.h>
#include <cuda_bf16.h>
#include <stdint.h>
#include <stdio.h>
#include "wgmma.cuh"

namespace mg {

// ------------------------------------------------------------------------------------------------ misc
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
    return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ bool elect_one() {
    uint32_t pred;
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "elect.sync _|p, 0xffffffff;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(pred));
    return pred != 0;
}

// Programmatic dependent launch: let the next kernel in the stream start launching, then wait until the previous grid has
// completed and its writes are visible (no-ops when the kernel was not launched with programmatic stream serialization).
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_prologue() {
    pdl_launch_dependents();
    pdl_wait();
}

// -------------------------------------------------------------------------------------------- mbarrier
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_mbar_init() {
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
    uint32_t ok;
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(ok)
        : "r"(smem_u32(bar)), "r"(parity)
        : "memory");
    return ok != 0;
}
// Bounded wait: a broken pipeline traps (-> cudaErrorLaunchFailure on the host) instead of hanging the GPU.
// (every failed try_wait suspends the thread for a system-dependent time, up to microseconds: 2^21 spins are seconds, far beyond
// any legitimate wait inside a millisecond kernel)
#ifndef MG_WATCHDOG_SPINS
#define MG_WATCHDOG_SPINS (1u << 21)
#endif
constexpr int kMaxDynSmem = 232448;       // 227 KB: the opt-in dynamic shared memory limit of one CTA on sm_90
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    uint32_t spins = 0;
    while (!mbar_try_wait(bar, parity)) {
        if (++spins > MG_WATCHDOG_SPINS) __trap();      // surfaces as a launch failure on the host (no call, no printf: keeps
    }                                                   // the hot loops small and the register allocation unconstrained)
}

// ------------------------------------------------------------------------------------------------- TMA
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* m) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
__device__ __forceinline__ void tma_load_2d(void* dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
        ::"r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
        : "memory");
}
__device__ __forceinline__ void tma_load_4d(void* dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1, int c2,
                                            int c3) {
    asm volatile(
        "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
        ::"r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2),
        "r"(c3)
        : "memory");
}

// ------------------------------------------------------------------------------------------------ wgmma
// Shared-memory matrix descriptor (sm_90 wgmma), 128-byte swizzle: dense [rows][64 x 16-bit] tiles as written by a SWIZZLE_128B
// TMA box with a 128-byte inner extent, 8-row groups `sbo_bytes` apart.  Tile base must be 1024-byte aligned.
//   [0,14) addr>>4   [16,30) LBO>>4   [32,46) SBO>>4   [62,64) layout=1 (SWIZZLE_128B)
// K-major operands advance 16 elements (32 bytes) along K by adding 2 to the descriptor.
__device__ __forceinline__ uint64_t make_sdesc_sw128(uint32_t smem_addr, uint32_t lbo_bytes = 16, uint32_t sbo_bytes = 1024) {
    uint64_t d = 0;
    d |= static_cast<uint64_t>((smem_addr & 0x3FFFF) >> 4);
    d |= static_cast<uint64_t>((lbo_bytes >> 4) & 0x3FFF) << 16;
    d |= static_cast<uint64_t>((sbo_bytes >> 4) & 0x3FFF) << 32;
    d |= static_cast<uint64_t>(1) << 62;
    return d;
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N> __device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// keeps the compiler from moving accesses of the accumulator registers across a wgmma wait
template <int N> __device__ __forceinline__ void reg_fence(float (&r)[N]) {
#pragma unroll
    for (int i = 0; i < N; ++i) asm volatile("" : "+f"(r[i])::"memory");
}
// named barrier over `count` threads (the consumer warpgroups of a CTA; id 0 is __syncthreads)
__device__ __forceinline__ void named_sync(uint32_t id, uint32_t count) {
    asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(count) : "memory");
}
template <uint32_t R> __device__ __forceinline__ void regs_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(R)); }
template <uint32_t R> __device__ __forceinline__ void regs_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(R)); }

// Two lanes of fp32 arithmetic (sm_90 has no packed fp32 instructions: one FFMA / FADD / FMUL per lane).
__device__ __forceinline__ float2 ffma2(float2 a, float2 b, float2 c) { return make_float2(fmaf(a.x, b.x, c.x), fmaf(a.y, b.y, c.y)); }
__device__ __forceinline__ float2 fadd2(float2 a, float2 b) { return make_float2(a.x + b.x, a.y + b.y); }
__device__ __forceinline__ float2 fmul2(float2 a, float2 b) { return make_float2(a.x * b.x, a.y * b.y); }

__device__ __forceinline__ float ex2_approx(float x) {      // MUFU.EX2, flush-to-zero
    float r;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
    return r;
}

// ------------------------------------------------------------------------------------- 16-bit helpers
template <bool BF16> struct H16;
template <> struct H16<false> {
    using T = __half;
    using T2 = __half2;
    static __device__ __forceinline__ uint32_t pack(float a, float b) {
        __half2 h = __floats2half2_rn(a, b);
        return *reinterpret_cast<uint32_t*>(&h);
    }
    static __device__ __forceinline__ float2 unpack(uint32_t u) {
        return __half22float2(*reinterpret_cast<__half2*>(&u));
    }
    static __device__ __forceinline__ T from_float(float a) { return __float2half_rn(a); }
    static __device__ __forceinline__ float to_float(T a) { return __half2float(a); }
};
template <> struct H16<true> {
    using T = __nv_bfloat16;
    using T2 = __nv_bfloat162;
    static __device__ __forceinline__ uint32_t pack(float a, float b) {
        __nv_bfloat162 h = __floats2bfloat162_rn(a, b);
        return *reinterpret_cast<uint32_t*>(&h);
    }
    static __device__ __forceinline__ float2 unpack(uint32_t u) {
        return __bfloat1622float2(*reinterpret_cast<__nv_bfloat162*>(&u));
    }
    static __device__ __forceinline__ T from_float(float a) { return __float2bfloat16_rn(a); }
    static __device__ __forceinline__ float to_float(T a) { return __bfloat162float(a); }
};

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}

}  // namespace mg
