// sm_90a warpgroup MMA wrappers: D[64 x N] (fp32, registers) (+)= A[64 x 16] * B[16 x N] with fp16 / bf16 operands.
// The SS form reads A and B through shared-memory descriptors; the RS form takes A from registers (four 32-bit registers of
// packed 16-bit pairs per thread, the layout of the fp32 accumulator fragment of an m64nNk16 MMA over the same 16 columns).
// Accumulator fragment of thread t of the warpgroup (warp w = t / 32, lane l): d[i] is row 16 w + l / 4 + 8 ((i / 2) % 2),
// column 8 (i / 4) + 2 (l % 4) + i % 2.  Inline PTX needs every accumulator register named: the lists below spell them out.
#pragma once
#include <stdint.h>

#define MG_R8(a, b, c, d, e, f, g, h) "%" #a ", %" #b ", %" #c ", %" #d ", %" #e ", %" #f ", %" #g ", %" #h
#define MG_REGS8 MG_R8(0, 1, 2, 3, 4, 5, 6, 7)
#define MG_REGS16 MG_REGS8 ", " MG_R8(8, 9, 10, 11, 12, 13, 14, 15)
#define MG_REGS32 MG_REGS16 ", " MG_R8(16, 17, 18, 19, 20, 21, 22, 23) ", " MG_R8(24, 25, 26, 27, 28, 29, 30, 31)
#define MG_REGS64 MG_REGS32 ", " MG_R8(32, 33, 34, 35, 36, 37, 38, 39) ", " MG_R8(40, 41, 42, 43, 44, 45, 46, 47) ", " \
    MG_R8(48, 49, 50, 51, 52, 53, 54, 55) ", " MG_R8(56, 57, 58, 59, 60, 61, 62, 63)
#define MG_REGS128 MG_REGS64 ", " MG_R8(64, 65, 66, 67, 68, 69, 70, 71) ", " MG_R8(72, 73, 74, 75, 76, 77, 78, 79) ", " \
    MG_R8(80, 81, 82, 83, 84, 85, 86, 87) ", " MG_R8(88, 89, 90, 91, 92, 93, 94, 95) ", " \
    MG_R8(96, 97, 98, 99, 100, 101, 102, 103) ", " MG_R8(104, 105, 106, 107, 108, 109, 110, 111) ", " \
    MG_R8(112, 113, 114, 115, 116, 117, 118, 119) ", " MG_R8(120, 121, 122, 123, 124, 125, 126, 127)
#define MG_D8(o) "+f"(d[o]), "+f"(d[o + 1]), "+f"(d[o + 2]), "+f"(d[o + 3]), "+f"(d[o + 4]), "+f"(d[o + 5]), "+f"(d[o + 6]), "+f"(d[o + 7])
#define MG_OUT8 MG_D8(0)
#define MG_OUT16 MG_OUT8, MG_D8(8)
#define MG_OUT32 MG_OUT16, MG_D8(16), MG_D8(24)
#define MG_OUT64 MG_OUT32, MG_D8(32), MG_D8(40), MG_D8(48), MG_D8(56)
#define MG_OUT128 MG_OUT64, MG_D8(64), MG_D8(72), MG_D8(80), MG_D8(88), MG_D8(96), MG_D8(104), MG_D8(112), MG_D8(120)

// SS: the operands after the accumulators are the A descriptor (%DA), the B descriptor (%DB), scale-d (%S) and trans-b (%TB)
#define MG_WGMMA_SS(N, T, REGS, DA, DB, S, TB, ...)                                                          \
    asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %" #S ", 0;\n"                                              \
                 "wgmma.mma_async.sync.aligned.m64n" #N "k16.f32." T "." T " {" REGS "}, %" #DA ", %" #DB ", "  \
                 "p, 1, 1, 0, %" #TB ";\n}\n"                                                                 \
                 : __VA_ARGS__                                                                                \
                 : "l"(da), "l"(db), "r"(scale_d), "n"(TRANS_B))

namespace mg {

template <int N, bool BF16> struct Wgmma;

#define MG_WGMMA_STRUCT(N, REGS, DA, DB, S, TB, ...)                                                         \
    template <bool BF16> struct Wgmma<N, BF16> {                                                             \
        template <int TRANS_B = 0>     /* 1: B is MN-major (N contiguous) */                                  \
        static __device__ __forceinline__ void ss(float* d, uint64_t da, uint64_t db, uint32_t scale_d) {    \
            if constexpr (BF16) MG_WGMMA_SS(N, "bf16", REGS, DA, DB, S, TB, __VA_ARGS__);                    \
            else MG_WGMMA_SS(N, "f16", REGS, DA, DB, S, TB, __VA_ARGS__);                                    \
        }                                                                                                     \
    };
MG_WGMMA_STRUCT(16, MG_REGS8, 8, 9, 10, 11, MG_OUT8)
MG_WGMMA_STRUCT(32, MG_REGS16, 16, 17, 18, 19, MG_OUT16)
MG_WGMMA_STRUCT(64, MG_REGS32, 32, 33, 34, 35, MG_OUT32)
MG_WGMMA_STRUCT(128, MG_REGS64, 64, 65, 66, 67, MG_OUT64)
MG_WGMMA_STRUCT(256, MG_REGS128, 128, 129, 130, 131, MG_OUT128)
#undef MG_WGMMA_STRUCT

// RS form, N = 64, B MN-major (the P V product of the attention kernel: A = P from registers, B = V [keys][64]):
// %32..%35 = A registers, %36 = B descriptor, %37 = scale-d
template <bool BF16> __device__ __forceinline__ void wgmma_rs_n64_tb(float* d, const uint32_t* a, uint64_t db, uint32_t scale_d) {
#define MG_WGMMA_RS(T)                                                                                        \
    asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %37, 0;\n"                                                 \
                 "wgmma.mma_async.sync.aligned.m64n64k16.f32." T "." T " {" MG_REGS32 "}, {%32, %33, %34, %35}, %36, " \
                 "p, 1, 1, 1;\n}\n"                                                                           \
                 : MG_OUT32                                                                                   \
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db), "r"(scale_d))
    if constexpr (BF16) MG_WGMMA_RS("bf16");
    else MG_WGMMA_RS("f16");
#undef MG_WGMMA_RS
}

}  // namespace mg

#undef MG_WGMMA_SS
#undef MG_OUT128
#undef MG_OUT64
#undef MG_OUT32
#undef MG_OUT16
#undef MG_OUT8
#undef MG_D8
#undef MG_REGS128
#undef MG_REGS64
#undef MG_REGS32
#undef MG_REGS16
#undef MG_REGS8
#undef MG_R8
