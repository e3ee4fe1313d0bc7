// TMA tensor-map construction + thread-local error string.  cuTensorMapEncodeTiled is fetched through
// cudaGetDriverEntryPoint so the library has no link-time dependency on libcuda.
#include "host_api.h"
#include <stdarg.h>
#include <stdio.h>
#include <mutex>

namespace mg {

static thread_local char g_err[1024] = "";
int set_error(const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
    return -1;
}
const char* last_error() { return g_err; }

bool& pdl_scope() {
    static thread_local bool on = false;
    return on;
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static EncodeTiledFn get_encode() {
    static EncodeTiledFn fn = nullptr;
    static std::once_flag once;
    std::call_once(once, [] {
        void* p = nullptr;
        cudaDriverEntryPointQueryResult qres;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) == cudaSuccess &&
            qres == cudaDriverEntryPointSuccess)
            fn = reinterpret_cast<EncodeTiledFn>(p);
    });
    return fn;
}

static int encode(CUtensorMap* m, const void* base, int rank, const cuuint64_t* dims, const cuuint64_t* strides_bytes,
                  const cuuint32_t* box, CUtensorMapDataType dtype = CU_TENSOR_MAP_DATA_TYPE_UINT16) {
    EncodeTiledFn fn = get_encode();
    if (!fn) return set_error("cuTensorMapEncodeTiled entry point unavailable (no CUDA driver?)");
    cuuint32_t estr[5] = {1, 1, 1, 1, 1};
    if (reinterpret_cast<uintptr_t>(base) & 15) return set_error("tensor map base %p not 16-byte aligned", base);
    for (int i = 0; i < rank - 1; ++i)
        if (strides_bytes[i] & 15) return set_error("tensor map stride[%d]=%llu not a multiple of 16 bytes", i, (unsigned long long)strides_bytes[i]);
    CUresult r = fn(m, dtype, rank, const_cast<void*>(base), dims, strides_bytes, box, estr,
                    CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                    CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS)
        return set_error("cuTensorMapEncodeTiled failed (%d): rank=%d dims=[%llu,%llu,%llu,%llu] box=[%u,%u,%u,%u]", (int)r, rank,
                         (unsigned long long)dims[0], (unsigned long long)(rank > 1 ? dims[1] : 0),
                         (unsigned long long)(rank > 2 ? dims[2] : 0), (unsigned long long)(rank > 3 ? dims[3] : 0), box[0],
                         rank > 1 ? box[1] : 0, rank > 2 ? box[2] : 0, rank > 3 ? box[3] : 0);
    return 0;
}

int make_map_2d(CUtensorMap* m, const void* base, uint64_t cols, uint64_t rows, uint64_t row_pitch_elems, uint32_t box_rows) {
    cuuint64_t dims[2] = {cols, rows};
    cuuint64_t strides[1] = {row_pitch_elems * 2};
    cuuint32_t box[2] = {64, box_rows};
    return encode(m, base, 2, dims, strides, box);
}
int make_map_nhwc(CUtensorMap* m, const void* base, uint64_t C, uint64_t Wp, uint64_t Hp, uint64_t B, uint32_t box_rows) {
    cuuint64_t dims[4] = {C, Wp, Hp, B};
    cuuint64_t strides[3] = {C * 2, C * Wp * 2, C * Wp * Hp * 2};
    cuuint32_t box[4] = {64, 16, box_rows, 1};
    if (C % 64) return set_error("NHWC tensor map needs C %% 64 == 0 (C=%llu)", (unsigned long long)C);
    return encode(m, base, 4, dims, strides, box);
}

}  // namespace mg
