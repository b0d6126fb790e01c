// Shared definitions for the fluidaudio_b200 CUDA library (sm_90a only).
#pragma once

#include <cstddef>
#include <cstdint>

#if defined(__CUDACC__)
#define FA_HD __host__ __device__ __forceinline__
#else
#define FA_HD inline
#endif

// Status codes of the C ABI (include/fluidaudio_b200.h).  Values 0..5 and 255 coincide with
// fastcluster_wrapper_status (reference: Sources/FastClusterWrapper/include/FastClusterWrapper.h:11-19).
enum : int {
    FA_OK = 0,
    FA_INVALID_ARGUMENT = 1,
    FA_INDEX_OVERFLOW = 2,
    FA_OUTPUT_TOO_SMALL = 3,
    FA_ALLOCATION_FAILURE = 4,
    FA_RUNTIME_ERROR = 5,
    FA_NO_DEVICE = 6,
    FA_CUDA_ERROR = 7,
    FA_UNSUPPORTED = 8,
    FA_UNKNOWN_ERROR = 255,
};

namespace fa {

// thread-local last-error text, set by the C ABI on every failure
void set_error(const char *fmt, ...);
const char *last_error();

#if defined(__CUDACC__)
// Float pairs (two frames, two columns) with every lane an independent round-to-nearest IEEE operation.  sm_90 has no
// packed FP32 instructions: each is two FADD / FMUL / FFMA, and the __f*_rn intrinsics keep the compiler from fusing a
// separate multiply and add, so results equal the scalar expressions bit for bit.
__device__ __forceinline__ float2 fadd2_rn(float2 a, float2 b) { return make_float2(__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y)); }
__device__ __forceinline__ float2 fmul2_rn(float2 a, float2 b) { return make_float2(__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y)); }
__device__ __forceinline__ float2 ffma2_rn(float2 a, float2 b, float2 c) {
    return make_float2(__fmaf_rn(a.x, b.x, c.x), __fmaf_rn(a.y, b.y, c.y));
}
#endif

} // namespace fa
