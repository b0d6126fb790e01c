// Shared definitions for the fluidaudio_b200 CUDA library (sm_90a only).
#pragma once

#include <cstddef>
#include <cstdint>

#if defined(__CUDACC__)
#include <atomic>
#include <utility>
#include <cuda_runtime.h>
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

// Slices one allocation into 256-byte aligned arrays.  Carver{nullptr} is a dry run: `off` then holds the bytes the
// arrays need (carve_arena below runs a layout both ways).
struct Carver {
    char *base = nullptr;
    size_t off = 0;
    template <typename T> T *take(size_t count) {
        off = (off + 255) & ~size_t(255);
        T *p = reinterpret_cast<T *>(base + off);
        off += count * sizeof(T);
        return p;
    }
};

#if defined(__CUDACC__)
// Status of a failed CUDA call: FA_ALLOCATION_FAILURE when memory ran out, FA_CUDA_ERROR otherwise.  It converts to
// the int codes used inside the library and to fa_status at the C ABI (the same numbers).
struct CudaStatus {
    int code;
    template <typename T> operator T() const { return static_cast<T>(code); }
};
inline CudaStatus cuda_failure(cudaError_t e, const char *expr, const char *file, int line) {
    set_error("%s failed: %s (%s:%d)", expr, cudaGetErrorString(e), file, line);
    return CudaStatus{e == cudaErrorMemoryAllocation ? FA_ALLOCATION_FAILURE : FA_CUDA_ERROR};
}
#define FA_CUDA_TRY(expr)                                                                 \
    do {                                                                                  \
        const cudaError_t e__ = (expr);                                                   \
        if (e__ != cudaSuccess) return fa::cuda_failure(e__, #expr, __FILE__, __LINE__); \
    } while (0)

// Grow-only device (or pinned host) buffer: keeps `p` when it already holds `bytes`, otherwise replaces it.  It never
// shrinks, and a failed allocation leaves `p` null and `cap` zero.
template <typename T> int grow_buffer(T *&p, size_t &cap, size_t bytes, bool pinned = false) {
    if (bytes <= cap) return FA_OK;
    if (p) pinned ? cudaFreeHost(p) : cudaFree(p);
    p = nullptr;
    cap = 0;
    void *q = nullptr;
    FA_CUDA_TRY(pinned ? cudaMallocHost(&q, bytes) : cudaMalloc(&q, bytes));
    p = static_cast<T *>(q);
    cap = bytes;
    return FA_OK;
}

// Lays out one scratch arena in a grow-only buffer.  `layout(Carver &)` takes every array of the arena in order and
// only assigns the pointers it gets, so it is safe to run twice: once over a null base to size the arena (plus `slack`
// bytes), then, after the buffer has grown to that size, over the buffer itself.
template <typename T, typename Layout>
int carve_arena(T *&buf, size_t &cap, Layout &&layout, size_t slack = 0, bool pinned = false) {
    Carver size{nullptr};
    layout(size);
    const int st = grow_buffer(buf, cap, size.off + slack, pinned);
    if (st != FA_OK) return st;
    Carver c{static_cast<char *>(static_cast<void *>(buf))};
    layout(c);
    return FA_OK;
}

// Kernel launches of the whole process (fa_kernel_launch_count), defined in capi.cu.  Every launch of the library goes
// through launch() or launch_cooperative(), which count it where it is issued and return its error:
// FA_CUDA_TRY(fa::launch(kernel, grid, block, smem, stream, args...)).
extern std::atomic<long long> g_launches;

template <typename... Params, typename... Args>
cudaError_t launch(void (*kernel)(Params...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream, Args &&...args) {
    kernel<<<grid, block, smem, stream>>>(std::forward<Args>(args)...);
    g_launches.fetch_add(1, std::memory_order_relaxed);
    return cudaGetLastError();
}

// The same for a kernel whose CTAs must all be resident at once (grid-wide synchronisation).  The arguments are
// converted to the kernel's parameter types (the kernel alone fixes them), since the launch passes their addresses.
template <typename T> struct kernel_param { using type = T; };
template <typename... Params>
cudaError_t launch_cooperative(void (*kernel)(Params...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream,
                               typename kernel_param<Params>::type... args) {
    void *argv[] = {&args...};
    const cudaError_t e =
        cudaLaunchCooperativeKernel(reinterpret_cast<const void *>(kernel), grid, block, argv, smem, stream);
    g_launches.fetch_add(1, std::memory_order_relaxed);
    return e != cudaSuccess ? e : cudaGetLastError();
}

// Properties of device `dev`, which must be sm_90: the library carries sm_90a code only.
inline int sm90_device_props(int dev, cudaDeviceProp &prop) {
    FA_CUDA_TRY(cudaGetDeviceProperties(&prop, dev));
    if (prop.major != 9) {
        set_error("fluidaudio_b200 requires an sm_90a device, found sm_%d%d", prop.major, prop.minor);
        return FA_NO_DEVICE;
    }
    return FA_OK;
}

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
