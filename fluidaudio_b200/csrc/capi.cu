// The runtime of libfluidaudio_b200.so's C ABI (declared in include/fluidaudio_b200.h): error text, the device check,
// the launch counter, devices, memory, copies and the global timer.  Each family's entry points are in its own
// <family>_abi.cu.  No exception and no CUDA type crosses this boundary; there is no CPU fallback behind it.  Every
// entry point that returns a status returns through guard() (c_abi.h).
#include "c_abi.h"

#include <atomic>
#include <chrono>
#include <cstdarg>
#include <cstdio>

namespace fa {

// The last failure's text on this thread, and how many times it has been set (error_serial).
struct ErrorText {
    char text[512];
    unsigned serial;
};
static thread_local ErrorText g_error{};
void set_error(const char *fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_error.text, sizeof(g_error.text), fmt, ap);
    va_end(ap);
    ++g_error.serial;
}
const char *last_error() { return g_error.text; }
unsigned error_serial() { return g_error.serial; }

const char *status_name(int status) {
    switch (status) {
    case FA_OK: return "FA_STATUS_OK";
    case FA_INVALID_ARGUMENT: return "FA_STATUS_INVALID_ARGUMENT";
    case FA_INDEX_OVERFLOW: return "FA_STATUS_INDEX_OVERFLOW";
    case FA_OUTPUT_TOO_SMALL: return "FA_STATUS_OUTPUT_TOO_SMALL";
    case FA_ALLOCATION_FAILURE: return "FA_STATUS_ALLOCATION_FAILURE";
    case FA_RUNTIME_ERROR: return "FA_STATUS_RUNTIME_ERROR";
    case FA_NO_DEVICE: return "FA_STATUS_NO_DEVICE";
    case FA_CUDA_ERROR: return "FA_STATUS_CUDA_ERROR";
    case FA_UNSUPPORTED: return "FA_STATUS_UNSUPPORTED";
    default: return "FA_STATUS_UNKNOWN_ERROR";
    }
}

std::atomic<long long> g_launches{0};

static int usable_device_count() {
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess) {
        cudaGetLastError();
        return 0;
    }
    int ok = 0;
    for (int i = 0; i < n; ++i) {
        cudaDeviceProp p;
        if (sm90_device_props(i, p) == FA_OK) ++ok;
    }
    return ok;
}

int require_device() {
    static std::atomic<int> cached{-1};
    int c = cached.load();
    if (c < 0) {
        c = usable_device_count();
        cached.store(c);
    }
    if (c <= 0) {
        set_error("no sm_90a (H100) device visible; fluidaudio_b200 has no CPU fallback");
        return FA_NO_DEVICE;
    }
    return FA_OK;
}

// timer state for fa_timer_*, per thread
static thread_local Event t_ev[2];

} // namespace fa

using namespace fa;

// ------------------------------------------------------------------------------------------------ runtime
FA_API const char *fa_version(void) { return "fluidaudio_b200 0.1.0 (sm_90a)"; }
FA_API const char *fa_last_error(void) { return fa::last_error(); }
FA_API int32_t fa_device_count(void) { return usable_device_count(); }

FA_API fa_status fa_set_device(int32_t ordinal) {
    return guard(__func__, [&]() -> int {
        if (require_device() != FA_OK) return FA_STATUS_NO_DEVICE;
        FA_CUDA_TRY(cudaSetDevice(ordinal));
        return FA_STATUS_OK;
    });
}

FA_API fa_status fa_device_synchronize(void) {
    return guard(__func__, [&]() -> int {
        if (require_device() != FA_OK) return FA_STATUS_NO_DEVICE;
        FA_CUDA_TRY(cudaDeviceSynchronize());
        return FA_STATUS_OK;
    });
}

FA_API int64_t fa_kernel_launch_count(void) { return g_launches.load(); }

FA_API fa_status fa_host_alloc(size_t bytes, void **out) {
    return guard(__func__, [&]() -> int {
        if (!out) return FA_STATUS_INVALID_ARGUMENT;
        if (require_device() != FA_OK) return FA_STATUS_NO_DEVICE;
        FA_CUDA_TRY(cudaMallocHost(out, bytes ? bytes : 1));
        return FA_STATUS_OK;
    });
}
FA_API fa_status fa_host_free(void *p) {
    return guard(__func__, [&]() -> int {
        if (p) FA_CUDA_TRY(cudaFreeHost(p));
        return FA_STATUS_OK;
    });
}
FA_API fa_status fa_device_alloc(size_t bytes, void **out) {
    return guard(__func__, [&]() -> int {
        if (!out) return FA_STATUS_INVALID_ARGUMENT;
        if (require_device() != FA_OK) return FA_STATUS_NO_DEVICE;
        FA_CUDA_TRY(cudaMalloc(out, bytes ? bytes : 1));
        return FA_STATUS_OK;
    });
}
FA_API fa_status fa_device_free(void *p) {
    return guard(__func__, [&]() -> int {
        if (p) FA_CUDA_TRY(cudaFree(p));
        return FA_STATUS_OK;
    });
}
FA_API fa_status fa_memcpy_h2d(void *dst, const void *src, size_t bytes) {
    return guard(__func__, [&]() -> int {
        if (require_device() != FA_OK) return FA_STATUS_NO_DEVICE;
        FA_CUDA_TRY(cudaMemcpy(dst, src, bytes, cudaMemcpyHostToDevice));
        return FA_STATUS_OK;
    });
}
FA_API fa_status fa_memcpy_d2h(void *dst, const void *src, size_t bytes) {
    return guard(__func__, [&]() -> int {
        if (require_device() != FA_OK) return FA_STATUS_NO_DEVICE;
        FA_CUDA_TRY(cudaMemcpy(dst, src, bytes, cudaMemcpyDeviceToHost));
        return FA_STATUS_OK;
    });
}

// Bare copy-engine probe: `reps` rounds of an H2D copy of h2d_bytes and a D2H copy of d2h_bytes issued together on two
// streams (device scratch allocated here), wall-clock per round.  bench.py uses it to name the floor under every
// host-buffer (end-to-end) number: what the PCIe / host-memory path delivers with no kernel in the way.
FA_API fa_status fa_memcpy_probe(const void *host_src, size_t h2d_bytes, void *host_dst, size_t d2h_bytes, int32_t reps,
                                 float *ms_per_round) {
    return guard(__func__, [&]() -> int {
        if (!ms_per_round || reps < 1 || (!host_src && h2d_bytes) || (!host_dst && d2h_bytes))
            return FA_STATUS_INVALID_ARGUMENT;
        if (require_device() != FA_OK) return FA_STATUS_NO_DEVICE;
        Stream s[2];
        DeviceBuffer<> a, b;
        int st = a.grow(h2d_bytes + 16);
        if (st == FA_OK) st = b.grow(d2h_bytes + 16);
        if (st != FA_OK) return st;
        FA_CUDA_TRY(cudaMemset(b.data(), 0, d2h_bytes + 16));
        for (auto &x : s)
            if (st == FA_OK) st = x.create();
        if (st != FA_OK) return st;
        FA_CUDA_TRY(cudaDeviceSynchronize());
        const auto t0 = std::chrono::steady_clock::now();
        for (int i = 0; i < reps; ++i) {
            if (h2d_bytes) FA_CUDA_TRY(cudaMemcpyAsync(a.data(), host_src, h2d_bytes, cudaMemcpyHostToDevice, s[0]));
            if (d2h_bytes) FA_CUDA_TRY(cudaMemcpyAsync(host_dst, b.data(), d2h_bytes, cudaMemcpyDeviceToHost, s[1]));
            FA_CUDA_TRY(cudaStreamSynchronize(s[0]));
            FA_CUDA_TRY(cudaStreamSynchronize(s[1]));
        }
        const auto t1 = std::chrono::steady_clock::now();
        *ms_per_round = (float)(std::chrono::duration<double, std::milli>(t1 - t0).count() / reps);
        return FA_STATUS_OK;
    });
}

// Events on the legacy default stream order against every blocking stream AND, because the library's own streams
// are non-blocking, the timed entry points synchronise their streams before returning (device-side async calls
// are timed by the caller bracketing fa_device_synchronize()).
FA_API fa_status fa_timer_start(void) {
    return guard(__func__, [&]() -> int {
        if (require_device() != FA_OK) return FA_STATUS_NO_DEVICE;
        if (!t_ev[0]) {
            const int st = create_timer(t_ev);
            if (st != FA_OK) return st;
        }
        FA_CUDA_TRY(cudaDeviceSynchronize());
        FA_CUDA_TRY(cudaEventRecord(t_ev[0], 0));
        return FA_STATUS_OK;
    });
}
FA_API fa_status fa_timer_stop_ms(float *elapsed_ms) {
    return guard(__func__, [&]() -> int {
        if (!elapsed_ms || !t_ev[0]) return FA_STATUS_INVALID_ARGUMENT;
        FA_CUDA_TRY(cudaDeviceSynchronize());
        FA_CUDA_TRY(cudaEventRecord(t_ev[1], 0));
        FA_CUDA_TRY(cudaEventSynchronize(t_ev[1]));
        FA_CUDA_TRY(cudaEventElapsedTime(elapsed_ms, t_ev[0], t_ev[1]));
        return FA_STATUS_OK;
    });
}
