// Shared definitions for the fluidaudio_b200 CUDA library (sm_90a only).
#pragma once

#include <cstddef>
#include <cstdint>

#if defined(__CUDACC__)
#include <atomic>
#include <cstdio>
#include <memory>
#include <type_traits>
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
// An argument check's refusal: sets the text and returns FA_INVALID_ARGUMENT (= FA_STATUS_INVALID_ARGUMENT).
template <typename... A> int refuse(const char *fmt, A... args) {
    set_error(fmt, args...);
    return FA_INVALID_ARGUMENT;
}

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
// Reports a failed CUDA call and consumes the runtime's last-error state of this thread.  launch() returns
// cudaGetLastError(), which also holds the error of any earlier runtime call: without this, a refused cudaMalloc would
// fail the next, unrelated launch on the thread with the same stale error.  A sticky error is not cleared by this.
inline CudaStatus cuda_failure(cudaError_t e, const char *expr, const char *file, int line) {
    set_error("%s failed: %s (%s:%d)", expr, cudaGetErrorString(e), file, line);
    (void)cudaGetLastError();
    return CudaStatus{e == cudaErrorMemoryAllocation ? FA_ALLOCATION_FAILURE : FA_CUDA_ERROR};
}
#define FA_CUDA_TRY(expr)                                                                 \
    do {                                                                                  \
        const cudaError_t e__ = (expr);                                                   \
        if (e__ != cudaSuccess) return fa::cuda_failure(e__, #expr, __FILE__, __LINE__); \
    } while (0)

// Owners of the library's CUDA resources.  Every cudaMalloc / cudaMallocHost, stream and event of the library is made
// here and released by a destructor, which ignores errors: the static context pool is torn down at process exit, when
// the runtime may already be gone.
template <bool Pinned> struct CudaFree {
    void operator()(void *p) const { Pinned ? cudaFreeHost(p) : cudaFree(p); }
};

// Grow-only device (or pinned host) buffer of T: grow() keeps the allocation when it already holds `bytes`, otherwise
// frees it before allocating the larger one (peak memory is the larger size alone).  It never shrinks, and a failed
// allocation leaves it empty.
template <typename T, bool Pinned> class GrowBuffer {
  public:
    GrowBuffer() = default;
    GrowBuffer(GrowBuffer &&o) noexcept : p_(std::move(o.p_)), cap_(std::exchange(o.cap_, 0)) {}
    GrowBuffer &operator=(GrowBuffer &&o) noexcept {
        p_ = std::move(o.p_);
        cap_ = std::exchange(o.cap_, 0);
        return *this;
    }
    int grow(size_t bytes) {
        if (bytes <= cap_) return FA_OK;
        p_.reset();
        cap_ = 0;
        void *q = nullptr;
        const cudaError_t e = Pinned ? cudaMallocHost(&q, bytes) : cudaMalloc(&q, bytes);
        if (e != cudaSuccess) {
            char what[64];
            std::snprintf(what, sizeof(what), "%s(%zu bytes)", Pinned ? "cudaMallocHost" : "cudaMalloc", bytes);
            return cuda_failure(e, what, __FILE__, __LINE__);
        }
        p_.reset(q);
        cap_ = bytes;
        return FA_OK;
    }
    T *data() const { return static_cast<T *>(p_.get()); }
    size_t capacity() const { return cap_; }

  private:
    std::unique_ptr<void, CudaFree<Pinned>> p_;
    size_t cap_ = 0;
};
template <typename T = void> using DeviceBuffer = GrowBuffer<T, false>;
template <typename T = void> using PinnedBuffer = GrowBuffer<T, true>;

// The device twins of one call's caller arrays.  On a device-buffer call a twin is the caller's own pointer: nothing is
// copied and the call stays asynchronous.  On a host-buffer call every twin is carved from one grow-only buffer, the
// inputs are copied in on the call's stream, back() copies the outputs out and sync() waits for them.  A null caller
// array has a null twin.  One per call, on the stack; it owns no memory.
class HostStaging {
  public:
    HostStaging(bool host, cudaStream_t stream) : host_(host), stream_(stream) {}

    // What carve()'s layout takes, in order: twins (an input's `slack` elements are carved but not copied) and scratch
    // (Carver::take), which is carved on either kind of call.
    class Layout : public Carver {
      public:
        template <typename T> const T *in(const T *p, size_t n, size_t slack = 0) {
            return twin(const_cast<T *>(p), n, slack, kIn);
        }
        template <typename T> T *out(T *p, size_t n) { return twin(p, n, 0, kOut); }
        template <typename T> T *inout(T *p, size_t n) { return twin(p, n, 0, kIn | kOut); }

      private:
        friend class HostStaging;
        Layout(char *base, HostStaging &s, bool record) : Carver{base}, s_(s), record_(record) {}
        template <typename T> T *twin(T *p, size_t n, size_t slack, int dir) {
            if (!p || !s_.host_) return p;
            T *t = take<T>(n + slack);
            if (record_ && s_.count_++ < kMaxTwins) s_.twins_[s_.count_ - 1] = Twin{p, t, n * sizeof(T), dir};
            return t;
        }
        HostStaging &s_;
        bool record_;
    };

    // `layout(Layout &)` takes every array in order and only assigns the pointers it gets, so it is safe to run twice:
    // once over a null base to size the arrays (plus `slack` bytes), then, after `buf` has grown to that size, over the
    // buffer itself.  Then the inputs' copies are queued.  A device-buffer call without scratch grows nothing.
    template <typename T, bool Pinned, typename L> int carve(GrowBuffer<T, Pinned> &buf, L &&layout, size_t slack = 0) {
        Layout size(nullptr, *this, false);
        layout(size);
        const int st = buf.grow(size.off + slack);
        if (st != FA_OK) return st;
        Layout c(static_cast<char *>(static_cast<void *>(buf.data())), *this, true);
        count_ = 0;
        layout(c);
        if (count_ > kMaxTwins) {
            set_error("internal: a call stages %d arrays, at most %d", count_, kMaxTwins);
            return FA_RUNTIME_ERROR;
        }
        for (int i = 0; i < count_; ++i)
            if ((twins_[i].dir & kIn) && twins_[i].bytes)
                FA_CUDA_TRY(cudaMemcpyAsync(twins_[i].dev, twins_[i].host, twins_[i].bytes, cudaMemcpyHostToDevice, stream_));
        return FA_OK;
    }
    // Queues the copy of every out / inout twin to its caller array: whole, or, when each holds `of` rows, its first
    // `rows` rows (outputs whose row count the device decides).
    cudaError_t back(size_t rows = 1, size_t of = 1) const {
        cudaError_t e = cudaSuccess;
        for (int i = 0; i < count_ && e == cudaSuccess; ++i) {
            const size_t bytes = twins_[i].bytes / of * rows;
            if ((twins_[i].dir & kOut) && bytes)
                e = cudaMemcpyAsync(twins_[i].host, twins_[i].dev, bytes, cudaMemcpyDeviceToHost, stream_);
        }
        return e;
    }
    // Queues the copy of the first n elements of one twin.
    template <typename T> cudaError_t back(T *p, const T *twin, size_t n) const {
        return host_ && p && n ? cudaMemcpyAsync(p, twin, n * sizeof(T), cudaMemcpyDeviceToHost, stream_) : cudaSuccess;
    }
    cudaError_t sync() const { return host_ ? cudaStreamSynchronize(stream_) : cudaSuccess; }
    // back() then sync(): the end of a host-buffer call whose outputs return whole
    cudaError_t finish() const {
        const cudaError_t e = back();
        return e != cudaSuccess ? e : sync();
    }

  private:
    enum : int { kIn = 1, kOut = 2, kMaxTwins = 16 };
    struct Twin {
        void *host, *dev;
        size_t bytes;
        int dir;
    };
    bool host_;
    cudaStream_t stream_;
    int count_ = 0;
    Twin twins_[kMaxTwins];
};

// Lays out one scratch arena in a grow-only buffer: a carve with Carver::take alone, which copies nothing.
template <typename T, bool Pinned, typename Layout>
int carve_arena(GrowBuffer<T, Pinned> &buf, Layout &&layout, size_t slack = 0) {
    return HostStaging(false, nullptr).carve(buf, layout, slack);
}

// Moves a session set's two per-slot device arrays (a_slot and b_slot elements per slot) into buffers of `grown` slots,
// keeping the first `slots`.  Both are allocated before anything is copied: a failed allocation changes neither.  The
// copies queue behind the set's pushes on `stream` and complete before the swap.
template <typename A, typename B>
int grow_slots(int slots, int grown, cudaStream_t stream, DeviceBuffer<A> &a, size_t a_slot, DeviceBuffer<B> &b,
               size_t b_slot) {
    DeviceBuffer<A> na;
    DeviceBuffer<B> nb;
    int st = na.grow((size_t)grown * a_slot * sizeof(A));
    if (st == FA_OK) st = nb.grow((size_t)grown * b_slot * sizeof(B));
    if (st != FA_OK) return st;
    if (slots) {
        FA_CUDA_TRY(cudaMemcpyAsync(na.data(), a.data(), (size_t)slots * a_slot * sizeof(A), cudaMemcpyDeviceToDevice, stream));
        FA_CUDA_TRY(cudaMemcpyAsync(nb.data(), b.data(), (size_t)slots * b_slot * sizeof(B), cudaMemcpyDeviceToDevice, stream));
        FA_CUDA_TRY(cudaStreamSynchronize(stream));
    }
    a = std::move(na);
    b = std::move(nb);
    return FA_OK;
}

// Owned stream and event: empty until create() succeeds, and usable wherever the raw handle is.
struct StreamDestroy {
    void operator()(cudaStream_t s) const { cudaStreamDestroy(s); }
};
struct EventDestroy {
    void operator()(cudaEvent_t e) const { cudaEventDestroy(e); }
};
struct Stream : std::unique_ptr<std::remove_pointer_t<cudaStream_t>, StreamDestroy> {
    operator cudaStream_t() const { return get(); }
    int create(unsigned flags = cudaStreamNonBlocking) {
        cudaStream_t s = nullptr;
        FA_CUDA_TRY(cudaStreamCreateWithFlags(&s, flags));
        reset(s);
        return FA_OK;
    }
};
struct Event : std::unique_ptr<std::remove_pointer_t<cudaEvent_t>, EventDestroy> {
    operator cudaEvent_t() const { return get(); }
    int create(unsigned flags = cudaEventDefault) {
        cudaEvent_t e = nullptr;
        FA_CUDA_TRY(cudaEventCreateWithFlags(&e, flags));
        reset(e);
        return FA_OK;
    }
};
// Creates both timer events, or neither: a failed creation leaves the timer unset, so the next start tries again.
inline int create_timer(Event (&ev)[2]) {
    int st = ev[0].create();
    if (st == FA_OK) st = ev[1].create();
    if (st != FA_OK) ev[0].reset();
    return st;
}

// Launch descriptors written in a pinned buffer and uploaded to its device twin.  An asynchronous call returns with its
// upload still queued, so the pinned copy may be rewritten (or replaced) only once that upload has read it: reserve()
// waits for the last upload before it grows the buffers, and upload() records the event reserve() waits on.
template <typename T = void> struct UploadStage {
    PinnedBuffer<T> host;
    DeviceBuffer<T> device;
    Event uploaded;
    bool in_flight = false;

    int reserve(size_t bytes) {
        if (in_flight) {
            FA_CUDA_TRY(cudaEventSynchronize(uploaded));
            in_flight = false;
        }
        const int st = device.grow(bytes);
        return st != FA_OK ? st : host.grow(bytes);
    }
    int upload(size_t bytes, cudaStream_t stream) {
        if (!uploaded) {
            const int st = uploaded.create(cudaEventDisableTiming);
            if (st != FA_OK) return st;
        }
        FA_CUDA_TRY(cudaMemcpyAsync(device.data(), host.data(), bytes, cudaMemcpyHostToDevice, stream));
        FA_CUDA_TRY(cudaEventRecord(uploaded, stream));
        in_flight = true;
        return FA_OK;
    }
};

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
