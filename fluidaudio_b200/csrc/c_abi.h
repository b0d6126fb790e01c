// The guard every status-returning C ABI entry point returns through (capi.cu, the *_abi.cu files, export_io.cu).  No
// exception crosses the extern "C" boundary, and a failing call leaves fa_last_error() text that describes its own
// failure.
#pragma once

#include "../../include/fluidaudio_b200.h"
#include "fa_common.cuh"

#include <cstdint>
#include <exception>
#include <new>

#define FA_API extern "C" __attribute__((visibility("default")))

namespace fa {

// Number of set_error calls on this thread so far: a call that leaves it unchanged has set no text.
unsigned error_serial();
// "FA_STATUS_INVALID_ARGUMENT" and so on.
const char *status_name(int status);
// FA_OK when an sm_90a device is visible, else FA_NO_DEVICE with error text (entry points that create a handle).
int require_device();
// A caller's buffer capacity as the library's signed lengths: one of 2^63 elements or more is as good as unlimited.
inline long long capacity(size_t n) { return n > (size_t)INT64_MAX ? INT64_MAX : (long long)n; }

// Runs `body` (returning an int status) and turns any exception it throws into a status with error text.  It throws
// nothing, so a thread of its own can run it (cluster_batch's lanes do).
template <typename F> int run_guarded(F &&body) noexcept {
    try {
        return body();
    } catch (const std::bad_alloc &) {
        set_error("host allocation failed");
        return FA_ALLOCATION_FAILURE;
    } catch (const std::exception &ex) {
        set_error("exception: %s", ex.what());
        return FA_RUNTIME_ERROR;
    } catch (...) {
        set_error("unknown exception");
        return FA_UNKNOWN_ERROR;
    }
}

// The body of the entry point `entry`.  A failure that set no text of its own gets "<entry>: <status name>", so the
// text of an earlier failure is never reported for this one.
template <typename F> fa_status guard(const char *entry, F &&body) noexcept {
    const unsigned serial = error_serial();
    const int st = run_guarded(body);
    if (st != FA_OK && error_serial() == serial) set_error("%s: %s", entry, status_name(st));
    return (fa_status)st;
}

} // namespace fa
