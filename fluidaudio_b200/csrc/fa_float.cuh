// Individually rounded float32 / float64 operations for the host- and device-callable arithmetic headers
// (prepare_core.cuh, sortformer_core.cuh, timeline_core.cuh), so that a kernel and its host build compute the same bits.
//
// On the device each helper is one __f*_rn / __d*_rn intrinsic, which the compiler never contracts into an FMA; on the
// host it is the plain operator, and every host build of these headers keeps contraction off.  Apple's vForce log /
// log1p are closed: f_log / f_log1p compute (float)log((double)x) and (float)log1p((double)x) on both sides instead.
// swift_min / swift_max restate Swift's min / max as the comparisons they are, so a NaN takes the branch it takes there.
#pragma once

#include "fa_common.cuh"
#include "fa_float_table.h"

#include <cmath>
#include <cstdint>
#include <cstring>

namespace fa {
namespace fp {

#if defined(__CUDA_ARCH__)
FA_HD float f_add(float a, float b) { return __fadd_rn(a, b); }
FA_HD float f_sub(float a, float b) { return __fsub_rn(a, b); }
FA_HD float f_mul(float a, float b) { return __fmul_rn(a, b); }
FA_HD float f_div(float a, float b) { return __fdiv_rn(a, b); }
FA_HD float f_sqrt(float a) { return __fsqrt_rn(a); }
FA_HD double d_add(double a, double b) { return __dadd_rn(a, b); }
FA_HD double d_mul(double a, double b) { return __dmul_rn(a, b); }
#else
FA_HD float f_add(float a, float b) { return a + b; }
FA_HD float f_sub(float a, float b) { return a - b; }
FA_HD float f_mul(float a, float b) { return a * b; }
FA_HD float f_div(float a, float b) { return a / b; }
FA_HD float f_sqrt(float a) { return std::sqrt(a); }
FA_HD double d_add(double a, double b) { return a + b; }
FA_HD double d_mul(double a, double b) { return a * b; }
#endif

namespace cr {

#if defined(__CUDA_ARCH__)
FA_HD uint64_t bits_of(double d) { return (uint64_t)__double_as_longlong(d); }
FA_HD double double_of(uint64_t b) { return __longlong_as_double((long long)b); }
FA_HD uint32_t bits_of(float f) { return (uint32_t)__float_as_uint(f); }
FA_HD float float_of(uint32_t b) { return __uint_as_float(b); }
#else
FA_HD uint64_t bits_of(double d) { uint64_t b; std::memcpy(&b, &d, 8); return b; }
FA_HD double double_of(uint64_t b) { double d; std::memcpy(&d, &b, 8); return d; }
FA_HD uint32_t bits_of(float f) { uint32_t b; std::memcpy(&b, &f, 4); return b; }
FA_HD float float_of(uint32_t b) { float f; std::memcpy(&f, &b, 4); return f; }
#endif

constexpr uint64_t kWindow = 3;   // float64 ulps either side of the result

// Whether float32 rounding changes within kWindow float64 ulps of the finite d: the float32 of |d| stepped kWindow ulps
// down and up differ.  Covers midpoints between normal and subnormal float32 values alike, and the overflow threshold.
FA_HD bool near_boundary(double d) {
    const uint64_t b = bits_of(d) & ~(1ull << 63);
    if (b >= 0x7ff0000000000000ull) return false;   // inf, NaN
    return (float)double_of(b < kWindow ? 0 : b - kWindow) != (float)double_of(b + kWindow);
}

// The float32 result of input x from table[0, n) (sorted by input bits), or fallback when x is not there.
FA_HD float lookup(const uint32_t (*table)[2], int n, float x, double fallback) {
    const uint32_t key = bits_of(x);
    int lo = 0, hi = n;
    while (lo < hi) {
        const int mid = (lo + hi) / 2;
        if (table[mid][0] < key) lo = mid + 1;
        else hi = mid;
    }
    return lo < n && table[lo][0] == key ? float_of(table[lo][1]) : (float)fallback;
}

} // namespace cr

FA_HD float f_exp(float x) {
    static constexpr uint32_t table[][2] = {FA_CR_EXP_TABLE};
    const double d = exp((double)x);
    return cr::near_boundary(d) ? cr::lookup(table, cr::kExpCount, x, d) : (float)d;
}
FA_HD float f_log(float x) {
    static constexpr uint32_t table[][2] = {FA_CR_LOG_TABLE};
    const double d = log((double)x);
    return cr::near_boundary(d) ? cr::lookup(table, cr::kLogCount, x, d) : (float)d;
}
FA_HD float f_log1p(float x) {
    static constexpr uint32_t table[][2] = {FA_CR_LOG1P_TABLE};
    const double d = log1p((double)x);
    return cr::near_boundary(d) ? cr::lookup(table, cr::kLog1pCount, x, d) : (float)d;
}

// Swift.min(x, y) = y < x ? y : x and Swift.max(x, y) = y >= x ? y : x
FA_HD float swift_min(float x, float y) { return y < x ? y : x; }
FA_HD float swift_max(float x, float y) { return y >= x ? y : x; }

} // namespace fp
} // namespace fa
