// Individually rounded float32 / float64 operations for the host- and device-callable arithmetic headers
// (prepare_core.cuh, sortformer_core.cuh, timeline_core.cuh), so that a kernel and its host build compute the same bits.
//
// On the device each helper is one __f*_rn / __d*_rn intrinsic, which the compiler never contracts into an FMA; on the
// host it is the plain operator, and every host build of these headers keeps contraction off.  Apple's vForce log /
// log1p are closed: f_log / f_log1p compute (float)log((double)x) and (float)log1p((double)x) on both sides instead.
// swift_min / swift_max restate Swift's min / max as the comparisons they are, so a NaN takes the branch it takes there.
#pragma once

#include "fa_common.cuh"

#include <cmath>

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
FA_HD float f_log(float x) { return (float)log((double)x); }
FA_HD float f_log1p(float x) { return (float)log1p((double)x); }

// Swift.min(x, y) = y < x ? y : x and Swift.max(x, y) = y >= x ? y : x
FA_HD float swift_min(float x, float y) { return y < x ? y : x; }
FA_HD float swift_max(float x, float y) { return y >= x ? y : x; }

} // namespace fp
} // namespace fa
