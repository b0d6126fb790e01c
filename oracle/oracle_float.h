// ORACLE — TEST INFRASTRUCTURE ONLY.  Not part of the shipped product path.
//
// Correctly rounded float32 exp, log and log1p for the oracles: the float32 nearest the exact function of the float32
// argument, the definition the library's fa_float.cuh meets by other means (DESIGN §4.7).  Here each is evaluated in
// x87 80-bit long double (glibc's expl / logl / log1pl) and rounded once to float32.  The 11 extra bits put every
// result except log1p's near zero far enough from a float32 rounding boundary that the one rounding is right.  For
// |x| < 2^-12, log1p at 0x1.800006p-21 and -0x1.7ffffap-21 lies about 1e-13 float32 ulps from a float32 midpoint,
// closer than a long double ulp, so there the series x - x^2/2 + x^3/3 - ... is summed in long double with x^2 exact,
// the error of the final addition x + tail is recovered exactly (Fast2Sum), and a sum that lands exactly on a midpoint
// is moved to the side that error says.  tests/test_float_rounding.py checks all three functions on every float32
// input.
#pragma once

#include <cmath>

namespace oracle_float {

inline float exp32(float x) { return (float)expl((long double)x); }

inline float log32(float x) { return (float)logl((long double)x); }

inline float log1p32(float x) {
    const long double l = x;
    if (std::fabs(x) >= 0x1p-12f) return (float)log1pl(l);
    const long double t = l * l;   // exact: 48 significant bits
    // -x^2/2 + x^3/3 - ... - x^8/8; the omitted terms are below 2^-84 |x|
    const long double tail =
        t * (-0.5L + l * (1.0L / 3 + l * (-0.25L + l * (0.2L + l * (-1.0L / 6 + l * (1.0L / 7 - l * 0.125L))))));
    const long double s = l + tail;
    const long double err = tail - (s - l);   // exact: x + tail = s + err (|tail| < |x|)
    const float f = (float)s;
    if (err == 0 || (long double)f == s) return f;
    const float g = std::nextafter(f, s > f ? INFINITY : -INFINITY);   // the float on s's other side
    if ((long double)f + ((long double)g - f) / 2 != s) return f;     // s is not a midpoint: its rounding stands
    return (err > 0) == (g > f) ? g : f;
}

} // namespace oracle_float
