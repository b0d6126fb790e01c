// Index arithmetic of sinc_kernel (resample_kernels.cu), host- and device-callable so that the CPU suite checks the very
// code the kernel runs (tests/emul/resample_emul.cpp).
//
// Output i reads the 2H inputs n0(i) - H + 1 .. n0(i) + H, n0(i) = floor(i * M / L), at phase (i * M) mod L.  A CTA owns
// outputs i0 .. i0 + last (last <= 255) and stages inputs n0(i0) - H + 1 .. n0(i0 + last) + H in shared memory; thread j
// finds its window at offset dn = n0(i0 + j) - n0(i0) there.  make_design keeps L, M < 2^32 (resample_plan.h).
#pragma once

#include "fa_common.cuh"

namespace fa {
namespace resample {

constexpr int kSincBlock = 256;   // outputs per CTA

// n0(i0) and the phase of output i0 without forming i0 * M, which passes 2^63 for long outputs at large L and M:
// i0 = q L + r gives i0 M / L = q M + r M / L, and r M < L M < 2^64.
FA_HD void sinc_cta_base(long long i0, long long L, long long M, long long &n0, unsigned long long &ph) {
    const unsigned long long uL = (unsigned long long)L, uM = (unsigned long long)M;
    const unsigned long long q = (unsigned long long)i0 / uL, rm = ((unsigned long long)i0 - q * uL) * uM;
    n0 = (long long)(q * uM + rm / uL);
    ph = rm % uL;
}

// Output i0 + j of a CTA: n0 = n0(i0) + dn and its phase.  base_ph + j * M must fit T: with T = unsigned that is
// sinc_narrow_index(L, M); T = unsigned long long holds it for every L, M < 2^32.
template <typename T> FA_HD void sinc_offset(T base_ph, unsigned j, T L, T M, T &dn, T &ph) {
    const T t = base_ph + (T)j * M;
    dn = t / L;
    ph = t - dn * L;
}

// inputs a CTA stages: from n0(i0) - H + 1 through n0(i0 + last) + H, every tap of every output it owns
template <typename T> FA_HD int sinc_span(T base_ph, unsigned last, T L, T M, int half) {
    return (int)((base_ph + (T)last * M) / L) + 2 * half;
}

// 32-bit offsets suffice: base_ph + 255 * M <= L - 1 + 255 * M < 2^32
FA_HD bool sinc_narrow_index(long long L, long long M) { return 255 * M + L < (1LL << 32); }

// dynamic shared memory of one CTA in floats: the largest span (base_ph <= L - 1) with a few to spare
FA_HD long long sinc_smem_floats(long long L, long long M, int taps) { return (255 * M) / L + taps + 12; }

} // namespace resample
} // namespace fa
