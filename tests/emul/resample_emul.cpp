// Host check of sinc_kernel's index arithmetic (fluidaudio_b200/csrc/resample_core.cuh; CPU test-suite only).
// Runs the helpers the kernel runs for one CTA, thread by thread:
//   extern "C" int resample_index(L, M, half, i0, count, wide, n0[count], ph[count], dn[count], span[1])
//     wide = 1: 64-bit offsets, 0: 32-bit offsets (the kernel takes those only when sinc_narrow_index holds)
//   extern "C" int resample_narrow(L, M)              sinc_narrow_index
//   extern "C" long long resample_smem_floats(L, M, taps)
#include "../../fluidaudio_b200/csrc/resample_core.cuh"

using namespace fa::resample;

template <typename T>
static void cta(long long L, long long M, int half, long long i0, int count, long long *n0, long long *ph, long long *dn,
                long long *span) {
    long long base_n0;
    unsigned long long base_ph;
    sinc_cta_base(i0, L, M, base_n0, base_ph);
    *span = sinc_span<T>((T)base_ph, (unsigned)(count - 1), (T)L, (T)M, half);
    for (int j = 0; j < count; ++j) {
        T d, p;
        sinc_offset<T>((T)base_ph, (unsigned)j, (T)L, (T)M, d, p);
        n0[j] = base_n0 + (long long)d;
        ph[j] = (long long)p;
        dn[j] = (long long)d;
    }
}

extern "C" int resample_index(long long L, long long M, int half, long long i0, int count, int wide, long long *n0,
                              long long *ph, long long *dn, long long *span) {
    if (count < 1 || count > kSincBlock) return 1;
    if (wide) cta<unsigned long long>(L, M, half, i0, count, n0, ph, dn, span);
    else cta<unsigned>(L, M, half, i0, count, n0, ph, dn, span);
    return 0;
}

extern "C" int resample_narrow(long long L, long long M) { return sinc_narrow_index(L, M) ? 1 : 0; }

extern "C" long long resample_smem_floats(long long L, long long M, int taps) { return sinc_smem_floats(L, M, taps); }
