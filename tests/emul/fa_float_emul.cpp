// Host build of fluidaudio_b200/csrc/fa_float.cuh's f_exp / f_log / f_log1p, for tests/test_float_rounding.py:
// evaluates one over a range of float32 bit patterns.  Compiled with g++ -O2 -ffp-contract=off like the other
// host builds.  fn: 0 = exp, 1 = log, 2 = log1p.
#include "../../fluidaudio_b200/csrc/fa_float.cuh"

#include <cstdint>
#include <cstring>

extern "C" void fa_float_emul_eval(int fn, uint64_t start, uint64_t count, uint32_t *out) {
    for (uint64_t i = 0; i < count; ++i) {
        float x, y;
        const uint32_t b = uint32_t(start + i);
        std::memcpy(&x, &b, 4);
        y = fn == 0 ? fa::fp::f_exp(x) : fn == 1 ? fa::fp::f_log(x) : fa::fp::f_log1p(x);
        std::memcpy(&out[i], &y, 4);
    }
}
