// oracle/oracle_float.h's exp32 / log32 / log1p32 over a range of float32 bit patterns, for
// tests/test_float_rounding.py.  Compiled with the oracles' flags (g++ -O2 -ffp-contract=off).  fn: 0 = exp, 1 = log,
// 2 = log1p.
#include "../../oracle/oracle_float.h"

#include <cstdint>
#include <cstring>

extern "C" void oracle_float_eval(int fn, uint64_t start, uint64_t count, uint32_t *out) {
    for (uint64_t i = 0; i < count; ++i) {
        float x, y;
        const uint32_t b = uint32_t(start + i);
        std::memcpy(&x, &b, 4);
        y = fn == 0 ? oracle_float::exp32(x) : fn == 1 ? oracle_float::log32(x) : oracle_float::log1p32(x);
        std::memcpy(&out[i], &y, 4);
    }
}
