// The reference for the float32 exp / log / log1p helpers, over every float32 bit pattern.  It shares no code with
// fluidaudio_b200/csrc/fa_float.cuh or oracle/oracle_float.h: the value at x is glibc's float64 function rounded once
// to float32, except at the "fragile" inputs, where the float64 result lies within 3 float64 ulps of a point at which
// float32 rounding changes (a midpoint, or the overflow threshold).  There the caller supplies the correctly rounded
// value (tests/float_exact.py resolves it with mpmath), so the reference is correctly rounded on every input.
//
// fn: 0 = exp, 1 = log, 2 = log1p.  NaN results compare equal to any NaN.
#include <algorithm>
#include <atomic>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <mutex>
#include <thread>
#include <vector>

namespace {

constexpr int kWindow = 3;

double eval64(int fn, float x) {
    const double d = x;
    return fn == 0 ? std::exp(d) : fn == 1 ? std::log(d) : std::log1p(d);
}

float bits_to_float(uint32_t b) { float f; std::memcpy(&f, &b, 4); return f; }
uint32_t float_bits(float f) { uint32_t b; std::memcpy(&b, &f, 4); return b; }

double step(double d, int64_t n) {   // d moved n float64 ulps away from zero (n may be negative), d >= 0 and finite
    uint64_t b; std::memcpy(&b, &d, 8);
    b = n < 0 && b < uint64_t(-n) ? 0 : b + n;
    std::memcpy(&d, &b, 8);
    return d;
}

// Whether float32 rounding of |d| changes anywhere within kWindow float64 ulps of it.
bool fragile(double d) {
    if (!std::isfinite(d)) return false;
    const double a = std::fabs(d);
    return (float)step(a, -kWindow) != (float)step(a, kWindow);
}

unsigned threads() { return std::max(1u, std::thread::hardware_concurrency()); }

// Runs body(lo, hi) over [0, 2^32) in 2^20-input blocks handed out to every hardware thread.
template <class F> void parallel_all(F body) {
    std::atomic<uint64_t> next{0};
    const uint64_t block = 1u << 20, total = uint64_t(1) << 32;
    std::vector<std::thread> pool;
    for (unsigned t = 0; t < threads(); ++t)
        pool.emplace_back([&] {
            for (uint64_t lo; (lo = next.fetch_add(block)) < total;) body(lo, lo + block);
        });
    for (auto& th : pool) th.join();
}

struct Fixups {
    const uint32_t* in;
    const uint32_t* val;
    int64_t n;
    bool find(uint32_t x, uint32_t* v) const {
        const uint32_t* p = std::lower_bound(in, in + n, x);
        if (p == in + n || *p != x) return false;
        *v = val[p - in];
        return true;
    }
};

uint32_t ref_bits(int fn, uint32_t xb, const Fixups& fx) {
    const float x = bits_to_float(xb);
    const double d = eval64(fn, x);
    uint32_t v;
    if (fragile(d) && fx.find(xb, &v)) return v;
    return float_bits((float)d);
}

bool same(uint32_t a, uint32_t b) {
    return a == b || (std::isnan(bits_to_float(a)) && std::isnan(bits_to_float(b)));
}

} // namespace

extern "C" {

// Every input whose float64 result is fragile, ascending, into out[0, cap); returns how many there are.
int64_t fr_scan(int fn, uint32_t* out, int64_t cap) {
    std::mutex m;
    std::vector<uint32_t> all;
    parallel_all([&](uint64_t lo, uint64_t hi) {
        std::vector<uint32_t> mine;
        for (uint64_t x = lo; x < hi; ++x)
            if (fragile(eval64(fn, bits_to_float(uint32_t(x))))) mine.push_back(uint32_t(x));
        std::lock_guard<std::mutex> g(m);
        all.insert(all.end(), mine.begin(), mine.end());
    });
    std::sort(all.begin(), all.end());
    for (int64_t i = 0; i < (int64_t)all.size() && i < cap; ++i) out[i] = all[i];
    return (int64_t)all.size();
}

// The reference at inputs[0, count), or at [start, start + count) when inputs is null, into out, with the fragile
// inputs' values from (fin, fval), sorted.
void fr_reference(int fn, uint64_t start, uint64_t count, const uint32_t* inputs, const uint32_t* fin,
                  const uint32_t* fval, int64_t nf, uint32_t* out) {
    if (count == 0) return;
    const Fixups fx{fin, fval, nf};
    const uint64_t per = (count + threads() - 1) / threads();
    std::vector<std::thread> pool;
    for (uint64_t lo = 0; lo < count; lo += per)
        pool.emplace_back([&, lo] {
            for (uint64_t i = lo; i < std::min(count, lo + per); ++i)
                out[i] = ref_bits(fn, inputs ? inputs[i] : uint32_t(start + i), fx);
        });
    for (auto& th : pool) th.join();
}

// Evaluates an implementation over [start, start + count) into out (float32 bits).
typedef void (*eval_range_fn)(int fn, uint64_t start, uint64_t count, uint32_t* out);

// Compares impl with the reference on all 2^32 inputs; returns the number of mismatches and writes the first cap of
// them as (input, got, expected) triples into bad.
int64_t fr_check(int fn, eval_range_fn impl, const uint32_t* fin, const uint32_t* fval, int64_t nf, uint32_t* bad,
                 int64_t cap) {
    const Fixups fx{fin, fval, nf};
    std::atomic<int64_t> n_bad{0};
    parallel_all([&](uint64_t lo, uint64_t hi) {
        std::vector<uint32_t> got(hi - lo);
        impl(fn, lo, hi - lo, got.data());
        for (uint64_t x = lo; x < hi; ++x) {
            const uint32_t want = ref_bits(fn, uint32_t(x), fx), g = got[x - lo];
            if (same(g, want)) continue;
            const int64_t k = n_bad.fetch_add(1);
            if (k < cap) { bad[3 * k] = uint32_t(x); bad[3 * k + 1] = g; bad[3 * k + 2] = want; }
        }
    });
    return n_bad.load();
}

} // extern "C"
