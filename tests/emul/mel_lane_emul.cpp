// Host lane-emulator of mel512_kernel's band sums, in the device's order (CPU and GPU test-suites; compiled with
// fluidaudio_b200/csrc/mel_tables.cpp by g++ -O2 -ffp-contract=off, so every float32 operation rounds as written).
// The transform is mel_core.cuh run lane by lane, as in mel_emul.cpp; the filterbank stage restates mel_dot_pairs: the
// plan's packed bands (pack_bands / pack_weights, swizzled, times 1/4) and one fmaf chain per mel over the band's bin quads
// in power-row position order, zero weights and the row's zero pad columns included.  On the float32-pair path every
// device operation before the log is an explicit round-to-nearest float32 operation, so these band sums are the device's
// bit for bit; the FP64 path differs only where nvcc contracts double multiply-adds.
//   extern "C" int mel_lane_frames(f32, audio, n, last, hop, win, off, pad, preemph, n_mels, fb[n_mels*257], window[win],
//                                  log_floor, clamped, T, defects, power[T*257] | null, E[T*n_mels], x[T*n_mels],
//                                  out[T*n_mels] | null)
//       f32: 0 the FP64 transform (one frame per warp), 1 float32 pairs.  power: 4|X_b|^2 in bin order; E: band sums; x:
//       the log argument; out: logf(x), the host's libm.
//   extern "C" int mel_lane_dot(power[rows*257], rows, n_mels, fb, defects, log_floor, clamped, E[rows*n_mels],
//                               x[rows*n_mels])
//       the filterbank stage alone, on power rows given in bin order.
// `defects` (0 = the kernel as written) injects one kernel defect per bit (kDefect* below), for the tests that show the
// comparison catches it.
#include "mel_core.cuh"
#include "mel_tables.h"

#include <algorithm>
#include <cmath>
#include <cstring>
#include <vector>

using namespace fa::mel;

enum {
    kDefectTwiddle = 1,        // lane 1's tw1[1] (W256^1) real part rounded one ulp toward zero
    kDefectWindow = 2,         // the window coefficient at win / 2 one ulp larger
    kDefectPowerMulAdd = 4,    // power xr*xr + xi*xi with three roundings instead of the FMA
    kDefectDotMulAdd = 8,      // band sum with separate multiply and add over the bare band: mel_dot
    kDefectTileFirst = 16,     // a tile's first sample (audio index >= 1) pre-emphasised with preemph_first
                               // (invisible: it feeds only buffer position 0 of the tile's first frame, see the tests)
    kDefectLastZero = 32,      // `last` taken as 0 for sample 0 of the clip
    kDefectNoSwizzle = 64,     // the band sum reads the power row in bin order against the swizzled weights
    kDefectStepFirst = 128,    // on a tile that takes the float4 interior pre-emphasis, the first sample of every step
                               // (whose predecessor comes from the step before) pre-emphasised with preemph_first
};

namespace {

struct Bands {
    MelBands b;
    std::vector<float> w;      // packed, swizzled, times 1/4: the plan's d_fb_w
    std::vector<float> fbq;    // dense filterbank times 1/4, and the bare band [lo0, hi0): mel_dot's operands
    std::vector<int> lo0, hi0;
};

Bands bands_of(const float *fb, int n_mels) {
    Bands B;
    const std::vector<float> dense(fb, fb + (size_t)n_mels * kBins);
    B.b = pack_bands(dense, n_mels, kBins);
    B.w = pack_weights(dense, B.b, kBins, true, 0.25f);
    B.fbq.resize(dense.size());
    for (size_t i = 0; i < dense.size(); ++i) B.fbq[i] = 0.25f * dense[i];
    B.lo0.assign(n_mels, 0);
    B.hi0.assign(n_mels, 0);
    for (int m = 0; m < n_mels; ++m) {
        int a = kBins, e = 0;
        for (int k = 0; k < kBins; ++k)
            if (dense[(size_t)m * kBins + k] != 0.0f) {
                a = std::min(a, k);
                e = k + 1;
            }
        B.lo0[m] = e ? a : 0;
        B.hi0[m] = e;
    }
    return B;
}

// log argument as log_value (mel_core.cuh) forms it
float log_arg(float v, float floor_, int clamped) { return clamped ? (floor_ >= v ? floor_ : v) : v + floor_; }

// One frame's band sums from its power row p (bin order, 257 values).
void band_sums(const Bands &B, const float *p, int n_mels, int defects, float *E) {
    float row[260];                       // the pair row's slot of this frame, positions 0..259; 257..259 are pad (zero)
    std::memset(row, 0, sizeof(row));
    for (int b = 0; b < kBins; ++b) row[(defects & kDefectNoSwizzle) ? b : pow_pos(b)] = p[b];
    for (int m = 0; m < n_mels; ++m) {
        if (defects & kDefectDotMulAdd) {
            float nat[kBins];
            std::memcpy(nat, p, sizeof(nat));
            E[m] = mel_dot(nat, B.fbq.data() + (size_t)m * kBins + B.lo0[m], B.lo0[m], B.hi0[m]);
            continue;
        }
        const int lo = B.b.lo[m], hi = B.b.hi[m];
        const float *w = B.w.data() + B.b.off[m];
        float acc = 0.0f;
        for (int k = lo; k < hi; ++k) acc = fmaf(row[k], w[k - lo], acc);   // mel_dot_pairs: ffma2_rn(x, c, acc)
        E[m] = acc;
    }
}

void twiddle_defect(LaneTables<double> &) {}
void twiddle_defect(LaneTables<f32x2> &t) { t.tw1[1].x = nextafterf(t.tw1[1].x, 0.0f); }

// kDefectPowerMulAdd: pass3_post of mel_core.cuh with the float32 pair power rounded three times (xr*xr + xi*xi); the
// FP64 path already forms its power that way, so there it is the kernel's own pass3_post
struct PowerMulAdd {
    void operator()(f32x2 zbx, f32x2 zby, f32x2 zcx, f32x2 zcy, float wx, float wy, float *prow, int ib, int ic) const {
        const f32x2 sr = vadd(zbx, zcx), si = vsub(zby, zcy);
        const f32x2 dr = vadd(zby, zcy), di = vsub(zcx, zbx);
        const f32x2 tr = vfnma_s(di, wy, vmul_s(dr, wx)), ti = vfma_s(dr, wy, vmul_s(di, wx));
        const f32x2 xr = vadd(sr, tr), xi = vadd(si, ti);
        const f32x2 yr = vsub(sr, tr), yi = vsub(si, ti);
        const float a = xr.a * xr.a, b = xi.a * xi.a, c = yr.a * yr.a, d = yi.a * yi.a;
        const float a2 = xr.b * xr.b, b2 = xi.b * xi.b, c2 = yr.b * yr.b, d2 = yi.b * yi.b;
        prow[2 * ib] = a + b;
        prow[2 * ic] = c + d;
        prow[2 * ib + 1] = a2 + b2;
        prow[2 * ic + 1] = c2 + d2;
    }
};
void pass3_defect(int l, const cpxv<f32x2> *buf, const LaneTables<f32x2> &T, float *prow) {
    const PowerMulAdd pp;
    f32x2 ar[4], ai[4], br[4], bi[4];
    for (int h = 0; h < 4; ++h) {
        const cpxv<f32x2> u = buf[T.a1 + 74 * h], v = buf[T.a2 + 74 * h];
        ar[h] = u.x;
        ai[h] = u.y;
        br[h] = v.x;
        bi[h] = v.y;
    }
    dft4(ar[0], ai[0], ar[1], ai[1], ar[2], ai[2], ar[3], ai[3]);
    dft4(br[0], bi[0], br[1], bi[1], br[2], bi[2], br[3], bi[3]);
    const bool z = l == 0;
    const float c1 = 0.92387953251128675613f, s1 = 0.38268343236508977173f;
    float wx[4], wy[4];
    recombination_roots(T, wx, wy);
    pp(ar[0], ai[0], z ? ar[0] : br[3], z ? ai[0] : bi[3], wx[0], wy[0], prow, T.k0s, T.kc0s);
    pp(ar[1], ai[1], z ? ar[3] : br[2], z ? ai[3] : bi[2], wx[1], wy[1], prow, T.k0s + 64, T.kc0s - 64);
    pp(ar[2], ai[2], z ? ar[2] : br[1], z ? ai[2] : bi[1], wx[2], wy[2], prow, T.k0s + 128, T.kc0s - 128);
    const int b3 = z ? pow_pos(32) : T.k0s + 192, c3 = z ? pow_pos(224) : T.kc0s - 192;
    pp(z ? br[0] : ar[3], z ? bi[0] : ai[3], z ? br[3] : br[0], z ? bi[3] : bi[0], z ? c1 : wx[3], z ? -s1 : wy[3], prow,
       b3, c3);
    if (z) pp(br[1], bi[1], br[2], bi[2], s1, -c1, prow, pow_pos(96), pow_pos(160));
}
void pass3(int l, const cpxv<double> *buf, const LaneTables<double> &T, float *prow, int) { pass3_post(l, buf, T, prow); }
void pass3(int l, const cpxv<f32x2> *buf, const LaneTables<f32x2> &T, float *prow, int defects) {
    if (defects & kDefectPowerMulAdd) pass3_defect(l, buf, T, prow);
    else pass3_post(l, buf, T, prow);
}

template <typename V>
int frames_t(const float *audio, long long n, float last, int hop, int win, int off, int pad, float preemph, int n_mels,
             const float *fb, const float *window, float log_floor, int clamped, long long T, int defects, float *power,
             float *E, float *x, float *out) {
    constexpr int kF = vtraits<V>::kFrames;
    if (hop & 1) return 1;
    std::vector<float> wv(window, window + win);
    if (defects & kDefectWindow) wv[win / 2] = nextafterf(wv[win / 2], INFINITY);
    std::vector<float> win_tab;
    std::vector<uint8_t> in_tab;
    place_window(wv, kNfft, off, win_tab, in_tab);
    std::vector<LaneTables<V>> tabs(32);
    for (int l = 0; l < 32; ++l) load_lane_tables(l, win_tab.data(), in_tab.data(), tabs[l]);
    if (defects & kDefectTwiddle) twiddle_defect(tabs[1]);
    const bool mid_full = off <= 64 && off + win >= 448;
    const Bands B = bands_of(fb, n_mels);
    alignas(16) cpxv<V> buf[kFftPad];
    std::vector<float> pfv((size_t)kNfft + hop + 8);
    float *pf = pfv.data();
    std::vector<float> prow2(kPairStride);
    float p[kBins];
    for (long long f = 0; f < T; f += kF) {
        // the kernel's tiles are kTileFrames frames from the clip's first: both frames of a pair lie in one tile, whose
        // pre-emphasis starts at audio index a0 (only frame f0 of the tile reads that sample, at buffer position 0)
        const long long a0 = (f - f % kTileFrames) * hop - pad;
        const long long pt_len = (long long)(kTileFrames - 1) * hop + kNfft;
        const bool float4_tile = (hop & 3) == 0 && a0 >= 1 && a0 + pt_len <= (n & ~3LL);   // preemphasize()'s interior test
        for (int j = 0; j < kNfft + (kF - 1) * hop; ++j) {
            const long long i = f * hop + j - pad;
            float v = 0.0f;
            if (i >= 0 && i < n) {
                if (preemph == 0.0f) v = audio[i];
                else if (i == 0) v = preemph_first(audio[0], (defects & kDefectLastZero) ? 0.0f : last, preemph);
                else if ((defects & kDefectTileFirst) && i == a0) v = preemph_first(audio[i], audio[i - 1], preemph);
                else if ((defects & kDefectStepFirst) && float4_tile && ((i - a0) & 3) == 0)
                    v = preemph_first(audio[i], audio[i - 1], preemph);
                else v = preemph_rest(audio[i], audio[i - 1], preemph);
            }
            pf[j] = v;
        }
        std::memset((void *)buf, 0, sizeof(buf));
        V re[32][8], im[32][8];
        for (int l = 0; l < 32; ++l) {
            if (mid_full) pass1<true>(l, pf, hop, tabs[l], buf); else pass1<false>(l, pf, hop, tabs[l], buf);
        }
        for (int l = 0; l < 32; ++l) pass2_load(l, buf, re[l], im[l]);
        for (int l = 0; l < 32; ++l) pass2_store(l, tabs[l], re[l], im[l], buf);
        std::fill(prow2.begin(), prow2.end(), 0.0f);
        for (int l = 0; l < 32; ++l) pass3(l, buf, tabs[l], prow2.data(), defects);
        for (int k = 0; k < kF && f + k < T; ++k) {
            for (int b = 0; b < kBins; ++b) p[b] = prow2[2 * pow_pos(b) + k];
            if (power) std::memcpy(power + (f + k) * kBins, p, sizeof(p));
            float *e = E + (f + k) * n_mels;
            band_sums(B, p, n_mels, defects, e);
            for (int m = 0; m < n_mels; ++m) {
                x[(f + k) * n_mels + m] = log_arg(e[m], log_floor, clamped);
                if (out) out[(f + k) * n_mels + m] = log_value(e[m], log_floor, clamped);
            }
        }
    }
    return 0;
}

} // namespace

extern "C" int mel_lane_frames(int f32, const float *audio, long long n, float last, int hop, int win, int off, int pad,
                               float preemph, int n_mels, const float *fb, const float *window, float log_floor,
                               int clamped, long long T, int defects, float *power, float *E, float *x, float *out) {
    return f32 ? frames_t<f32x2>(audio, n, last, hop, win, off, pad, preemph, n_mels, fb, window, log_floor, clamped, T,
                                 defects, power, E, x, out)
               : frames_t<double>(audio, n, last, hop, win, off, pad, preemph, n_mels, fb, window, log_floor, clamped, T,
                                  defects, power, E, x, out);
}

extern "C" int mel_lane_dot(const float *power, long long rows, int n_mels, const float *fb, int defects, float log_floor,
                            int clamped, float *E, float *x) {
    const Bands B = bands_of(fb, n_mels);
    for (long long r = 0; r < rows; ++r) {
        band_sums(B, power + r * kBins, n_mels, defects, E + r * n_mels);
        for (int m = 0; m < n_mels; ++m) x[r * n_mels + m] = log_arg(E[r * n_mels + m], log_floor, clamped);
    }
    return 0;
}
