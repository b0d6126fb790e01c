// Device-side AudioConverter stage: PCM (float32 / int16, any channel count, planar or interleaved, any rate) ->
// mono float32 at the model rate, written straight into the buffer the log-mel kernel reads (no host round trip).
// See resample_plan.h for the reference lines and the filter design.
#include "resample_plan.h"
#include "call_context.h"
#include "resample_core.cuh"

#include <algorithm>
#include <cmath>
#include <numeric>

namespace fa {
namespace resample {

// ------------------------------------------------------------------------------------------------ design (host)
bool rational_ratio(double in_rate, double out_rate, long long &L, long long &M) {
    double scale = 1.0;
    if (std::fabs(in_rate - std::round(in_rate)) > 1e-9 || std::fabs(out_rate - std::round(out_rate)) > 1e-9) scale = 1000.0;
    if (!(out_rate * scale < 0x1p53) || !(in_rate * scale < 0x1p53)) return false;   // past 2^53 the grid is not exact
    const long long a = (long long)std::llround(out_rate * scale), b = (long long)std::llround(in_rate * scale);
    if (a <= 0 || b <= 0) return false;
    const long long g = std::gcd(a, b);
    L = a / g;
    M = b / g;
    return std::fabs((double)a / scale - out_rate) < 1e-6 && std::fabs((double)b / scale - in_rate) < 1e-6;
}

static double bessel_i0(double x) {   // power series, converges for every x; 60 terms are exact to double for x <= 20
    double sum = 1.0, term = 1.0;
    const double q = 0.25 * x * x;
    for (int k = 1; k < 200; ++k) {
        term *= q / ((double)k * (double)k);
        sum += term;
        if (term < 1e-18 * sum) break;
    }
    return sum;
}

int make_design(double in_rate, double out_rate, Design &d) {
    if (!(in_rate > 0) || !(out_rate > 0)) return FA_INVALID_ARGUMENT;
    if (!rational_ratio(in_rate, out_rate, d.L, d.M)) {
        fa::set_error("sample rates %.6f -> %.6f are not on a 1/1000 Hz grid", in_rate, out_rate);
        return FA_UNSUPPORTED;
    }
    if (d.L >= (1LL << 32) || d.M >= (1LL << 32)) {   // sinc_kernel's phase arithmetic (resample_core.cuh)
        fa::set_error("sample rates %.6f -> %.6f reduce to %lld/%lld: terms of 2^32 or more are not supported", in_rate,
                      out_rate, d.L, d.M);
        return FA_UNSUPPORTED;
    }
    const double lower = std::min(1.0, (double)d.L / (double)d.M);
    d.fc = lower * kRolloff;
    d.half = (int)std::ceil((double)kZeros / lower);
    d.taps = 2 * d.half;
    d.exact = d.L <= kMaxExactPhases;
    d.phases = d.exact ? (int)d.L : kInterpPhases;
    if ((255.0 * (double)d.M / (double)d.L + d.taps + 8) * sizeof(float) > 200.0 * 1024.0) {
        fa::set_error("resampling ratio %lld/%lld needs a filter window larger than shared memory", d.L, d.M);
        return FA_UNSUPPORTED;
    }
    const int rows = d.exact ? d.phases : d.phases + 1;
    d.row_stride = (d.taps + 3) & ~3;   // rows padded with zero taps to whole float4s (16-byte aligned coefficient loads)
    d.table.assign((size_t)rows * d.row_stride, 0.0f);
    const double pi = 3.14159265358979323846, i0b = bessel_i0(kBeta);
    std::vector<double> row(d.taps);
    for (int p = 0; p < rows; ++p) {
        const double frac = (double)p / (double)d.phases;
        double sum = 0.0;
        for (int k = 0; k < d.taps; ++k) {
            const double t = (double)(k - d.half + 1) - frac;   // input sample n0 - H + 1 + k sits at offset t from the output
            double g = 0.0;
            if (std::fabs(t) < (double)d.half) {
                const double x = pi * d.fc * t;
                const double s = std::fabs(x) < 1e-12 ? 1.0 : std::sin(x) / x;
                const double u = t / (double)d.half;
                g = d.fc * s * bessel_i0(kBeta * std::sqrt(std::max(0.0, 1.0 - u * u))) / i0b;
            }
            row[k] = g;
            sum += g;
        }
        for (int k = 0; k < d.taps; ++k) d.table[(size_t)p * d.row_stride + k] = (float)(row[k] / sum);
    }
    return FA_OK;
}

long long output_count(long long frames, double in_rate, double out_rate) {
    if (in_rate == out_rate) return frames;
    const double ratio = in_rate / out_rate;
    return (long long)((double)frames / ratio);   // AudioConverter.swift:417-418
}

bool is_identity(const AudioFormat &f) {
    return f.in_rate == f.out_rate && f.channels == 1 && f.format == kPcmF32;
}

int resolve_algorithm(const AudioFormat &f) {
    if (f.algorithm == kAlgoSinc || f.algorithm == kAlgoLinear) return f.algorithm;
    return f.channels > 2 ? kAlgoLinear : kAlgoSinc;
}

long long outputs_ready(const AudioFormat &f, const Design &d, long long frames, long long frames_avail,
                        long long out_total) {
    if (frames_avail >= frames) return out_total;
    long long ready;
    if (f.in_rate == f.out_rate) ready = frames_avail;
    else if (resolve_algorithm(f) == kAlgoLinear) ready = (long long)((double)(frames_avail - 2) / (f.in_rate / f.out_rate)) - 1;
    else ready = ((frames_avail - d.half - 1) * d.L) / d.M - 1;   // n0(i) + H < frames_avail
    return std::max(0LL, std::min(ready, out_total));
}

// ------------------------------------------------------------------------------------------------ kernels
struct Source {
    const void *pcm;
    long long frames;
    int channels;
    int format;
    int interleaved;
    float weight;   // 1 / channels (float32, AudioConverter.swift:401)
};

// mono sample n: float32 sum over channels in channel order, times 1/channels (AudioConverter.swift:403-409).
// int16 is widened like AVAudioPCMBuffer's int16 -> float conversion: v / 32768.
__device__ __forceinline__ float mono_at(const Source &s, long long n) {
    if (s.channels == 1)   // the common mono cases without the channel loop
        return s.format == kPcmI16 ? (float)__ldg(reinterpret_cast<const short *>(s.pcm) + n) * (1.0f / 32768.0f)
                                   : __ldg(reinterpret_cast<const float *>(s.pcm) + n);
    if (s.channels == 2 && s.interleaved && s.format == kPcmI16) {   // stereo WAV: one 32-bit load per frame
        const short2 v = __ldg(reinterpret_cast<const short2 *>(s.pcm) + n);
        return __fmul_rn(__fadd_rn(__fadd_rn(0.0f, (float)v.x * (1.0f / 32768.0f)), (float)v.y * (1.0f / 32768.0f)), s.weight);
    }
    float sum = 0.0f;
    for (int c = 0; c < s.channels; ++c) {
        const long long at = s.interleaved ? n * s.channels + c : (long long)c * s.frames + n;
        const float v = s.format == kPcmI16 ? (float)__ldg(reinterpret_cast<const short *>(s.pcm) + at) * (1.0f / 32768.0f)
                                            : __ldg(reinterpret_cast<const float *>(s.pcm) + at);
        sum = __fadd_rn(sum, v);
    }
    return s.channels == 1 ? sum : __fmul_rn(sum, s.weight);
}

// same rate: mixdown / format conversion only
__global__ void __launch_bounds__(256) mixdown_kernel(Source s, float *out, long long o_begin, long long o_end) {
    const long long i = o_begin + (long long)blockIdx.x * 256 + threadIdx.x;
    if (i < o_end) out[i] = i < s.frames ? mono_at(s, i) : 0.0f;
}

// AudioConverter.linearResample (:417-434), float32 operations individually rounded, source position in double
__global__ void __launch_bounds__(256) linear_kernel(Source s, double ratio, float *out, long long o_begin, long long o_end) {
    const long long i = o_begin + (long long)blockIdx.x * 256 + threadIdx.x;
    if (i >= o_end) return;
    const double src = (double)i * ratio;
    const long long idx = (long long)src;
    const float frac = (float)(src - (double)idx);
    float v = 0.0f;
    if (idx < s.frames - 1)
        v = __fadd_rn(__fmul_rn(mono_at(s, idx), __fsub_rn(1.0f, frac)), __fmul_rn(mono_at(s, idx + 1), frac));
    else if (idx < s.frames)
        v = mono_at(s, idx);
    out[i] = v;
}

// Kaiser-windowed-sinc polyphase.  One CTA = 256 consecutive outputs; their input span (mixed down, widened) is staged
// in shared memory once, every thread then runs its 2H-tap dot product out of shared memory: coefficients as 16-byte
// loads through the read-only path (a single row when L == 1, i.e. integer decimation: every lane reads the same
// address), four independent accumulators, index arithmetic relative to one 64-bit division per CTA (resample_core.cuh).
// Idx = unsigned when base_ph + 255 * M fits 32 bits (sinc_narrow_index: every whole-Hz pair of audio rates), else
// unsigned long long.  Rows are padded to whole float4s, so when H is odd the last float4 holds two zero taps: they are
// skipped, not multiplied, so that an output depends on its 2H-tap window only (0 * NaN would be NaN).
template <typename Idx>
__global__ void __launch_bounds__(kSincBlock)
sinc_kernel(Source s, long long L, long long M, int half, int phases, int exact, int row_stride,
            const float *__restrict__ tab, float *out, long long o_begin, long long o_end) {
    extern __shared__ float xs[];
    __shared__ long long base_n0;
    __shared__ Idx base_ph;
    const long long i0 = o_begin + (long long)blockIdx.x * kSincBlock;
    if (threadIdx.x == 0) {
        long long n0;
        unsigned long long ph;
        sinc_cta_base(i0, L, M, n0, ph);
        base_n0 = n0;
        base_ph = (Idx)ph;
    }
    __syncthreads();
    const Idx uL = (Idx)L, uM = (Idx)M;
    const int last = (int)(min(i0 + kSincBlock - 1, o_end - 1) - i0);
    const long long n_lo = base_n0 - half + 1;
    const int span = sinc_span<Idx>(base_ph, (unsigned)last, uL, uM, half);
    for (int j = threadIdx.x; j < span; j += kSincBlock) {
        const long long n = n_lo + j;
        xs[j] = (n >= 0 && n < s.frames) ? mono_at(s, n) : 0.0f;
    }
    __syncthreads();
    const long long i = i0 + threadIdx.x;
    if (i >= o_end) return;
    Idx dn, ph;
    sinc_offset<Idx>(base_ph, threadIdx.x, uL, uM, dn, ph);
    const float *x = xs + dn;          // input n0 - H + 1 + k sits at xs[dn + k]
    const int nq = half >> 1;          // whole float4s of taps; with H odd two more taps follow in a padded float4
    float a0 = 0.0f, a1 = 0.0f, a2 = 0.0f, a3 = 0.0f;
    if (exact) {
        const float4 *row = reinterpret_cast<const float4 *>(tab + (size_t)ph * row_stride);
#pragma unroll 4
        for (int q = 0; q < nq; ++q) {
            const float4 c = __ldg(row + q);
            a0 = fmaf(c.x, x[4 * q], a0);
            a1 = fmaf(c.y, x[4 * q + 1], a1);
            a2 = fmaf(c.z, x[4 * q + 2], a2);
            a3 = fmaf(c.w, x[4 * q + 3], a3);
        }
        if (half & 1) {
            const float4 c = __ldg(row + nq);
            a0 = fmaf(c.x, x[4 * nq], a0);
            a1 = fmaf(c.y, x[4 * nq + 1], a1);
        }
    } else {
        const double pos = (double)ph / (double)L * (double)phases;
        const int p = (int)pos;
        const float a = (float)(pos - (double)p);
        const float4 *r0 = reinterpret_cast<const float4 *>(tab + (size_t)p * row_stride), *r1 = r0 + (row_stride >> 2);
#pragma unroll 2
        for (int q = 0; q < nq; ++q) {
            const float4 c0 = __ldg(r0 + q), c1 = __ldg(r1 + q);
            a0 = fmaf(fmaf(a, c1.x - c0.x, c0.x), x[4 * q], a0);
            a1 = fmaf(fmaf(a, c1.y - c0.y, c0.y), x[4 * q + 1], a1);
            a2 = fmaf(fmaf(a, c1.z - c0.z, c0.z), x[4 * q + 2], a2);
            a3 = fmaf(fmaf(a, c1.w - c0.w, c0.w), x[4 * q + 3], a3);
        }
        if (half & 1) {
            const float4 c0 = __ldg(r0 + nq), c1 = __ldg(r1 + nq);
            a0 = fmaf(fmaf(a, c1.x - c0.x, c0.x), x[4 * nq], a0);
            a1 = fmaf(fmaf(a, c1.y - c0.y, c0.y), x[4 * nq + 1], a1);
        }
    }
    out[i] = (a0 + a1) + (a2 + a3);
}

template <typename Idx>
static int launch_sinc(const Source &s, const Design &d, const float *d_tab, float *d_out, long long o_begin,
                       long long o_end, unsigned grid, cudaStream_t stream) {
    const size_t smem = sizeof(float) * (size_t)sinc_smem_floats(d.L, d.M, d.taps);
    if (smem > 48 * 1024)
        FA_CUDA_TRY(cudaFuncSetAttribute(sinc_kernel<Idx>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    FA_CUDA_TRY(fa::launch(sinc_kernel<Idx>, grid, kSincBlock, smem, stream, s, d.L, d.M, d.half, d.phases, d.exact ? 1 : 0,
                           d.row_stride, d_tab, d_out, o_begin, o_end));
    return FA_OK;
}

int launch_convert(const void *d_pcm, long long frames, const AudioFormat &f, const Design &d, const float *d_tab,
                   float *d_out, long long o_begin, long long o_end, cudaStream_t stream) {
    if (o_end <= o_begin) return FA_OK;
    Source s{d_pcm, frames, f.channels, f.format, f.interleaved, 1.0f / (float)f.channels};
    const unsigned grid = (unsigned)((o_end - o_begin + 255) / 256);
    if (f.in_rate == f.out_rate) {
        FA_CUDA_TRY(fa::launch(mixdown_kernel, grid, 256, 0, stream, s, d_out, o_begin, o_end));
    } else if (resolve_algorithm(f) == kAlgoLinear) {
        FA_CUDA_TRY(fa::launch(linear_kernel, grid, 256, 0, stream, s, f.in_rate / f.out_rate, d_out, o_begin, o_end));
    } else {
        return sinc_narrow_index(d.L, d.M) ? launch_sinc<unsigned>(s, d, d_tab, d_out, o_begin, o_end, grid, stream)
                                           : launch_sinc<unsigned long long>(s, d, d_tab, d_out, o_begin, o_end, grid, stream);
    }
    return FA_OK;
}

int convert_host(const void *pcm, long long frames, const AudioFormat &f, float *out, long long n) {
    Design d;
    if (f.in_rate != f.out_rate) {
        const int st = make_design(f.in_rate, f.out_rate, d);
        if (st != FA_OK) return st;
    }
    const size_t bytes = (size_t)frames * f.channels * (f.format == kPcmI16 ? 2 : 4);
    return with_context(0, [&](CallContext &C) -> int {
        HostStaging H(true, C.stream);
        const char *d_pcm;
        const float *d_tab;
        float *d_out;
        int st = H.carve(C.d_buf, [&](HostStaging::Layout &l) {
            d_pcm = l.in(static_cast<const char *>(pcm), bytes, 16);
            d_tab = l.in(d.table.empty() ? nullptr : d.table.data(), d.table.size());
            d_out = l.out(out, (size_t)n);
        });
        if (st != FA_OK) return st;
        st = launch_convert(d_pcm, frames, f, d, d_tab, d_out, 0, n, C.stream);
        if (st != FA_OK) return st;
        FA_CUDA_TRY(H.finish());
        return FA_OK;
    });
}

} // namespace resample
} // namespace fa
