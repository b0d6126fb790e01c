// Sample-rate / format / channel conversion to mono float32 ahead of the log-mel kernel (SURVEY §8a row R1).
//
// Reference: Sources/FluidAudio/Shared/AudioConverter.swift
//   :60-71   resample(_:from:)          identity when the rate already matches, else AVAudioConverter
//   :299-370 convertBuffer              <= 2 channels: AVAudioConverter (Mastering algorithm, max quality :372-375);
//                                       > 2 channels: linearResample
//   :388-442 linearResample             mean mixdown, src = i * ratio, two-tap float32 lerp, outCount = Int(n / ratio)
//
// AVAudioConverter is closed Apple code: its filter cannot be restated, only replaced.  The replacement here is a
// DOCUMENTED Kaiser-windowed-sinc polyphase resampler (design below), "parity unpinned" for sample values against
// Apple's; the reference's own tests pin only the output LENGTH within 1 % (AudioConverterTests.swift:129-176), which
// holds by construction (outCount = floor(n * out / in), the same rule linearResample uses).  The > 2-channel linear
// path IS in-repo arithmetic and is reproduced bit for bit (float32 operations individually rounded, the source
// position in double).
//
// Filter design (oracle/oracle.py::sinc_design / sinc_resample restate it in float64):
//   ratio out/in = L/M in lowest terms: on the 1 Hz grid when both rates are whole, else on the 1/1000 Hz grid,
//   fc = min(1, L/M) * kRolloff (1 = input Nyquist), H = ceil(kZeros / min(1, L/M)) input samples either side, taps = 2H,
//   g(t) = fc * sinc(fc * t) * I0(beta * sqrt(1 - (t/H)^2)) / I0(beta),  |t| < H,
//   row p (phase p/P of an input sample) holds g(k - p/P), k = -H+1 .. H, normalised to unit DC gain;
//   P = L when L <= kMaxExactPhases (every output lands exactly on a row), otherwise P = kInterpPhases rows (+ 1 stored)
//   blended linearly: pos = ph / L * P in double, p = (int)pos, a = (float)(pos - p), taps c_p + a (c_{p+1} - c_p).
//   y[i] = sum_k row[p(i)][k] * x[n0(i) - H + 1 + k],   n0 = floor(i * M / L),  phase ph = (i * M) mod L.
//   Samples outside [0, n) are zero (the converter's start-up / drain behaviour, without added latency: output i is
//   centred on input time i * M / L).
// Guarantees of make_design / sinc_kernel:
//   * FA_UNSUPPORTED (with a message) for a rate off the 1/1000 Hz grid, a reduced term L or M >= 2^32, and a window
//     that does not fit shared memory: (255 M / L + 2H + 8) floats > 200 KB, i.e. decimation by more than 168.
//   * phases exact for every accepted (L, M) and any output index (resample_core.cuh; 32-bit offsets when
//     255 M + L < 2^32, 64-bit otherwise).
//   * output i depends on its 2H-tap window only: a NaN / Inf input makes exactly the outputs whose window holds it
//     non-finite (rows are padded to whole float4s; the padding is never multiplied).
//   * error bar against the float64 evaluation, per output: (taps/4 + 6) * 2^-24 * sum_k A_k |x_k|, A_k = |g_k|, or
//     |g_{p,k}| + |g_{p+1,k}| where two rows are blended (four FMA chains, two adds, float32 taps, the blend).
#pragma once

#include "../../include/fluidaudio_b200.h"
#include "fa_common.cuh"
#include <cuda_runtime.h>
#include <vector>

namespace fa {
namespace resample {

constexpr double kRolloff = 0.94;       // pass band edge as a fraction of the lower Nyquist frequency
constexpr int kZeros = 24;              // zero crossings of the sinc either side (at the lower rate)
constexpr double kBeta = 12.0;          // Kaiser beta: ~ -118 dB stop band
constexpr int kMaxExactPhases = 2048;
constexpr int kInterpPhases = 1024;

enum : int { kPcmF32 = 0, kPcmI16 = 1 };
enum : int { kAlgoAuto = 0, kAlgoSinc = 1, kAlgoLinear = 2 };

struct AudioFormat {
    double in_rate;
    double out_rate;
    int32_t channels;
    int32_t format;        // kPcmF32 / kPcmI16
    int32_t interleaved;   // 1: [frames x channels], 0: planar [channels x frames]
    int32_t algorithm;     // kAlgoAuto: <= 2 channels sinc, > 2 channels linear (AudioConverter.swift:303-305)
};

struct Design {
    long long L = 1, M = 1;   // out/in = L/M
    int half = 0;             // H
    int taps = 0;             // 2H
    int row_stride = 0;       // floats per table row: taps rounded up to a multiple of four (zero padded)
    int phases = 1;           // P (rows; P + 1 rows stored when interpolating)
    bool exact = true;        // every output lands on a row
    double fc = 1.0;
    std::vector<float> table; // [(exact ? P : P + 1) x row_stride]
};

// out/in reduced to L/M on the 1 Hz grid when both rates are whole, otherwise on the 1/1000 Hz grid (false: off grid)
bool rational_ratio(double in_rate, double out_rate, long long &L, long long &M);
int make_design(double in_rate, double out_rate, Design &d);
long long output_count(long long frames, double in_rate, double out_rate);   // Int(Double(n) / (in / out))
bool is_identity(const AudioFormat &f);   // mono float32 at the output rate: nothing to do
int resolve_algorithm(const AudioFormat &f);

// Device-side conversion of frames [0, frames) of `pcm` (device pointer, layout per `f`) into out[o_begin, o_end).
// tab: device copy of Design::table (sinc only).  `frames_avail`: input frames already resident (<= frames): outputs
// whose filter window reaches beyond it must not be requested yet (see outputs_ready).
int launch_convert(const void *d_pcm, long long frames, const AudioFormat &f, const Design &d, const float *d_tab,
                   float *d_out, long long o_begin, long long o_end, cudaStream_t stream);
// number of leading outputs computable when only the first `frames_avail` input frames are resident
long long outputs_ready(const AudioFormat &f, const Design &d, long long frames, long long frames_avail,
                        long long out_total);
// The converter stage on host buffers, on a leased call context: frames [0, frames) of `pcm` (layout per `f`) into the
// n = output_count(frames, f.in_rate, f.out_rate) > 0 samples of `out`.  Returns once `out` holds them.
int convert_host(const void *pcm, long long frames, const AudioFormat &f, float *out, long long n);

// The C ABI's check of a caller's fa_audio_format, with error text when it fails, and its conversion (resample_abi.cu):
// shared by fa_audio_resample and fa_audio_to_mel.
bool audio_format_ok(const fa_audio_format *f);
AudioFormat to_format(const fa_audio_format *f);

} // namespace resample
} // namespace fa
