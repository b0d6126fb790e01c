// LS-EEND live feature streams: LSEENDFeatureProvider (Diarizer/LS-EEND/LSEENDPreprocessor.swift:46-384) for many
// sessions at once.  This header holds the arithmetic every push plans with before anything runs: the derived sizes of
// the provider's init (:46-114, LSEENDTypes.swift:53-57) and the queue lengths, mel frames and chunks of one push.  Plain
// C++ (no CUDA), so the CPU test-suite compiles it with g++ (tests/emul/lseend_plan_shim.cpp).  The device state and
// the kernels are in lseend_streams.cu, the C ABI in lseend_abi.cu.
#pragma once

#include "../../../include/fluidaudio_b200.h"
#include "fa_common.cuh"

#include <algorithm>
#include <cstdint>

namespace fa {
namespace lseend {

struct Config {
    int sample_rate, n_mels, hop_length, win_length, context_size, subsampling, chunk_size, conv_delay, precision;
};

// What the provider's init derives from the metadata.
struct Sizes {
    int n_fft;            // next power of two >= win_length (LSEENDTypes.swift:55-57)
    int mel_frames;       // (chunk_size - 1) * subsampling + 2 * context_size + 1: the rows of one model-input chunk
    int chunk_mels;       // subsampling * chunk_size: mel rows one chunk advances the mel queue by
    int mel_context;      // mel_frames - chunk_mels = 2 * context_size + 1 - subsampling; may be negative
    int chunk_samples;    // hop * chunk_mels: samples one audio chunk advances the audio queue by
    int audio_left;       // n_fft / 2: zeros the audio queue starts with
    int audio_context;    // n_fft - hop: left (n_fft / 2) plus right (n_fft / 2 - hop) context of the audio queue
    int flush_samples;    // (context_size + conv_delay * subsampling) * hop + n_fft / 2
    int mask_length;      // conv_delay + chunk_size: the decoder mask, conv_delay zeros then chunk_size ones
    int audio_capacity;   // chunk_samples + audio_context: a session carries fewer audio samples than this
};

// Every size stays below 2^28, so each product the planning forms fits int64 with room to spare.
constexpr long long kMaxSize = 1LL << 28;

// The config's derived sizes, or FA_INVALID_ARGUMENT with error text.  No device: the kernels' own limits (nFFT >= 32,
// n_mels <= 512) are the mel plan's to check when a handle is created.
inline int resolve(const Config &c, Sizes &s) {
    if (c.sample_rate < 1 || c.n_mels < 1 || c.hop_length < 1 || c.win_length < 1 || c.context_size < 0 ||
        c.subsampling < 1 || c.chunk_size < 1 || c.conv_delay < 0 || c.win_length > (1 << 24)) {
        set_error("lseend stream config: sample_rate, n_mels, hop_length, win_length (<= 2^24), subsampling and "
                  "chunk_size must be positive, context_size and conv_delay non-negative");
        return FA_INVALID_ARGUMENT;
    }
    if (c.hop_length > c.win_length) {
        set_error("lseend stream config: hop_length (%d) must not exceed win_length (%d)", c.hop_length, c.win_length);
        return FA_INVALID_ARGUMENT;
    }
    if (c.precision != FA_MEL_PRECISION_F64 && c.precision != FA_MEL_PRECISION_F32) {
        set_error("lseend stream config: precision must be FA_MEL_PRECISION_F64 (0) or FA_MEL_PRECISION_F32 (1)");
        return FA_INVALID_ARGUMENT;
    }
    long long n_fft = 1;
    while (n_fft < c.win_length) n_fft <<= 1;
    const long long chunk_mels = (long long)c.subsampling * c.chunk_size;
    const long long mel_frames = (long long)(c.chunk_size - 1) * c.subsampling + 2LL * c.context_size + 1;
    const long long chunk_samples = (long long)c.hop_length * chunk_mels;
    const long long flush = ((long long)c.context_size + (long long)c.conv_delay * c.subsampling) * c.hop_length + n_fft / 2;
    const long long mask = (long long)c.conv_delay + c.chunk_size;
    if (chunk_mels >= kMaxSize || mel_frames >= kMaxSize || chunk_samples + n_fft >= kMaxSize || flush >= kMaxSize ||
        mask >= kMaxSize || mel_frames * c.n_mels >= kMaxSize) {
        set_error("lseend stream config: derived sizes exceed 2^28 (chunk %lld samples, %lld mel frames)", chunk_samples,
                  mel_frames);
        return FA_INVALID_ARGUMENT;
    }
    s = Sizes{(int)n_fft,
              (int)mel_frames,
              (int)chunk_mels,
              (int)(mel_frames - chunk_mels),
              (int)chunk_samples,
              (int)(n_fft / 2),
              (int)(n_fft - c.hop_length),
              (int)flush,
              (int)mask,
              (int)(chunk_samples + n_fft - c.hop_length)};
    return FA_OK;
}

// The host mirror of one session: the unread lengths of both queues, cmnCount, decoderMaskEnd, and the same four of
// the snapshot when one was taken.
struct Lengths {
    long long audio, mel, cmn_count;
    int mask_end;
};
struct Session {
    Lengths now, snap;
    bool has_snapshot;
};

// A fresh provider (:94-109): nFFT/2 zero samples, context_size zero mel rows, a zero mean, nothing emitted.
inline Lengths fresh(const Config &c, const Sizes &s) { return Lengths{s.audio_left, c.context_size, 0, 0}; }

// One push of n samples (and the silence drain after them when drain is set), then every ready chunk emitted.
struct Step {
    long long zeros;     // drain samples appended after the pushed ones: flushSampleCount plus the chunk-boundary shortfall
    long long unread;    // audio samples in the queue before it is processed: carried + n + zeros
    long long consumed;  // samples popAllChunks drops: audio chunks * chunk_samples
    long long frames;    // mel rows processAudioQueue computes: audio chunks * chunk_mels
    long long chunks;    // model-input chunks emitted
    Lengths next;
};

inline Step plan_push(const Config &c, const Sizes &s, const Lengths &m, long long n, bool drain) {
    Step t{};
    long long u = m.audio + n;
    if (drain) {   // drainRightContextWithSilence (:158-180)
        u += s.flush_samples;
        const long long over = std::max(0LL, u - s.audio_context);
        const long long shortfall = (s.chunk_samples - over % s.chunk_samples) % s.chunk_samples;
        t.zeros = s.flush_samples + shortfall;
        u += shortfall;
    }
    t.unread = u;
    // popAllChunks (:370-376): nothing below one padded chunk, else every whole chunk past the context
    const long long k = u >= s.chunk_samples + s.audio_context ? (u - s.audio_context) / s.chunk_samples : 0;
    t.consumed = k * s.chunk_samples;
    t.frames = k * s.chunk_mels;
    // popNextChunk (:362-367) until the queue holds fewer than mel_frames rows
    const long long rows = m.mel + t.frames;
    t.chunks = rows >= s.mel_frames ? (rows - s.mel_frames) / s.chunk_mels + 1 : 0;
    // emitNextChunk (:193): the mask window advances by chunk_size per chunk, capped at the mask's length
    const long long end = std::min<long long>(m.mask_end + t.chunks * c.chunk_size, s.mask_length);
    t.next = Lengths{u - t.consumed, rows - t.chunks * s.chunk_mels, m.cmn_count + t.frames, (int)end};
    return t;
}

// The decoder-mask window of the chunk that leaves decoderMaskEnd at `end`, and its warm-up count (:193-198).
FA_HD float mask_value(int end, int chunk_size, int conv_delay, int t) {
    return end - chunk_size + t >= conv_delay ? 1.0f : 0.0f;
}
FA_HD int warmup_frames(int end, int chunk_size, int mask_length) {
    return mask_length - end < chunk_size ? mask_length - end : chunk_size;
}

#if defined(__CUDACC__)
// processAudioQueue's scaling and cumulative mean (:259-276) down mel column m of T time-major rows x[t * M + m], in
// place, from the running mean `mean` after count0 frames; returns the new mean.  Per frame: alpha = 1 / Float(count),
// vDSP_vintb (mean + alpha * (v - mean)) and vDSP_vsub, every operation rounded to float32.  fa_mel_lseend_features and
// the live streams both run it, so their features agree bit for bit.
__device__ __forceinline__ float scale_cmn_column(float *x, long long T, int M, int m, float mean, long long count0,
                                                  float scale) {
    for (long long t = 0; t < T; ++t) {
        const float alpha = __fdiv_rn(1.0f, (float)(count0 + t + 1));
        const float v = __fmul_rn(x[t * M + m], scale);
        mean = __fadd_rn(mean, __fmul_rn(alpha, __fsub_rn(v, mean)));
        x[t * M + m] = __fsub_rn(v, mean);
    }
    return mean;
}
#endif

} // namespace lseend
} // namespace fa
