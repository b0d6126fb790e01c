// The thin per-caller adapters that sit directly behind AudioMelSpectrogram in the reference (SURVEY.md 8f rank 3),
// as device epilogues of the mel kernel: the log-mel never leaves HBM between the STFT and the adapter.
//
//   unified:  UnifiedMelExtractor.features(window:validCount:)   ASR/Parakeet/Unified/UnifiedMelExtractor.swift:52-113
//             center-padded log-mel with a fixed frame count, NeMo per-feature (per mel bin) mean / unbiased-std
//             normalisation over the valid frames, pad frames zeroed, packed [1, nMels, T].
//   lseend:   LSEENDPreprocessor.processAudioQueue            Diarizer/LS-EEND/LSEENDPreprocessor.swift:249-283
//             .prePadded log-mel (preemph 0, periodic Hann, clamped floor) * 1/ln(10), cumulative mean normalisation
//             with state (mean per mel, frame count) carried from call to call.
//
// Both normalisations are sequential in time by definition (the reference's loops) and independent across mel bins:
// one thread per mel bin walks the frames in order with individually rounded float32 operations, so the result is the
// reference's arithmetic exactly; loads are coalesced across bins.  Sizes are tiny (<= 512 bins x a few thousand
// frames), the point is fusion with the producer, not throughput.
#include "call_context.h"
#include "fa_common.cuh"
#include "lseend/lseend_plan.h"
#include "mel_plan.h"

#include <algorithm>
#include <cmath>
#include <cuda_runtime.h>

namespace fa {
namespace mel {

constexpr int kBinsPerCta = 128;
constexpr int kTile = 32;

// x: time-major [T x M]; out: mel-major [M x T].  valid >= 1.
__global__ void __launch_bounds__(kBinsPerCta) per_feature_norm_kernel(const float *__restrict__ x, long long T, int M,
                                                                       long long valid, float *__restrict__ out) {
    __shared__ float tile[kBinsPerCta][kTile + 1];
    const int m0 = blockIdx.x * kBinsPerCta, m = m0 + threadIdx.x;
    const bool live = m < M;
    float mean = 0.0f, sd = 1.0f;
    if (live) {
        for (long long t = 0; t < valid; ++t) mean = __fadd_rn(mean, x[t * M + m]);
        mean = __fdiv_rn(mean, (float)valid);
        float var_sum = 0.0f;
        for (long long t = 0; t < valid; ++t) {
            const float d = __fsub_rn(x[t * M + m], mean);
            var_sum = __fadd_rn(var_sum, __fmul_rn(d, d));
        }
        const float denom = (float)(valid > 1 ? valid - 1 : 1);
        sd = __fadd_rn(__fsqrt_rn(__fdiv_rn(var_sum, denom)), 1e-5f);
    }
    const int rows = min(kBinsPerCta, M - m0);
    for (long long t0 = 0; t0 < T; t0 += kTile) {
        const int nt = (int)min((long long)kTile, T - t0);
        if (live)
            for (int i = 0; i < nt; ++i) {
                const long long t = t0 + i;
                tile[threadIdx.x][i] = t < valid ? __fdiv_rn(__fsub_rn(x[t * M + m], mean), sd) : 0.0f;
            }
        __syncthreads();
        const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
        for (int r = warp; r < rows; r += kBinsPerCta / 32)
            if (lane < nt) out[(long long)(m0 + r) * T + t0 + lane] = tile[r][lane];
        __syncthreads();
    }
}

// Same statistics, time-major in place (the standalone UnifiedMelExtractor.normalizePerFeature entry point of the C ABI).
__global__ void per_feature_norm_inplace_kernel(float *x, long long T, int M, long long valid) {
    const int m = blockIdx.x * blockDim.x + threadIdx.x;
    if (m >= M) return;
    float mean = 0.0f;
    for (long long t = 0; t < valid; ++t) mean = __fadd_rn(mean, x[t * M + m]);
    mean = __fdiv_rn(mean, (float)valid);
    float var_sum = 0.0f;
    for (long long t = 0; t < valid; ++t) {
        const float d = __fsub_rn(x[t * M + m], mean);
        var_sum = __fadd_rn(var_sum, __fmul_rn(d, d));
    }
    const float denom = (float)(valid > 1 ? valid - 1 : 1);
    const float sd = __fadd_rn(__fsqrt_rn(__fdiv_rn(var_sum, denom)), 1e-5f);
    for (long long t = 0; t < T; ++t) x[t * M + m] = t < valid ? __fdiv_rn(__fsub_rn(x[t * M + m], mean), sd) : 0.0f;
}

// host buffer in, host buffer out (x: [T x M] time-major, normalised in place), staged in the context's d_buf; valid >= 1
int normalize_per_feature_host(CallContext &C, float *x, long long T, int M, long long valid) {
    HostStaging H(true, C.stream);
    float *d;
    const int st = H.carve(C.d_buf, [&](HostStaging::Layout &l) { d = l.inout(x, (size_t)T * M); });
    if (st != FA_OK) return st;
    FA_CUDA_TRY(fa::launch(per_feature_norm_inplace_kernel, (M + kBinsPerCta - 1) / kBinsPerCta, kBinsPerCta, 0, C.stream, d,
                           T, M, valid));
    FA_CUDA_TRY(H.finish());
    return FA_OK;
}

// x: time-major [T x M], in place; state: mean[M] (in/out), count (in: frames seen before this call)
__global__ void lseend_scale_cmn_kernel(float *x, long long T, int M, float *mean_io, long long count0, float scale) {
    const int m = blockIdx.x * blockDim.x + threadIdx.x;
    if (m >= M) return;
    mean_io[m] = lseend::scale_cmn_column(x, T, M, m, mean_io[m], count0, scale);
}

// Both adapters return exactly T rows and size their staging for T; a handle with pad_to > 1 would have the mel kernel
// write ceil_to(T, pad_to) rows.  The reference builds both extractors with padTo 0, so such a handle is refused up front,
// before any copy or launch and with the caller's state untouched (as MelStreamSet::check_config does for streams).
static int check_adapter_config(const MelPlan &p, const char *what) {
    if (!p.cfg.neutral()) {   // both restate NeMo-flavoured AudioMelSpectrogram callers
        fa::set_error("%s: needs an AudioMelSpectrogram handle, not one with fa_mel_ex_config fields set", what);
        return FA_INVALID_ARGUMENT;
    }
    if (p.cfg.pad_to > 1) {
        fa::set_error("%s: pad_to must be 0 or 1 (the features hold exactly their frames), got %d", what, p.cfg.pad_to);
        return FA_INVALID_ARGUMENT;
    }
    return FA_OK;
}

int unified_features(MelPlan &p, const float *window, long long n, long long valid_count, float *out, long long out_len,
                     long long *total_frames, int *valid_frames) {
    int st = check_adapter_config(p, "unified mel features");
    if (st != FA_OK) return st;
    const int M = p.cfg.n_mels, hop = p.cfg.hop_length;
    const long long T = n / hop + 1;                                   // UnifiedMelExtractor.swift:30
    const long long valid = std::min<long long>(valid_count / hop, T); // :71
    if (total_frames) *total_frames = T;
    if (valid_frames) *valid_frames = (int)valid;
    if (out_len < T * M) {
        fa::set_error("unified mel features need %lld floats, buffer has %lld", T * M, out_len);
        return FA_OUTPUT_TOO_SMALL;
    }
    cudaStream_t s = p.streams[1];
    HostStaging H(true, s);
    const float *d_audio;
    float *d_flat, *d_pack;
    st = H.carve(p.staging, [&](HostStaging::Layout &l) {
        d_audio = l.in(window, (size_t)n, 16);
        d_flat = l.take<float>((size_t)(T * M));
        d_pack = l.out(out, (size_t)(T * M));
    });
    if (st != FA_OK) return st;
    long long ml = 0, nf = 0;
    st = p.compute_device(d_audio, n, 0.0f, FA_MEL_PAD_CENTER, T, FA_MEL_TIME_MAJOR, d_flat, T * M, &ml, &nf, s);
    if (st != FA_OK) return st;
    if (valid <= 0) {
        FA_CUDA_TRY(cudaMemsetAsync(d_pack, 0, sizeof(float) * T * M, s));
    } else {
        FA_CUDA_TRY(fa::launch(per_feature_norm_kernel, (M + kBinsPerCta - 1) / kBinsPerCta, kBinsPerCta, 0, s, d_flat, T, M,
                               valid, d_pack));
    }
    FA_CUDA_TRY(H.finish());
    return FA_OK;
}

int lseend_features(MelPlan &p, const float *chunk, long long n, float *cmn_mean, long long *cmn_count, float *out,
                    long long out_len, long long *frames) {
    int st = check_adapter_config(p, "LS-EEND features");
    if (st != FA_OK) return st;
    const int M = p.cfg.n_mels;
    const long long T = p.frame_count(n, FA_MEL_PAD_PREPADDED, -1);
    if (frames) *frames = T;
    if (T <= 0) return FA_OK;
    if (out_len < T * M) {
        fa::set_error("LS-EEND features need %lld floats, buffer has %lld", T * M, out_len);
        return FA_OUTPUT_TOO_SMALL;
    }
    cudaStream_t s = p.streams[1];
    HostStaging H(true, s);
    const float *d_audio;
    float *d_flat, *d_mean;
    st = H.carve(p.staging, [&](HostStaging::Layout &l) {
        d_audio = l.in(chunk, (size_t)n, 16);
        d_flat = l.out(out, (size_t)(T * M));
        d_mean = l.inout(cmn_mean, (size_t)M);
    });
    if (st != FA_OK) return st;
    long long ml = 0, nf = 0;
    st = p.compute_device(d_audio, n, 0.0f, FA_MEL_PAD_PREPADDED, -1, FA_MEL_TIME_MAJOR, d_flat, T * M, &ml, &nf, s);
    if (st != FA_OK) return st;
    const float scale = 1.0f / logf(10.0f);   // LSEENDPreprocessor.swift:36, Float arithmetic
    FA_CUDA_TRY(fa::launch(lseend_scale_cmn_kernel, (M + 127) / 128, 128, 0, s, d_flat, T, M, d_mean, *cmn_count, scale));
    FA_CUDA_TRY(H.finish());
    *cmn_count += T;
    return FA_OK;
}

// ------------------------------------------------------------------------------------------------ torch-style frontends
// CohereMelSpectrogram.compute's CMVN and padOrTruncate (CoherePipeline.swift:220-263).  x: the log-mel, time-major
// [T x M] with T > valid; out: mel-major [M x W].  When valid > 1 every mel bin is normalised with the mean and the
// unbiased std (a non-finite std counts as 0) of ALL its valid frames, even those past W: padOrTruncate runs after
// compute.  Frames >= valid are zero, and so are the pad columns up to W.
__global__ void __launch_bounds__(kBinsPerCta) cohere_cmvn_kernel(const float *__restrict__ x, int M, long long valid,
                                                                  long long W, float eps, float *__restrict__ out) {
    __shared__ float tile[kBinsPerCta][kTile + 1];
    const int m0 = blockIdx.x * kBinsPerCta, m = m0 + threadIdx.x;
    const bool live = m < M, cmvn = valid > 1;
    float mean = 0.0f, denom = 1.0f;
    if (live && cmvn) {
        for (long long t = 0; t < valid; ++t) mean = __fadd_rn(mean, x[t * M + m]);
        mean = __fdiv_rn(mean, (float)valid);
        float ssq = 0.0f;
        for (long long t = 0; t < valid; ++t) {
            const float d = __fsub_rn(x[t * M + m], mean);
            ssq = __fadd_rn(ssq, __fmul_rn(d, d));
        }
        float sd = __fsqrt_rn(__fdiv_rn(ssq, (float)(valid - 1)));
        if (!isfinite(sd)) sd = 0.0f;
        denom = __fadd_rn(sd, eps);
    }
    const long long keep = valid < W ? valid : W;
    const int rows = min(kBinsPerCta, M - m0);
    for (long long t0 = 0; t0 < W; t0 += kTile) {
        const int nt = (int)min((long long)kTile, W - t0);
        if (live)
            for (int i = 0; i < nt; ++i) {
                const long long t = t0 + i;
                float v = 0.0f;
                if (t < keep) v = cmvn ? __fdiv_rn(__fsub_rn(x[t * M + m], mean), denom) : x[t * M + m];
                tile[threadIdx.x][i] = v;
            }
        __syncthreads();
        const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
        for (int r = warp; r < rows; r += kBinsPerCta / 32)
            if (lane < nt) out[(long long)(m0 + r) * W + t0 + lane] = tile[r][lane];
        __syncthreads();
    }
}

// Does the handle restate the class?  Filterbank kind, edge, spectrum and log mode, and exactly T rows (pad_to <= 1).
static int check_class(const MelPlan &p, const char *what, int fb_kind, int edge, float power, int log_mode) {
    const MelConfig &c = p.cfg;
    const bool any_power = power < 0.0f;   // CohereMelSpectrogram.Config.magPower is a parameter
    if (c.fb_kind != fb_kind || c.center_edge != edge || (!any_power && c.spectrum_power != power) ||
        c.log_floor_mode != log_mode || c.pad_to > 1 || (fb_kind == FA_MEL_FB_COHERE && c.affine())) {
        fa::set_error("%s: the handle is not configured as its reference class (see its fa_mel_preset_*)", what);
        return FA_INVALID_ARGUMENT;
    }
    return FA_OK;
}

static int check_out(const char *what, long long need, long long out_len) {
    if (out_len < need) {
        fa::set_error("%s need %lld floats, buffer has %lld", what, need, out_len);
        return FA_OUTPUT_TOO_SMALL;
    }
    return FA_OK;
}

int cohere_features(MelPlan &p, const float *audio, long long n, long long fixed_frames, float *out, long long out_len,
                    long long *frames, long long *valid_frames) {
    const char *what = "Cohere mel features";
    int st = check_class(p, what, FA_MEL_FB_COHERE, FA_MEL_EDGE_ZERO, -1.0f, 0);
    if (st != FA_OK) return st;
    const int M = p.cfg.n_mels, hop = p.cfg.hop_length;
    const long long T = 1 + n / hop, valid = n / hop;   // padded.count = n + nFFT: 1 + n / hop frames (:146), :120
    const long long W = fixed_frames < 0 ? T : fixed_frames;
    if (frames) *frames = W;
    if (valid_frames) *valid_frames = std::min(valid, W);
    st = check_out(what, W * M, out_len);
    if (st != FA_OK) return st;
    cudaStream_t s = p.streams[1];
    HostStaging H(true, s);
    const float *d_audio;
    float *d_flat, *d_pack;
    st = H.carve(p.staging, [&](HostStaging::Layout &l) {
        d_audio = l.in(audio, (size_t)n, 16);
        d_flat = l.take<float>((size_t)(T * M));
        d_pack = l.out(out, (size_t)(W * M));
    });
    if (st != FA_OK) return st;
    st = p.launch_clip(d_audio, n, T, FA_MEL_TIME_MAJOR, d_flat, s);
    if (st != FA_OK) return st;
    FA_CUDA_TRY(fa::launch(cohere_cmvn_kernel, (M + kBinsPerCta - 1) / kBinsPerCta, kBinsPerCta, 0, s, d_flat, M, valid, W,
                           1.0e-5f, d_pack));   // Config.cmvnEpsilon
    FA_CUDA_TRY(H.finish());
    return FA_OK;
}

// host clip in, one launch of T frames in `layout`, rows out
static int run_clip(MelPlan &p, const float *audio, long long n, long long T, int layout, float *out) {
    cudaStream_t s = p.streams[1];
    HostStaging H(true, s);
    const float *d_audio;
    float *d_out;
    int st = H.carve(p.staging, [&](HostStaging::Layout &l) {
        d_audio = l.in(audio, (size_t)n, 16);
        d_out = l.out(out, (size_t)(T * p.cfg.n_mels));
    });
    if (st != FA_OK) return st;
    st = p.launch_clip(d_audio, n, T, layout, d_out, s);
    if (st != FA_OK) return st;
    FA_CUDA_TRY(H.finish());
    return FA_OK;
}

int styletts2_features(MelPlan &p, const float *audio, long long n, float *out, long long out_len, long long *frames) {
    const char *what = "StyleTTS2 mel features";
    int st = check_class(p, what, FA_MEL_FB_STYLETTS2, FA_MEL_EDGE_REFLECT, 2.0f, 0);
    if (st != FA_OK) return st;
    const long long T = 1 + n / p.cfg.hop_length;   // reflectPad keeps n + nFFT samples, an empty clip nFFT zeros (:78-87)
    if (frames) *frames = T;
    st = check_out(what, T * p.cfg.n_mels, out_len);
    return st != FA_OK ? st : run_clip(p, audio, n, T, FA_MEL_MEL_MAJOR, out);
}

int luxtts_features(MelPlan &p, const float *audio, long long n, float *out, long long out_len, long long *frames) {
    const char *what = "LuxTTS mel features";
    int st = check_class(p, what, FA_MEL_FB_LUXTTS, FA_MEL_EDGE_REFLECT, 1.0f, 1);
    if (st != FA_OK) return st;
    // lhotse's count (:44-47).  It never exceeds the STFT's 1 + n / hop (:67), so the reference's replicate-last-frame
    // branch (:126-130) is never taken and the frames are the first T STFT frames.
    const long long hop = p.cfg.hop_length, T = n > 0 ? (n + hop / 2) / hop : 0;
    if (frames) *frames = T;
    if (T == 0) return FA_OK;
    st = check_out(what, T * p.cfg.n_mels, out_len);
    return st != FA_OK ? st : run_clip(p, audio, n, T, FA_MEL_TIME_MAJOR, out);
}

} // namespace mel
} // namespace fa
