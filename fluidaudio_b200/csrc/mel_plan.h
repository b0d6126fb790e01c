// Host-side plan + launch descriptors of the fused log-mel kernel: the kernels, init, launch and the device entry points
// are in mel_kernels.cu, the host-buffer pipelines in mel_pipeline.cu, the tables the plan uploads in mel_tables.cpp.
#pragma once

#include "fa_common.cuh"
#include "mel_tables.h"
#include "resample_plan.h"
#include "session_table.h"
#include <cuda_runtime.h>
#include <algorithm>
#include <limits>
#include <vector>

namespace fa {
struct CallContext;   // call_context.h

namespace mel {

struct cpx;

// One unit of work = a run of frames of one clip.  A long clip is cut into several units so that H2D copies,
// kernels and D2H copies of successive units overlap; a batch of clips is simply many units in one launch.
struct MelUnit {
    long long audio_off;     // float offset of the clip's sample 0 inside the audio buffer (multiple of 4 for TMA)
    long long n;             // samples in the clip
    long long out_off;       // float offset of the clip's output inside the output buffer
    long long out_stride;    // mel-major layout: row stride (= padded frame count); unused for time-major
    long long frame_begin;   // first frame of this unit
    long long frame_count;   // frames in this unit
    float last;              // lastAudioSample (pre-emphasis state), x[-1]
    int tile_begin;          // first tile index of this unit inside its launch
};

struct MelLaunch {
    const float *audio;
    float *out;
    const MelUnit *units;
    int num_units;
    int total_tiles;
    int hop;
    int pad;            // audio index of buffer position j of frame f is f*hop + j - pad
    float preemph;
    int n_mels;
    float log_floor;
    int log_clamped;
    int ot_stride;      // floats per row of the staged output tile: n_mels + 4 (16-byte aligned rows) or n_mels + 1
    int out_vec4;       // n_mels % 4 == 0 and out + every unit's out_off is 16-byte aligned: copy-out in float4 stores
    int log_normal;     // log_floor is a normal float: the denormal handling of the device log can be skipped
    int layout;         // 0 time-major [T x nMels], 1 mel-major [nMels x stride]
    const void *lane_tab;   // [32] LaneTables<V> of the launch's window placement and precision (mel_core.cuh)
    const float *win_tab;
    const uint8_t *in_tab;
    const float *fb_w;
    const int *fb_lo;
    const int *fb_hi;
    const int *fb_off;
    const int4 *fb_slots;   // mel512_kernel's filterbank schedule: {first bin, quads, weight offset, mel bin or -1} per slot
    int n_slots;
    int fb_nnz, fb_cap;
    int pt_len, pt_cap, raw_cap;
    int use_tma;
    int mid_full;          // window covers buffer positions [64, 448): pass 1 skips the in-window select for slots 1..6
    unsigned inv_n_mels;   // ceil(2^32 / n_mels): idx / n_mels == umulhi(idx, inv) for idx < 2^16 (n_mels > 1; 0 for 1)
    int inline_unit;       // single-unit launch: the descriptor travels in the kernel parameters (unit0), units is not read
    MelUnit unit0;
};

struct MelPlan {
    MelConfig cfg{};
    std::vector<float> window;       // [win]
    std::vector<float> filterbank;   // [n_mels x 257] dense, as the reference exposes it (getFilterbank)
    int fb_nnz = 0, fb_cap = 0;
    int pt_len = 0, pt_cap = 0, raw_cap = 0;
    size_t smem_bytes = 0;
    int num_sms = 0;
    int precision = FA_MEL_PRECISION_F64;   // transform arithmetic: FP64 (one frame per warp) or F32 (float32 frame pairs)
    int pipeline_chunks = 24;        // units a long host-buffer call is cut into (H2D / kernel / D2H overlap)
    bool zero_copy_out = false;      // time-major output in a pinned host buffer: the kernel stores straight into it
                                     // (opt-in: the staged copy is the default)
    // declared before the buffers, so destroyed after them
    Stream streams[3];               // h2d, compute, d2h
    std::vector<Event> events;
    Event timer[2];                  // fa_mel_timer_*: events on the compute stream

    bool generic = false;            // nFFT != 512 or odd hop: mel_generic_kernel (FP64 transform whatever `precision`)
    int generic_warps = 0, generic_prow = 0, generic_log2n = 0;
    DeviceBuffer<> d_generic_tw;     // FP64 twiddles W_n^k, k < n/2

    DeviceBuffer<> d_lane_tab[2][2];   // [window placement][precision]
    DeviceBuffer<float> d_win_tab_mode[2];
    DeviceBuffer<uint8_t> d_in_tab_mode[2];
    DeviceBuffer<float> d_fb_w;
    DeviceBuffer<int> d_fb_lo, d_fb_hi, d_fb_off;
    DeviceBuffer<int4> d_fb_slots;
    int n_slots = 0;

    // buffers grown on demand
    UploadStage<MelUnit> units;                    // unit descriptors of every launch
    DeviceBuffer<> staging;                        // the host-buffer entry points' arrays (HostStaging, fa_common.cuh)
    // AudioConverter stage ahead of the kernel (fa_audio_to_mel): the polyphase table of the last ratio
    resample::Design rs_design;
    double rs_in = 0.0, rs_out = 0.0;
    DeviceBuffer<float> d_rs_tab;

    int init(const MelConfig &c);
    long long frame_count(long long n, int mode, long long expected) const;
    int ensure_events(size_t count);
    // kernel launch over `count` units at d_u (device) whose host mirror is h_u, numbered by number_tiles (the last unit
    // gives the tile total; h_u is also read for the alignment of the audio and of the output rows).
    // inline_unit: a single unit travels in the kernel parameters and d_u is not read.
    int launch(const MelUnit *d_u, const MelUnit *h_u, int count, bool inline_unit, const float *d_audio_base,
               float *d_out_base, int mode, int layout, cudaStream_t stream);

    // mode: FA_MEL_PAD_* / FA_MEL_LEGACY_COMPUTE; layout: FA_MEL_TIME_MAJOR / FA_MEL_MEL_MAJOR
    int compute_device(const float *d_in, long long n, float last, int mode, long long expected, int layout,
                       float *d_out_buf, long long out_len, long long *mel_length, long long *num_frames,
                       cudaStream_t stream);
    // PCM in any AudioFormat (host) -> [device: mixdown + resample to cfg.sample_rate] -> log-mel (host).  Only the raw
    // PCM crosses PCIe on the way in (int16 halves the bytes); *resampled = samples at the model rate.  Mono float32 at
    // the model rate (resample::is_identity) is copied straight into the kernel's input, with no conversion kernel.
    int compute_host(const void *pcm, long long frames, const resample::AudioFormat &f, float last, int mode,
                     long long expected, int layout, float *out, long long out_len, long long *mel_length,
                     long long *num_frames, long long *resampled);
    int ensure_resampler(double in_rate, double out_rate);
    int compute_batch_host(const float *audio, const int64_t *offsets, int count, const float *last, int mode,
                           int layout, float *out, const int64_t *out_offsets, int64_t *mel_lengths,
                           int64_t *num_frames);
    int compute_batch_device(const float *d_in, const int64_t *offsets, int count, const float *last, int mode,
                             int layout, float *d_out_buf, const int64_t *out_offsets, int64_t *mel_lengths,
                             int64_t *num_frames, cudaStream_t stream);
    // One .center launch of exactly T frames of one n-sample clip at d_in, whatever n (an empty clip reads zeros): the
    // torch-style frontends count their frames by their own rules (mel_adapters.cu).  last = 0.
    int launch_clip(const float *d_in, long long n, long long T, int layout, float *d_out_buf, cudaStream_t stream);
    // CUDA-event timing on the stream the mel kernels are launched on (device-resident entry points are asynchronous).
    // timer_stop_ms refuses a timer that was never started.
    int timer_start();
    int timer_stop_ms(float *elapsed_ms);
};

// Numbers a run of units that one launch covers: sets each unit's tile_begin and returns the run's tile total.
int number_tiles(MelUnit *u, int count);

// Shape rules of the entry points (mel_kernels.cu), shared with the host-buffer pipelines (mel_pipeline.cu).
inline long long ceil_to(long long v, long long m) { return ((v + m - 1) / m) * m; }
// bytes of the unit descriptors of a call with `count` units
inline size_t unit_bytes(int count) { return (size_t)std::max(count, 64) * sizeof(MelUnit); }
// Output shape of one clip, reported through mel_length / num_frames: T frames computed, Tp rows returned.  Empty input
// gives T = 0 and one pad row (none in mode FA_MEL_LEGACY_COMPUTE), which the caller zeroes.  Fails when out_len floats
// cannot hold Tp rows.
int clip_shape(const MelPlan &p, long long n, int mode, long long expected, long long out_len, long long &T,
               long long &Tp, long long *mel_length, long long *num_frames);
constexpr long long kUnchecked = std::numeric_limits<long long>::max();   // batch calls take no output lengths

// mel_stream.cu: live streams on one plan, SortformerDiarizer's incremental mel stream (SortformerDiarizer.swift:204-217,
// :417-424, :842-901) for many sessions at once.  Per session, the samples not yet consumed by a frame (the carry, fewer
// than nFFT/2 + win/2 of them) and the pre-emphasis state `last` stay in HBM; the counters stay on the host.  One push
// advances any number of sessions with one ingest launch and one mel launch.
struct MelStreamJob;

// A session's host counters: samples carried in d_carry, real samples received, frames emitted, finished.
struct MelSession {
    long long carry_len, received, emitted;
    bool finished;
};

struct MelStreamSet {
    int capacity = 0;                    // floats per session in d_carry: round_up4(nFFT/2 + win/2)
    SessionTable<MelSession> table;
    DeviceBuffer<float> d_carry;         // [slots x capacity]
    DeviceBuffer<float> d_last;          // [slots] lastAudioSample
    // push staging: descriptors (units, then jobs) and the arena the ingest kernel assembles every emitting session's
    // contiguous input in
    UploadStage<> desc;
    DeviceBuffer<float> d_arena;

    static int check_config(const MelConfig &c);   // pad_to <= 1 and hop <= win, or FA_INVALID_ARGUMENT
    int open(MelPlan &p, int *session);
    int close(int session);
    // rows the next push of `n` samples (finish 0/1) to `session` emits
    long long frames(const MelPlan &p, int session, long long n, bool finish) const;
    // Session sessions[i] receives audio[offsets[i] .. offsets[i+1]); its frames[i] rows start at row sum_{j<i} frames[j]
    // of out.  device: audio and out are HBM and the call is asynchronous on the compute stream; otherwise both are host
    // buffers, the samples travel in one copy, the rows in one copy, and the call returns after one synchronisation.
    int push(MelPlan &p, int count, const int *sessions, const float *audio, const int64_t *offsets, const int *finish,
             bool device, float *out, long long out_len, int64_t *frames);
};

// mel_adapters.cu: device epilogues for the callers directly behind AudioMelSpectrogram (host buffers in and out)
int normalize_per_feature_host(CallContext &C, float *x, long long T, int M, long long valid);
int unified_features(MelPlan &p, const float *window, long long n, long long valid_count, float *out, long long out_len,
                     long long *total_frames, int *valid_frames);
int lseend_features(MelPlan &p, const float *chunk, long long n, float *cmn_mean, long long *cmn_count, float *out,
                    long long out_len, long long *frames);
// the torch-style frontends (CoherePipeline.swift, StyleTTS2MelExtractor.swift, LuxTtsMelExtractor.swift)
int cohere_features(MelPlan &p, const float *audio, long long n, long long fixed_frames, float *out, long long out_len,
                    long long *frames, long long *valid_frames);
int styletts2_features(MelPlan &p, const float *audio, long long n, float *out, long long out_len, long long *frames);
int luxtts_features(MelPlan &p, const float *audio, long long n, float *out, long long out_len, long long *frames);

} // namespace mel
} // namespace fa
