// LuxTTS synthesis on the GPU (luxtts.h, luxtts_core.cuh).
//
// Each live request owns one slot in HBM: its float32 state x in the FmDecoder's [1024 x 100] layout (zero past
// features_length x 100) and a meta row of its geometry.  The host mirrors the plan and the step, which is all a call
// needs to check before anything runs.  Kernels (requests on blockIdx.x, element tiles on blockIdx.y):
//   luxtts_rms_kernel          one CTA per request: the mean square of the capped prompt in a fixed float64 tree
//   luxtts_gain_kernel         the capped prompts, gained when boosted, packed into scratch for the mel batch
//   (the mel batch)            MelPlan::compute_batch_device on the handle's LuxTTS plan, .center, time-major
//   luxtts_epilogue_kernel     speech_condition, padding_mask, the meta row and the noise x0 into the slot
//   luxtts_text_kernel         text_condition through tokensIndex
//   luxtts_inputs_kernel       x and t for the FmDecoder
//   luxtts_advance_kernel      one anchor-Euler update
//   luxtts_vocoder_kernel      the vocoder's [100 x bucket] mel, a 32 x 32 shared-memory tile transpose
//   luxtts_finish_kernel       truncate, clip and rescale the vocoder's audio into the packed output
#include "luxtts.h"

#include <algorithm>
#include <cmath>
#include <cstring>
#include <cuda_runtime.h>
#include <vector>

namespace fa {
namespace luxtts {

namespace {

constexpr int kThreads = 256;
constexpr int kSlotTiles = kSlotFloats / kThreads;   // 400 CTAs of 256 elements cover a slot
constexpr float kFeatScale = 0.1f, kTargetRms = 0.1f;

struct BeginJob {
    long long src, n;       // the prompt's offset in the call's audio and its capped sample count
    long long gained, mel;  // its offsets in the gained-prompt and mel scratch
    uint64_t s0;            // the noise state before the first draw
    float gain, rms;
    int boosted, slot, prompt_frames, features, gen, tokens;
};

struct StepJob {
    int slot, step;
};

struct FinishJob {
    long long out, len;   // the request's first packed sample and its sample count
    int slot, pad;
};

__device__ __forceinline__ const int *meta_of(const int *meta, int slot) { return meta + (size_t)slot * kMetaFields; }

__global__ void __launch_bounds__(kRmsLanes)
    luxtts_rms_kernel(const BeginJob *__restrict__ jobs, const float *__restrict__ audio, float *__restrict__ rms) {
    __shared__ double part[kRmsLanes];
    const BeginJob J = jobs[blockIdx.x];
    part[threadIdx.x] = rms_lane(audio + J.src, J.n, threadIdx.x);
    __syncthreads();
    for (int s = kRmsLanes / 2; s > 0; s >>= 1) {
        if ((int)threadIdx.x < s) part[threadIdx.x] = dadd(part[threadIdx.x], part[threadIdx.x + s]);
        __syncthreads();
    }
    if (threadIdx.x == 0) rms[blockIdx.x] = J.n > 0 ? rms_of(part[0], J.n) : 0.0f;
}

__global__ void __launch_bounds__(kThreads)
    luxtts_gain_kernel(const BeginJob *__restrict__ jobs, const float *__restrict__ audio, float *__restrict__ gained) {
    const BeginJob J = jobs[blockIdx.x];
    const long long k = (long long)blockIdx.y * kThreads + threadIdx.x;
    if (k >= J.n) return;
    const float v = audio[J.src + k];
    gained[J.gained + k] = J.boosted ? __fmul_rn(v, J.gain) : v;
}

__global__ void __launch_bounds__(kThreads)
    luxtts_epilogue_kernel(const BeginJob *__restrict__ jobs, const float *__restrict__ mel, float *__restrict__ x,
                           int *__restrict__ meta, float *__restrict__ speech, float *__restrict__ mask) {
    const int i = blockIdx.x;
    const BeginJob J = jobs[i];
    const int e = blockIdx.y * kThreads + threadIdx.x, f = e / kFeat;
    speech[(size_t)i * kSlotFloats + e] = f < J.prompt_frames ? __fmul_rn(mel[J.mel + e], kFeatScale) : 0.0f;
    x[(size_t)J.slot * kSlotFloats + e] = f < J.features ? gaussian_at(J.s0, (uint64_t)e) : 0.0f;
    if (e % kFeat == 0) mask[(size_t)i * kMaxFrames + f] = f >= J.features ? 1.0f : 0.0f;
    if (e < kMetaFields) {
        meta[(size_t)J.slot * kMetaFields + e] = e == kPromptFrames ? J.prompt_frames : e == kFeatures ? J.features
                                               : e == kGen ? J.gen : e == kTokens ? J.tokens : e == kBoosted ? J.boosted
                                               : e == kRmsBits ? __float_as_int(J.rms) : 0;
    }
}

__global__ void __launch_bounds__(kThreads)
    luxtts_text_kernel(const StepJob *__restrict__ jobs, const int *__restrict__ meta, const float *__restrict__ embeds,
                       long long row_stride, long long request_stride, float *__restrict__ out) {
    const int i = blockIdx.x;
    const int *M = meta_of(meta, jobs[i].slot);
    const int e = blockIdx.y * kThreads + threadIdx.x, f = e / kFeat, d = e - f * kFeat;
    const int L = M[kFeatures], S = M[kTokens];
    float v = 0.0f;
    if (f < L) v = embeds[(size_t)i * request_stride + (size_t)token_index(f, S, L / S) * row_stride + d];
    out[(size_t)i * kSlotFloats + e] = v;
}

__global__ void __launch_bounds__(kThreads)
    luxtts_inputs_kernel(const StepJob *__restrict__ jobs, const float *__restrict__ x, float *__restrict__ out,
                         float *__restrict__ t) {
    const int i = blockIdx.x;
    const StepJob J = jobs[i];
    const int k = blockIdx.y * kThreads + threadIdx.x;   // float4 index
    reinterpret_cast<float4 *>(out + (size_t)i * kSlotFloats)[k] =
        reinterpret_cast<const float4 *>(x + (size_t)J.slot * kSlotFloats)[k];
    if (k == 0) t[i] = (float)time_step(J.step);
}

__global__ void __launch_bounds__(kThreads)
    luxtts_advance_kernel(const StepJob *__restrict__ jobs, const int *__restrict__ meta, const float *__restrict__ v,
                          long long row_stride, long long request_stride, float *__restrict__ x) {
    const int i = blockIdx.x;
    const StepJob J = jobs[i];
    const int e = blockIdx.y * kThreads + threadIdx.x, f = e / kFeat, d = e - f * kFeat;
    if (f >= meta_of(meta, J.slot)[kFeatures]) return;
    float *X = x + (size_t)J.slot * kSlotFloats + e;
    const float vv = v[(size_t)i * request_stride + (size_t)f * row_stride + d];
    *X = anchor_euler(*X, vv, (float)time_step(J.step), (float)time_step(J.step + 1), J.step == kSteps - 1);
}

constexpr int kTile = 32, kTileRows = 8;

__global__ void __launch_bounds__(kTile * kTileRows)
    luxtts_vocoder_kernel(const StepJob *__restrict__ jobs, const int *__restrict__ meta, const float *__restrict__ x,
                          int bucket, float inv_scale, float log_floor, float *__restrict__ out) {
    __shared__ float tile[kTile][kTile + 1];
    const int i = blockIdx.x;
    const int *M = meta_of(meta, jobs[i].slot);
    const int P = M[kPromptFrames], G = M[kGen];
    const float *X = x + (size_t)jobs[i].slot * kSlotFloats;
    const int f0 = blockIdx.y * kTile, m0 = blockIdx.z * kTile;
    for (int j = threadIdx.y; j < kTile; j += kTileRows) {   // frame f0 + j, mel m0 + threadIdx.x: coalesced in m
        const int f = f0 + j, m = m0 + threadIdx.x;
        tile[j][threadIdx.x] = f < G && m < kFeat ? __fmul_rn(X[(size_t)(P + f) * kFeat + m], inv_scale) : log_floor;
    }
    __syncthreads();
    for (int j = threadIdx.y; j < kTile; j += kTileRows) {   // mel m0 + j, frame f0 + threadIdx.x: coalesced in f
        const int m = m0 + j, f = f0 + threadIdx.x;
        if (m < kFeat && f < bucket) out[((size_t)i * kFeat + m) * bucket + f] = tile[threadIdx.x][j];
    }
}

__global__ void __launch_bounds__(kThreads)
    luxtts_finish_kernel(const FinishJob *__restrict__ jobs, const int *__restrict__ meta, const float *__restrict__ audio,
                         long long row_stride, float *__restrict__ out) {
    const int i = blockIdx.x;
    const FinishJob J = jobs[i];
    const long long k = (long long)blockIdx.y * kThreads + threadIdx.x;
    if (k >= J.len) return;
    const int *M = meta_of(meta, J.slot);
    float s = clip_unit(audio[(size_t)i * row_stride + k]);
    if (M[kBoosted]) s = __fmul_rn(s, __fdiv_rn(__int_as_float(M[kRmsBits]), kTargetRms));
    out[J.out + k] = s;
}

unsigned tiles(long long n, long long per) { return (unsigned)std::max(1LL, (n + per - 1) / per); }

} // namespace

// ------------------------------------------------------------------------------------------------ requests
int RequestSet::init() {
    int st = stream.create();
    if (st != FA_OK) return st;
    fa_mel_ex_config c;
    fa_mel_preset_luxtts(&c);
    mel::MelConfig m{c.base.sample_rate, c.base.n_mels,  c.base.n_fft,          c.base.hop_length,
                     c.base.win_length,  c.base.preemph, c.base.pad_to,         c.base.log_floor,
                     c.base.log_floor_mode, c.base.window_periodic};
    m.fb_kind = c.filterbank;
    m.filter_sample_rate = c.filter_sample_rate;
    m.f_min = c.f_min;
    m.f_max = c.f_max;
    m.center_edge = c.center_edge;
    m.spectrum_power = c.spectrum_power;
    m.log_mean = c.log_mean;
    m.log_std = c.log_std;
    return mel.init(m);
}

int RequestSet::check(int count, const int *ids, const char *where, int min_step, int max_step) const {
    if (count < 0 || (count > 0 && !ids)) return refuse("%s: count %d must be >= 0 and ids non-null", where, count);
    const int st = table.check(count, ids, where);
    if (st != FA_OK) return st;
    for (int i = 0; i < count; ++i) {
        const int s = table[ids[i]].step;
        if (s < min_step || s > max_step)
            return refuse("%s: request %d is at step %d, the call needs step %d..%d", where, ids[i], s, min_step, max_step);
    }
    return FA_OK;
}

int RequestSet::open_all(int count, const Mirror *next, int32_t *ids) {
    auto grow = [&](int grown) {
        return grow_slots(table.slots(), grown, stream, d_x, (size_t)kSlotFloats, d_meta, (size_t)kMetaFields);
    };
    auto init = [](int) { return FA_OK; };   // the epilogue kernel writes the slot and its meta row
    for (int i = 0; i < count; ++i) {
        int id = -1;
        const int st = table.open(64, grow, init, &id);
        if (st != FA_OK) {
            for (int j = 0; j < i; ++j) table.close(ids[j], "fa_luxtts_begin");
            return st;
        }
        table[id] = next[i];
        ids[i] = id;
    }
    return FA_OK;
}

int RequestSet::begin(const BeginArgs &a, bool device) {
    const char *where = device ? "fa_luxtts_begin_device" : "fa_luxtts_begin";
    const int count = a.count;
    if (count < 0) return refuse("%s: count %d < 0", where, count);
    if (count == 0) return FA_OK;
    if (!a.offsets || !a.prompt_tokens || !a.text_tokens || !a.speeds || !a.seeds || !a.reasons || !a.ids || !a.plans ||
        !a.speech_condition || !a.padding_mask)
        return refuse("%s: offsets, token counts, speeds, seeds, reasons, ids, plans and both outputs must be non-null",
                      where);
    if (a.offsets[0] < 0) return refuse("%s: offsets[0] is negative (%lld)", where, (long long)a.offsets[0]);
    for (int i = 0; i < count; ++i) {
        if (a.offsets[i + 1] < a.offsets[i] || a.offsets[i + 1] > (1LL << 62))
            return refuse("%s: offsets decrease at %d or pass 2^62", where, i);
        if (a.prompt_tokens[i] < 0 || a.text_tokens[i] < 0)
            return refuse("%s: request %d has a negative token count", where, i);
    }
    const long long span = a.offsets[count] - a.offsets[0];
    if (span > 0 && !a.prompt) return refuse("%s: prompt is NULL with %lld samples", where, span);

    std::vector<Mirror> next((size_t)count);
    std::vector<int64_t> gained_at((size_t)count + 1, 0), mel_at((size_t)count + 1, 0);
    long long max_n = 0;
    for (int i = 0; i < count; ++i) {
        const long long n = a.offsets[i + 1] - a.offsets[i];
        next[i].plan = plan_request(n, a.prompt_tokens[i], a.text_tokens[i], a.speeds[i]);
        const long long capped = std::min(n, kMaxPrompt);
        max_n = std::max(max_n, capped);
        gained_at[i + 1] = gained_at[i] + capped;
        mel_at[i + 1] = mel_at[i] + (1 + capped / kHop) * kFeat;   // the .center frames of the capped prompt
    }

    int st = desc.reserve((size_t)count * sizeof(BeginJob));
    if (st != FA_OK) return st;
    float *d_gained, *d_mel, *d_rms;
    st = carve_arena(d_scratch, [&](Carver &c) {
        d_gained = c.take<float>((size_t)gained_at[count] + 16);
        d_mel = c.take<float>((size_t)mel_at[count]);
        d_rms = c.take<float>((size_t)count);
    });
    if (st != FA_OK) return st;
    st = h_rms.grow((size_t)count * sizeof(float));
    if (st != FA_OK) return st;
    HostStaging H(!device, stream);
    const float *src = nullptr;
    float *k_sc, *k_pm;
    st = H.carve(d_io, [&](HostStaging::Layout &l) {
        src = l.in(span > 0 ? a.prompt + a.offsets[0] : nullptr, (size_t)span);
        k_sc = l.out(a.speech_condition, (size_t)count * kSlotFloats);
        k_pm = l.out(a.padding_mask, (size_t)count * kMaxFrames);
    });
    if (st != FA_OK) return st;
    auto *jobs = static_cast<BeginJob *>(desc.host.data());
    for (int i = 0; i < count; ++i) {
        const Plan &p = next[i].plan;
        jobs[i] = BeginJob{a.offsets[i] - a.offsets[0], gained_at[i + 1] - gained_at[i], gained_at[i],
                           mel_at[i], seed_state(a.seeds[i]), 1.0f, 0.0f, 0, 0, p.prompt_frames, p.features_length,
                           p.gen_frames, p.token_count};
    }
    st = desc.upload((size_t)count * sizeof(BeginJob), stream);
    if (st != FA_OK) return st;
    const auto *d_jobs = static_cast<const BeginJob *>(desc.device.data());
    FA_CUDA_TRY(launch(luxtts_rms_kernel, count, kRmsLanes, 0, stream, d_jobs, src, d_rms));
    FA_CUDA_TRY(cudaMemcpyAsync(h_rms.data(), d_rms, (size_t)count * sizeof(float), cudaMemcpyDeviceToHost, stream));
    FA_CUDA_TRY(cudaStreamSynchronize(stream));

    int refused = -1;
    for (int i = 0; i < count; ++i) {
        Mirror &m = next[i];
        int r = m.plan.reason;
        m.rms = h_rms.data()[i];
        if ((r == kOk || r >= kSilent) && !(m.rms > 0)) r = kSilent;   // synthesize checks the RMS before the mel
        m.plan.reason = r;
        a.reasons[i] = r;
        if (r != kOk && refused < 0) refused = i;
        m.boosted = r == kOk && m.rms < kTargetRms;
    }
    if (refused >= 0)
        return refuse("%s: request %d is refused with reason %d (see reasons)", where, refused, next[refused].plan.reason);

    st = open_all(count, next.data(), a.ids);
    if (st != FA_OK) return st;
    auto fail = [&](int status) {
        for (int i = 0; i < count; ++i) table.close(a.ids[i], where);
        return status;
    };
    st = desc.reserve((size_t)count * sizeof(BeginJob));
    if (st != FA_OK) return fail(st);
    jobs = static_cast<BeginJob *>(desc.host.data());
    for (int i = 0; i < count; ++i) {
        const Plan &p = next[i].plan;
        jobs[i] = BeginJob{a.offsets[i] - a.offsets[0], gained_at[i + 1] - gained_at[i], gained_at[i], mel_at[i],
                           seed_state(a.seeds[i]), next[i].boosted ? kTargetRms / next[i].rms : 1.0f, next[i].rms,
                           next[i].boosted ? 1 : 0, a.ids[i], p.prompt_frames, p.features_length, p.gen_frames,
                           p.token_count};
    }
    st = desc.upload((size_t)count * sizeof(BeginJob), stream);
    if (st != FA_OK) return fail(st);
    d_jobs = static_cast<const BeginJob *>(desc.device.data());
    cudaError_t e = launch(luxtts_gain_kernel, dim3((unsigned)count, tiles(max_n, kThreads)), kThreads, 0, stream,
                           d_jobs, src, d_gained);
    if (e != cudaSuccess) return fail(cuda_failure(e, "luxtts_gain_kernel", __FILE__, __LINE__));
    st = mel.compute_batch_device(d_gained, gained_at.data(), count, nullptr, FA_MEL_PAD_CENTER, FA_MEL_TIME_MAJOR, d_mel,
                                  mel_at.data(), nullptr, nullptr, stream);
    if (st != FA_OK) return fail(st);
    e = launch(luxtts_epilogue_kernel, dim3((unsigned)count, kSlotTiles), kThreads, 0, stream, d_jobs, d_mel, d_x.data(),
               d_meta.data(), k_sc, k_pm);
    if (e != cudaSuccess) return fail(cuda_failure(e, "luxtts_epilogue_kernel", __FILE__, __LINE__));
    e = H.finish();
    if (e != cudaSuccess) return fail(cuda_failure(e, "the begin outputs' copy", __FILE__, __LINE__));
    for (int i = 0; i < count; ++i) a.plans[i] = next[i];
    return FA_OK;
}

int RequestSet::text_condition(int count, const int *ids, const float *embeds, long long row_stride,
                               long long request_stride, bool device, float *out) {
    const char *where = device ? "fa_luxtts_text_condition_device" : "fa_luxtts_text_condition";
    int st = check(count, ids, where, 0, kSteps);
    if (st != FA_OK) return st;
    if (count == 0) return FA_OK;
    if (!embeds || !out) return refuse("%s: token_embeds and text_condition must be non-null", where);
    if (row_stride < kFeat || row_stride > (1LL << 40)) return refuse("%s: row_stride %lld < 100", where, row_stride);
    for (int i = 0; i < count; ++i)
        if (request_stride < (table[ids[i]].plan.token_count + 1LL) * row_stride || request_stride > (1LL << 50))
            return refuse("%s: request_stride %lld does not hold request %d's %d rows", where, request_stride, ids[i],
                          table[ids[i]].plan.token_count + 1);
    const long long in_n = (count - 1LL) * request_stride + table[ids[count - 1]].plan.token_count * row_stride + kFeat;
    st = desc.reserve((size_t)count * sizeof(StepJob));
    if (st != FA_OK) return st;
    HostStaging H(!device, stream);
    const float *k_in;
    float *k_out;
    st = H.carve(d_io, [&](HostStaging::Layout &l) {
        k_in = l.in(embeds, (size_t)in_n);
        k_out = l.out(out, (size_t)count * kSlotFloats);
    });
    if (st != FA_OK) return st;
    auto *jobs = static_cast<StepJob *>(desc.host.data());
    for (int i = 0; i < count; ++i) jobs[i] = StepJob{ids[i], table[ids[i]].step};
    st = desc.upload((size_t)count * sizeof(StepJob), stream);
    if (st != FA_OK) return st;
    FA_CUDA_TRY(launch(luxtts_text_kernel, dim3((unsigned)count, kSlotTiles), kThreads, 0, stream,
                       static_cast<const StepJob *>(desc.device.data()), d_meta.data(), k_in, row_stride,
                       request_stride, k_out));
    FA_CUDA_TRY(H.finish());
    return FA_OK;
}

int RequestSet::model_inputs(int count, const int *ids, bool device, float *x, float *t) {
    const char *where = device ? "fa_luxtts_model_inputs_device" : "fa_luxtts_model_inputs";
    int st = check(count, ids, where, 0, kSteps - 1);
    if (st != FA_OK) return st;
    if (count == 0) return FA_OK;
    if (!x || !t) return refuse("%s: x and t must be non-null", where);
    if (device && (reinterpret_cast<uintptr_t>(x) & 15)) return refuse("%s: x must be 16-byte aligned", where);
    st = desc.reserve((size_t)count * sizeof(StepJob));
    if (st != FA_OK) return st;
    HostStaging H(!device, stream);
    float *k_x, *k_t;
    st = H.carve(d_io, [&](HostStaging::Layout &l) {
        k_x = l.out(x, (size_t)count * kSlotFloats);
        k_t = l.out(t, (size_t)count);
    });
    if (st != FA_OK) return st;
    auto *jobs = static_cast<StepJob *>(desc.host.data());
    for (int i = 0; i < count; ++i) jobs[i] = StepJob{ids[i], table[ids[i]].step};
    st = desc.upload((size_t)count * sizeof(StepJob), stream);
    if (st != FA_OK) return st;
    FA_CUDA_TRY(launch(luxtts_inputs_kernel, dim3((unsigned)count, kSlotFloats / 4 / kThreads), kThreads, 0, stream,
                       static_cast<const StepJob *>(desc.device.data()), d_x.data(), k_x, k_t));
    FA_CUDA_TRY(H.finish());
    return FA_OK;
}

int RequestSet::advance(int count, const int *ids, const float *v, long long row_stride, long long request_stride,
                        bool device) {
    const char *where = device ? "fa_luxtts_advance_device" : "fa_luxtts_advance";
    int st = check(count, ids, where, 0, kSteps - 1);
    if (st != FA_OK) return st;
    if (count == 0) return FA_OK;
    if (!v) return refuse("%s: v must be non-null", where);
    if (row_stride < kFeat || row_stride > (1LL << 40)) return refuse("%s: row_stride %lld < 100", where, row_stride);
    for (int i = 0; i < count; ++i)
        if (request_stride < (long long)table[ids[i]].plan.features_length * row_stride || request_stride > (1LL << 50))
            return refuse("%s: request_stride %lld does not hold request %d's %d rows", where, request_stride, ids[i],
                          table[ids[i]].plan.features_length);
    const long long in_n =
        (count - 1LL) * request_stride + (table[ids[count - 1]].plan.features_length - 1LL) * row_stride + kFeat;
    st = desc.reserve((size_t)count * sizeof(StepJob));
    if (st != FA_OK) return st;
    HostStaging H(!device, stream);
    const float *k_v;
    st = H.carve(d_io, [&](HostStaging::Layout &l) { k_v = l.in(v, (size_t)in_n); });
    if (st != FA_OK) return st;
    auto *jobs = static_cast<StepJob *>(desc.host.data());
    for (int i = 0; i < count; ++i) jobs[i] = StepJob{ids[i], table[ids[i]].step};
    st = desc.upload((size_t)count * sizeof(StepJob), stream);
    if (st != FA_OK) return st;
    FA_CUDA_TRY(launch(luxtts_advance_kernel, dim3((unsigned)count, kSlotTiles), kThreads, 0, stream,
                       static_cast<const StepJob *>(desc.device.data()), d_meta.data(), k_v, row_stride,
                       request_stride, d_x.data()));
    FA_CUDA_TRY(H.sync());
    for (int i = 0; i < count; ++i) ++table[ids[i]].step;
    return FA_OK;
}

int RequestSet::vocoder_input(int count, const int *ids, int bucket, bool device, float *mel_out) {
    const char *where = device ? "fa_luxtts_vocoder_input_device" : "fa_luxtts_vocoder_input";
    int st = check(count, ids, where, kSteps, kSteps);
    if (st != FA_OK) return st;
    if (bucket != kBucketSmall && bucket != kBucketLarge) return refuse("%s: bucket %d is not 282 or 555", where, bucket);
    for (int i = 0; i < count; ++i)
        if (table[ids[i]].plan.bucket != bucket)
            return refuse("%s: request %d has bucket %d, not %d", where, ids[i], table[ids[i]].plan.bucket, bucket);
    if (count == 0) return FA_OK;
    if (!mel_out) return refuse("%s: mel must be non-null", where);
    st = desc.reserve((size_t)count * sizeof(StepJob));
    if (st != FA_OK) return st;
    HostStaging H(!device, stream);
    float *k_mel;
    st = H.carve(d_io, [&](HostStaging::Layout &l) { k_mel = l.out(mel_out, (size_t)count * kFeat * bucket); });
    if (st != FA_OK) return st;
    auto *jobs = static_cast<StepJob *>(desc.host.data());
    for (int i = 0; i < count; ++i) jobs[i] = StepJob{ids[i], kSteps};
    st = desc.upload((size_t)count * sizeof(StepJob), stream);
    if (st != FA_OK) return st;
    // invScale = 1 / featScale and log(logMelFloor), float32 as in synthesize
    const float inv_scale = 1.0f / kFeatScale, log_floor = std::log(1e-7f);
    FA_CUDA_TRY(launch(luxtts_vocoder_kernel, dim3((unsigned)count, tiles(bucket, kTile), tiles(kFeat, kTile)),
                       dim3(kTile, kTileRows), 0, stream, static_cast<const StepJob *>(desc.device.data()),
                       d_meta.data(), d_x.data(), bucket, inv_scale, log_floor, k_mel));
    FA_CUDA_TRY(H.finish());
    return FA_OK;
}

int RequestSet::finish(int count, const int *ids, const float *audio, long long row_stride, long long row_length,
                       bool device, float *samples, long long capacity, int64_t *lengths, int64_t *total) {
    const char *where = device ? "fa_luxtts_finish_device" : "fa_luxtts_finish";
    int st = check(count, ids, where, kSteps, kSteps);
    if (st != FA_OK) return st;
    if (!total || (count > 0 && !lengths)) return refuse("%s: lengths and total must be non-null", where);
    if (row_length < 0 || row_stride < row_length || row_stride > (1LL << 50))
        return refuse("%s: row_length %lld and row_stride %lld need 0 <= row_length <= row_stride", where, row_length,
                      row_stride);
    long long sum = 0, max_len = 0;
    for (int i = 0; i < count; ++i) {
        lengths[i] = std::min((long long)(table[ids[i]].plan.gen_frames - 1) * kHop48k, row_length);
        sum += lengths[i];
        max_len = std::max(max_len, (long long)lengths[i]);
    }
    *total = sum;
    if (sum > 0 && !audio) return refuse("%s: audio is NULL with %lld samples to keep", where, sum);
    if (sum > capacity) {
        set_error("%s: %lld samples, capacity %lld", where, sum, capacity);
        return FA_OUTPUT_TOO_SMALL;
    }
    if (sum > 0 && !samples) return refuse("%s: samples is NULL with %lld samples", where, sum);
    if (sum > 0) {
        st = desc.reserve((size_t)count * sizeof(FinishJob));
        if (st != FA_OK) return st;
        HostStaging H(!device, stream);
        const float *k_in;
        float *k_out;
        st = H.carve(d_io, [&](HostStaging::Layout &l) {
            k_in = l.in(audio, (size_t)((count - 1LL) * row_stride + row_length));
            k_out = l.out(samples, (size_t)sum);
        });
        if (st != FA_OK) return st;
        auto *jobs = static_cast<FinishJob *>(desc.host.data());
        long long at = 0;
        for (int i = 0; i < count; ++i) {
            jobs[i] = FinishJob{at, lengths[i], ids[i], 0};
            at += lengths[i];
        }
        st = desc.upload((size_t)count * sizeof(FinishJob), stream);
        if (st != FA_OK) return st;
        FA_CUDA_TRY(launch(luxtts_finish_kernel, dim3((unsigned)count, tiles(max_len, kThreads)), kThreads, 0, stream,
                           static_cast<const FinishJob *>(desc.device.data()), d_meta.data(), k_in, row_stride, k_out));
        FA_CUDA_TRY(H.finish());
    }
    for (int i = 0; i < count; ++i) table.close(ids[i], where);
    return FA_OK;
}

int RequestSet::close(int id) { return table.close(id, "fa_luxtts_close"); }

int RequestSet::state(int id, Mirror *m, float *x) {
    const int st = table.check(1, &id, "fa_luxtts_request_state");
    if (st != FA_OK) return st;
    if (x)
        FA_CUDA_TRY(cudaMemcpyAsync(x, d_x.data() + (size_t)id * kSlotFloats, kSlotFloats * sizeof(float),
                                    cudaMemcpyDeviceToHost, stream));
    FA_CUDA_TRY(cudaStreamSynchronize(stream));
    *m = table[id];
    return FA_OK;
}

} // namespace luxtts
} // namespace fa
