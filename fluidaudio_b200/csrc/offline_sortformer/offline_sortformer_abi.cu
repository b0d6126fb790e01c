// C ABI of offline Sortformer windows (declared in include/fluidaudio_b200_offline_sortformer.h) over
// offline_sortformer_kernels.cu.  Every argument is checked here before any copy or launch; every entry point returns
// through guard() (c_abi.h), and the data-taking calls lease the pooled call context (call_context.h).
#include "../../../include/fluidaudio_b200_offline_sortformer.h"
#include "../c_abi.h"
#include "offline_sortformer.h"

// The family's entry points: C linkage, exported, returning the main header's fa_status.  The library-wide guard scan
// (tests/test_abi_errors.py) keeps a closed list of family headers; tests/test_offline_sortformer_abi.py holds every
// entry point spelled this way to the same rule: one statement, `return guard(__func__, ...)`.
#define FA_OFFLINE_SORTFORMER_API FA_API fa_status

using namespace fa;
using namespace fa::offline_sortformer;

namespace {

constexpr long long kMaxFrames = 1LL << 40;
constexpr long long kMaxWindows = 1LL << 24;

// Checks the frame counts and sums the files' windows and output rows
int count_files(const char *where, int count, const int64_t *mel_frames, int overlap, long long *windows,
                long long *rows) {
    *windows = *rows = 0;
    for (int i = 0; i < count; ++i) {
        if (mel_frames[i] < 0 || mel_frames[i] > kMaxFrames)
            return refuse("%s: mel_frames[%d] = %lld is outside 0 .. 2^40", where, i, (long long)mel_frames[i]);
        *windows += window_count(mel_frames[i], overlap);
        *rows += total_out(mel_frames[i]);
    }
    if (*windows > kMaxWindows) return refuse("%s: the files have %lld windows, more than 2^24", where, *windows);
    return FA_STATUS_OK;
}

int model_inputs_call(int overlap, int count, const float *mel, const int64_t *mel_offsets, const int64_t *mel_frames,
                      int64_t capacity, float *model_mel, int32_t *mel_length, bool device) {
    const char *where = device ? "fa_offline_sortformer_model_inputs_device" : "fa_offline_sortformer_model_inputs";
    if (count < 0) return refuse("%s: count %d < 0", where, count);
    if (count == 0) return FA_STATUS_OK;
    if (!mel_offsets || !mel_frames) return refuse("%s: mel_offsets and mel_frames must be non-null", where);
    if (capacity < 0) return refuse("%s: window_capacity %lld < 0", where, (long long)capacity);
    overlap = clamp_overlap(overlap);
    long long windows, rows;
    int st = count_files(where, count, mel_frames, overlap, &windows, &rows);
    if (st != FA_STATUS_OK) return st;
    for (int i = 0; i < count; ++i)
        if (mel_frames[i] > 0 && (mel_offsets[i] < 0 || mel_offsets[i] > (1LL << 62) - mel_frames[i] * kMels))
            return refuse("%s: mel_offsets[%d] = %lld is negative or its rows pass 2^62", where, i,
                          (long long)mel_offsets[i]);
    if (windows > capacity) {
        set_error("%s: the files have %lld windows, window_capacity is %lld", where, windows, (long long)capacity);
        return FA_STATUS_OUTPUT_TOO_SMALL;
    }
    if (windows == 0) return FA_STATUS_OK;
    if (!mel || !model_mel || !mel_length) return refuse("%s: mel, model_mel and mel_length must be non-null", where);
    if (require_device() != FA_OK) return FA_STATUS_NO_DEVICE;
    return with_context(0, [&](CallContext &C) {
        return model_inputs(C, overlap, count, mel, mel_offsets, mel_frames, windows, device, model_mel, mel_length);
    });
}

int stitch_call(int overlap, int count, const int64_t *mel_frames, const float *preds, float *predictions,
                int32_t *mappings, bool device) {
    const char *where = device ? "fa_offline_sortformer_stitch_device" : "fa_offline_sortformer_stitch";
    if (count < 0) return refuse("%s: count %d < 0", where, count);
    if (count == 0) return FA_STATUS_OK;
    if (!mel_frames) return refuse("%s: mel_frames is NULL", where);
    overlap = clamp_overlap(overlap);
    long long windows, rows;
    int st = count_files(where, count, mel_frames, overlap, &windows, &rows);
    if (st != FA_STATUS_OK) return st;
    if (windows == 0) return FA_STATUS_OK;
    if (!preds || !predictions) return refuse("%s: speaker_preds and predictions must be non-null", where);
    if (require_device() != FA_OK) return FA_STATUS_NO_DEVICE;
    return with_context(0, [&](CallContext &C) {
        return stitch(C, overlap, count, mel_frames, preds, windows, rows, device, predictions, mappings);
    });
}

} // namespace

FA_OFFLINE_SORTFORMER_API fa_offline_sortformer_plan(int32_t overlap, int32_t count, const int64_t *mel_frames,
                                                     int64_t *window_counts, int64_t *output_frames) {
    return guard(__func__, [&]() -> int {
        if (count < 0) return refuse("fa_offline_sortformer_plan: count %d < 0", count);
        if (count == 0) return FA_STATUS_OK;
        if (!mel_frames || !window_counts || !output_frames)
            return refuse("fa_offline_sortformer_plan: mel_frames, window_counts and output_frames must be non-null");
        for (int i = 0; i < count; ++i)
            if (mel_frames[i] < 0 || mel_frames[i] > kMaxFrames)
                return refuse("fa_offline_sortformer_plan: mel_frames[%d] = %lld is outside 0 .. 2^40", i,
                              (long long)mel_frames[i]);
        const int ov = clamp_overlap(overlap);
        for (int i = 0; i < count; ++i) {
            window_counts[i] = window_count(mel_frames[i], ov);
            output_frames[i] = total_out(mel_frames[i]);
        }
        return FA_STATUS_OK;
    });
}

FA_OFFLINE_SORTFORMER_API fa_offline_sortformer_model_inputs(int32_t overlap, int32_t count, const float *mel,
                                                             const int64_t *mel_offsets, const int64_t *mel_frames,
                                                             int64_t window_capacity, float *model_mel,
                                                             int32_t *mel_length) {
    return guard(__func__, [&] {
        return model_inputs_call(overlap, count, mel, mel_offsets, mel_frames, window_capacity, model_mel, mel_length,
                                 false);
    });
}

FA_OFFLINE_SORTFORMER_API fa_offline_sortformer_model_inputs_device(int32_t overlap, int32_t count, const float *d_mel,
                                                                    const int64_t *mel_offsets,
                                                                    const int64_t *mel_frames, int64_t window_capacity,
                                                                    float *d_model_mel, int32_t *d_mel_length) {
    return guard(__func__, [&] {
        return model_inputs_call(overlap, count, d_mel, mel_offsets, mel_frames, window_capacity, d_model_mel,
                                 d_mel_length, true);
    });
}

FA_OFFLINE_SORTFORMER_API fa_offline_sortformer_stitch(int32_t overlap, int32_t count, const int64_t *mel_frames,
                                                       const float *speaker_preds, float *predictions,
                                                       int32_t *mappings) {
    return guard(__func__, [&] {
        return stitch_call(overlap, count, mel_frames, speaker_preds, predictions, mappings, false);
    });
}

FA_OFFLINE_SORTFORMER_API fa_offline_sortformer_stitch_device(int32_t overlap, int32_t count, const int64_t *mel_frames,
                                                              const float *d_speaker_preds, float *d_predictions,
                                                              int32_t *d_mappings) {
    return guard(__func__, [&] {
        return stitch_call(overlap, count, mel_frames, d_speaker_preds, d_predictions, d_mappings, true);
    });
}
