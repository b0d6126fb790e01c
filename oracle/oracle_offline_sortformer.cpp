// ORACLE — TEST INFRASTRUCTURE ONLY.  Not part of the shipped product path.
//
// A sequential CPU restatement of OfflineSortformerDiarizer's window work (Sources/FluidAudio/Diarizer/Sortformer/
// Offline/OfflineSortformerDiarizer.swift: runOffline's copy at :98-119 and processComplete's window loop at :279-363)
// and of SortformerSpeakerStitcher.alignment with its recursive permutation enumeration (SortformerSpeakerStitcher.swift:
// 27-90), line by line in the reference's order.  processComplete calls the model through a callback, one window at a
// time, in the reference's order.  Built with -O2 -ffp-contract=off on baseline x86-64.
#include <algorithm>
#include <cfloat>
#include <cstdint>
#include <functional>
#include <vector>

namespace {

constexpr int kWindowOutputFrames = 384, kSubsamplingFactor = 8, kNumSpeakers = 4, kMelFeatures = 128;
constexpr int kWindowMelFrames = kWindowOutputFrames * kSubsamplingFactor;

// permute(_:_:_:): heap-free recursive enumeration, body called once per permutation
void permute(std::vector<int> &array, int k, const std::function<void(const std::vector<int> &)> &body) {
    if (k == (int)array.size()) {
        body(array);
        return;
    }
    for (int i = k; i < (int)array.size(); ++i) {
        std::swap(array[k], array[i]);
        permute(array, k + 1, body);
        std::swap(array[k], array[i]);
    }
}

std::vector<int> alignment(const float *global, size_t global_count, const float *window, size_t window_count,
                           int frames, int num_speakers) {
    std::vector<int> identity(num_speakers > 0 ? num_speakers : 0);
    for (int i = 0; i < num_speakers; ++i) identity[i] = i;
    if (!(frames > 0 && num_speakers > 0 && global_count >= (size_t)frames * num_speakers &&
          window_count >= (size_t)frames * num_speakers))
        return identity;
    std::vector<std::vector<float>> correlation(num_speakers, std::vector<float>(num_speakers, 0.0f));
    for (int f = 0; f < frames; ++f) {
        const int base = f * num_speakers;
        for (int g = 0; g < num_speakers; ++g) {
            const float gv = global[base + g];
            if (!(gv != 0)) continue;
            for (int w = 0; w < num_speakers; ++w) correlation[g][w] += gv * window[base + w];
        }
    }
    std::vector<int> best_perm = identity;
    float best_score = -FLT_MAX;
    std::vector<int> perm = identity;
    permute(perm, 0, [&](const std::vector<int> &candidate) {
        float score = 0;
        for (int g = 0; g < num_speakers; ++g) score += correlation[g][candidate[g]];
        if (score > best_score) {
            best_score = score;
            best_perm = candidate;
        }
    });
    std::vector<int> mapping = identity;
    for (int g = 0; g < num_speakers; ++g) mapping[best_perm[g]] = g;
    return mapping;
}

} // namespace

extern "C" {

typedef void (*oracle_osf_model)(const float *mel, int32_t mel_length, float *speaker_preds, void *ctx);

// runOffline's copy into mel [128 x 3072] (channels-first) and mel_length from validMelFrames time-major rows
void oracle_osf_run_offline(const float *mel_time_major, int64_t valid_mel_frames, float *dst, int32_t *mel_length) {
    const int64_t feature_count = kMelFeatures;
    const int64_t window_frames = kWindowMelFrames;
    const int64_t frames = std::min(valid_mel_frames, window_frames);
    for (int64_t t = 0; t < frames; ++t) {
        const int64_t src_base = t * feature_count;
        for (int64_t c = 0; c < feature_count; ++c) dst[c * window_frames + t] = mel_time_major[src_base + c];
    }
    if (frames < window_frames) {
        for (int64_t c = 0; c < feature_count; ++c) {
            const int64_t row_base = c * window_frames;
            for (int64_t t = frames; t < window_frames; ++t) dst[row_base + t] = 0;
        }
    }
    *mel_length = (int32_t)frames;
}

// SortformerSpeakerStitcher.alignment: mapping [num_speakers]
void oracle_osf_alignment(const float *global, const float *window, int64_t frames, int64_t num_speakers,
                          int32_t *mapping) {
    const size_t n = frames > 0 && num_speakers > 0 ? (size_t)(frames * num_speakers) : 0;
    const std::vector<int> m = alignment(global, n, window, n, (int)frames, (int)num_speakers);
    for (size_t i = 0; i < m.size(); ++i) mapping[i] = m[i];
}

// processComplete from `computeFlatTransposed`'s rows [num_mel_frames x 128] to the finalized predictions it rebuilds
// the timeline from: global [totalOut x 4], each window's mapping [windows x 4] (mappings may be NULL), *windows.
// Returns totalOut.
int64_t oracle_osf_process_complete(const float *mel_flat, int64_t num_mel_frames, int64_t overlap_output_frames,
                                    oracle_osf_model model, void *ctx, float *global_out, int32_t *mappings,
                                    int64_t *windows) {
    *windows = 0;
    const int64_t feature_count = kMelFeatures;
    const int64_t window_mel = kWindowMelFrames;
    const int64_t out_per_window = kWindowOutputFrames;
    const int64_t speakers = kNumSpeakers;
    const int64_t sub = kSubsamplingFactor;
    if (!(num_mel_frames > 0)) return 0;

    const int64_t overlap_out = std::max<int64_t>(0, std::min(overlap_output_frames, out_per_window - 1));
    const int64_t hop_out = out_per_window - overlap_out;
    const int64_t hop_mel = hop_out * sub;

    const int64_t total_out = (num_mel_frames + sub - 1) / sub;
    std::vector<float> global((size_t)(total_out * speakers), 0.0f);
    std::vector<bool> filled((size_t)total_out, false);
    std::vector<float> mel((size_t)(feature_count * window_mel));
    std::vector<float> preds((size_t)(out_per_window * speakers));

    int64_t mel_start = 0;
    int64_t window_index = 0;
    while (mel_start < num_mel_frames) {
        const int64_t valid_mel = std::min(window_mel, num_mel_frames - mel_start);
        std::vector<float> slice(mel_flat + mel_start * feature_count,
                                 mel_flat + (mel_start + valid_mel) * feature_count);
        int32_t mel_length = 0;
        oracle_osf_run_offline(slice.data(), valid_mel, mel.data(), &mel_length);
        model(mel.data(), mel_length, preds.data(), ctx);

        const int64_t valid_out = std::min(out_per_window, (valid_mel + sub - 1) / sub);
        const int64_t g_start = mel_start / sub;

        std::vector<int> mapping(speakers);
        for (int s = 0; s < speakers; ++s) mapping[s] = s;
        if (window_index > 0 && overlap_out > 0) {
            const int64_t ov = std::min(std::min(overlap_out, valid_out), std::max<int64_t>(0, total_out - g_start));
            if (ov > 0) {
                std::vector<float> g_overlap((size_t)(ov * speakers), 0.0f), w_overlap((size_t)(ov * speakers), 0.0f);
                for (int64_t j = 0; j < ov; ++j) {
                    const int64_t g_base = (g_start + j) * speakers;
                    const int64_t w_base = j * speakers;
                    for (int64_t s = 0; s < speakers; ++s) {
                        g_overlap[w_base + s] = global[g_base + s];
                        w_overlap[w_base + s] = preds[w_base + s];
                    }
                }
                mapping = alignment(g_overlap.data(), g_overlap.size(), w_overlap.data(), w_overlap.size(), (int)ov,
                                    (int)speakers);
            }
        }
        if (mappings)
            for (int64_t s = 0; s < speakers; ++s) mappings[window_index * speakers + s] = mapping[s];

        for (int64_t j = 0; j < valid_out; ++j) {
            const int64_t gf = g_start + j;
            if (!(gf < total_out)) break;
            const int64_t out_base = gf * speakers;
            const int64_t in_base = j * speakers;
            if (filled[gf]) {
                for (int64_t w = 0; w < speakers; ++w) {
                    const int64_t idx = out_base + mapping[w];
                    global[idx] = (global[idx] + preds[in_base + w]) * 0.5f;
                }
            } else {
                for (int64_t w = 0; w < speakers; ++w) global[out_base + mapping[w]] = preds[in_base + w];
                filled[gf] = true;
            }
        }

        window_index += 1;
        if (valid_mel < window_mel) break;
        mel_start += hop_mel;
    }
    *windows = window_index;
    std::copy(global.begin(), global.end(), global_out);
    return total_out;
}

} // extern "C"
