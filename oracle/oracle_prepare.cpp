// ORACLE — TEST INFRASTRUCTURE ONLY.  Not part of the shipped product path.
//
// Sequential float32 restatement of the arithmetic of OfflineDiarizerManager.prepare, written from the Swift sources
// (paths under Sources/FluidAudio/Diarizer/Offline), loop for loop as the reference runs it:
//   Segmentation/OfflineSegmentationProcessor.swift:55-56,118-190,303   windows and chunk offsets
//   Segmentation/OfflineSegmentationProcessor.swift:15-24,321-405        powerset decoding, histogram, speech frames
//   Utils/VDSPOperations.swift:142-155                                   logSumExp
//   Extraction/WeightInterpolation.swift:19-146                          resample
//   Extraction/OfflineEmbeddingExtractor.swift:338-351,381-387,421-707,807-842   the embedding stage's bookkeeping
// Built with -O2 -ffp-contract=off on baseline x86-64: every operation is rounded as written.  expf / logf are the host
// libm's (Apple's vvexpf is closed) and every vDSP sum runs in index order (vDSP's order is closed).
#include <algorithm>
#include <cfloat>
#include <climits>
#include <cmath>
#include <cstdint>
#include <vector>

namespace {

float swift_min(float x, float y) { return y < x ? y : x; }
float swift_max(float x, float y) { return y >= x ? y : x; }

const int kPowerset[8][3] = {{-1, -1, -1}, {0, -1, -1}, {1, -1, -1}, {2, -1, -1},
                             {0, 1, -1},   {0, 2, -1},  {1, 2, -1},  {0, 1, 2}};

float log_sum_exp(const float *x, int n) {
    float max_element = x[0];
    for (int i = 1; i < n; ++i)
        if (max_element < x[i]) max_element = x[i];
    const float shift = -max_element;
    std::vector<float> shifted(n);
    for (int i = 0; i < n; ++i) shifted[i] = x[i] + shift;
    for (int i = 0; i < n; ++i) shifted[i] = expf(shifted[i]);
    float sum = 0;
    for (int i = 0; i < n; ++i) sum += shifted[i];
    return logf(sum) + max_element;
}

std::vector<float> resample(const std::vector<float> &input, int output_length) {
    if (input.empty() || output_length <= 0) return {};
    const int input_length = (int)input.size();
    if (input_length == output_length) return input;
    std::vector<float> output(output_length);
    const float scale = (float)output_length / (float)input_length;
    for (int index = 0; index < output_length; ++index) {
        const float position = ((float)index + 0.5f) / scale - 0.5f;
        const float clamped = swift_min(swift_max(position, 0.0f), (float)(input_length - 1));
        const int left = (int)std::floor(clamped);
        const int right = std::min(left + 1, input_length - 1);
        const float weight_right = clamped - (float)left;
        const float weight_left = 1 - weight_right;
        output[index] = input[left] * weight_left + input[right] * weight_right;
    }
    return output;
}

float sum_of(const std::vector<float> &v) {
    float s = 0;
    for (float x : v) s += x;
    return s;
}

float dot_of(const std::vector<float> &a, const std::vector<float> &b) {
    float s = 0;
    for (size_t i = 0; i < a.size(); ++i) s += a[i] * b[i];
    return s;
}

float mask_cosine(const std::vector<float> &a, const std::vector<float> &b) {
    if (a.size() != b.size() || a.empty()) return 0;
    const float dot = dot_of(a, b), norm_a = dot_of(a, a), norm_b = dot_of(b, b);
    const float denom = std::sqrt(norm_a) * std::sqrt(norm_b);
    return denom > 0 ? dot / denom : 0;
}

long long samples_per_window(int sample_rate, double window_duration) {
    return (long long)((double)sample_rate * window_duration);
}
long long samples_per_step(int sample_rate, double window_duration, double step_ratio) {
    return std::max(1LL, (long long)((double)samples_per_window(sample_rate, window_duration) * step_ratio));
}

} // namespace

extern "C" {

// samplesPerWindow / samplesPerStep and the offsets stride(from: 0, to: totalSamples, by: stepSize) yields
long long oracle_seg_window_count(long long total_samples, int sample_rate, double window_duration, double step_ratio,
                                  long long *window, long long *step) {
    *window = samples_per_window(sample_rate, window_duration);
    *step = samples_per_step(sample_rate, window_duration, step_ratio);
    long long n = 0;
    for (long long offset = 0; offset < total_samples; offset += *step) ++n;
    return n;
}

// populateWindow (:118-187) for every window: out [count x window], offsets [count]
void oracle_seg_windows(const float *audio, long long total_samples, int sample_rate, double window_duration,
                        double step_ratio, float *out, double *offsets) {
    const long long chunk = samples_per_window(sample_rate, window_duration);
    const long long step = samples_per_step(sample_rate, window_duration, step_ratio);
    long long index = 0;
    for (long long offset = 0; offset < total_samples; offset += step, ++index) {
        const long long available = std::max(0LL, std::min(chunk, total_samples - offset));
        float *dst = out + index * chunk;
        for (long long i = 0; i < available; ++i) dst[i] = audio[offset + i];
        for (long long i = available; i < chunk; ++i) dst[i] = 0;
        offsets[index] = (double)offset / (double)sample_rate;
    }
}

// :321-405 for chunks x frames frames of `classes` logits
void oracle_seg_decode(const float *logits, int chunks, int frames, int classes, float onset, float *log_probs,
                       float *weights, long long *histogram, long long *speech_frames, float *speech_probability) {
    const int speaker_count = 3;
    for (int k = 0; k < 8; ++k) histogram[k] = 0;
    *speech_frames = 0;
    std::vector<float> probability(classes);
    for (long long frame = 0; frame < (long long)chunks * frames; ++frame) {
        const float *x = logits + frame * classes;
        float *lp = log_probs + frame * classes;
        int best_index = 0;
        float best_value = -FLT_MAX;
        for (int cls = 0; cls < classes; ++cls)
            if (x[cls] > best_value) {
                best_value = x[cls];
                best_index = cls;
            }
        const float shift = -log_sum_exp(x, classes);
        for (int cls = 0; cls < classes; ++cls) lp[cls] = x[cls] + shift;
        for (int cls = 0; cls < classes; ++cls) probability[cls] = expf(lp[cls]);
        if (best_index < 8) histogram[best_index] += 1;
        const int winning = std::min(best_index, 7);
        float *w = weights + frame * speaker_count;
        for (int s = 0; s < speaker_count; ++s) w[s] = 0;
        for (int k = 0; k < 3; ++k)
            if (kPowerset[winning][k] >= 0 && kPowerset[winning][k] < speaker_count) w[kPowerset[winning][k]] = 1.0f;
        const float speech = swift_max(0.0f, swift_min(1.0f, 1 - probability[0]));
        if (speech_probability) speech_probability[frame] = speech;
        if (speech >= onset) *speech_frames += 1;
    }
}

void oracle_weight_resample(const float *rows, long long row_count, int in_len, int out_len, float *out) {
    for (long long r = 0; r < row_count; ++r) {
        const std::vector<float> y = resample(std::vector<float>(rows + r * in_len, rows + (r + 1) * in_len), out_len);
        std::copy(y.begin(), y.end(), out + r * out_len);
    }
}

// InterpolationCoefficients.init (:28-49)
void oracle_interp_table(int in_len, int out_len, int *left, int *right, float *w_left, float *w_right) {
    const float scale = (float)out_len / (float)in_len;
    for (int index = 0; index < out_len; ++index) {
        const float position = ((float)index + 0.5f) / scale - 0.5f;
        const float clamped = swift_min(swift_max(position, 0.0f), (float)(in_len - 1));
        left[index] = (int)std::floor(clamped);
        right[index] = std::min(left[index] + 1, in_len - 1);
        w_right[index] = clamped - (float)left[index];
        w_left[index] = 1 - w_right[index];
    }
}

// The chunk loop (:651-707) and processChunk (:421-613).  Per emitted entry (capacity chunks * speakers): the
// TimedEmbedding metadata, maskSum, whether the base mask was the fallback, the entry whose embedding the skip strategy
// reuses (-1: its own), maskToUse and the resampled mask.  counters: evaluated, empty, fallback, skipped.
// active [chunks]: 1 when the chunk reached the embedding stage.  sums [chunks x speakers x 3]: baseSum, cleanSum and
// maskEnergy as far as they were computed (NaN beyond).  Returns the number of entries.
int oracle_embedding_plan(const float *weights, int chunks, int frames, int speakers, const double *chunk_offsets,
                          int offsets_count, double frame_duration_in, long long total_samples, int sample_rate,
                          double window_duration, int exclude_overlap, double min_segment_duration, float skip_threshold,
                          int weight_frames, int fbank_batch, int *chunk_index, int *speaker_index, int *start_frame,
                          int *end_frame, double *start_time, double *end_time, float *mask_sum_out, int *used_fallback,
                          int *reuse_of, float *frame_weights, float *model_weights, long long *counters, int *active,
                          float *sums) {
    const float overlap_threshold = 1e-3f;
    const bool skipping = skip_threshold >= 0;
    const long long chunk_size = samples_per_window(sample_rate, window_duration);
    for (int k = 0; k < 4; ++k) counters[k] = 0;
    for (long long i = 0; sums && i < (long long)chunks * speakers * 3; ++i) sums[i] = NAN;
    int count = 0, in_batch = 0;
    std::vector<int> cache_entry(speakers, -1);
    std::vector<std::vector<float>> cache_mask(speakers);
    if (frames <= 0 || speakers <= 0) chunks = 0;
    for (int c = 0; c < chunks; ++c) {
        if (active) active[c] = 0;
        const double frame_duration = frame_duration_in > 0 ? frame_duration_in : window_duration / (double)std::max(1, frames);
        const double given = c < offsets_count ? chunk_offsets[c] : (double)c * window_duration;
        const double offset = std::isfinite(given) ? given : (double)c * window_duration;
        const double estimated = std::round(offset * (double)sample_rate);
        const long long est = estimated <= -9e18 ? LLONG_MIN / 2 : (estimated >= 9e18 ? LLONG_MAX / 2 : (long long)estimated);
        const long long start = std::max(0LL, std::min(est, total_samples));
        const long long end = std::min(start + chunk_size, total_samples);
        if (!(start < end)) continue;
        if (active) active[c] = 1;

        int min_frames = 1;
        if (frame_duration > 0) min_frames = std::max(1, (int)std::ceil(min_segment_duration / frame_duration));
        const float *w = weights + (long long)c * frames * speakers;
        std::vector<bool> overlap(frames, false);
        if (exclude_overlap)
            for (int f = 0; f < frames; ++f) {
                int n = 0;
                for (int s = 0; s < speakers; ++s)
                    if (w[f * speakers + s] > overlap_threshold && ++n > 1) {
                        overlap[f] = true;
                        break;
                    }
            }
        for (int s = 0; s < speakers; ++s) {
            counters[0] += 1;
            float *trace = sums ? sums + ((long long)c * speakers + s) * 3 : nullptr;
            std::vector<float> base(frames);
            for (int f = 0; f < frames; ++f) base[f] = w[f * speakers + s];
            const float base_sum = sum_of(base);
            if (trace) trace[0] = base_sum;
            if (base_sum <= 0) {
                counters[1] += 1;
                continue;
            }
            std::vector<float> clean = base;
            if (exclude_overlap)
                for (int f = 0; f < frames; ++f)
                    if (overlap[f]) clean[f] = 0;
            const float clean_sum = sum_of(clean);
            if (trace) trace[1] = clean_sum;
            if (clean_sum < (float)frames * 0.2f) {
                counters[1] += 1;
                continue;
            }
            const bool use_clean = clean_sum >= (float)min_frames;
            const std::vector<float> &mask = use_clean ? clean : base;
            const float mask_sum = use_clean ? clean_sum : base_sum;
            if (!use_clean) counters[2] += 1;
            if (mask_sum <= 0) {
                counters[1] += 1;
                continue;
            }
            const std::vector<float> resampled = resample(mask, weight_frames);
            const float energy = sum_of(resampled);
            if (trace) trace[2] = energy;
            if (energy <= 0) {
                counters[1] += 1;
                continue;
            }
            int reused = -1;
            if (skipping && cache_entry[s] >= 0 && mask_cosine(mask, cache_mask[s]) >= skip_threshold) {
                reused = cache_entry[s];
                counters[3] += 1;
            } else if (skipping) {
                cache_entry[s] = count;
                cache_mask[s] = mask;
            }
            int first = 0, last = -1;
            for (int f = 0; f < frames; ++f)
                if (mask[f] > overlap_threshold) {
                    first = f;
                    break;
                }
            for (int f = frames - 1; f >= 0; --f)
                if (mask[f] > overlap_threshold) {
                    last = f;
                    break;
                }
            if (last < 0) last = first;
            chunk_index[count] = c;
            speaker_index[count] = s;
            start_frame[count] = first;
            end_frame[count] = last;
            start_time[count] = offset + (double)first * frame_duration;
            end_time[count] = offset + (double)(last + 1) * frame_duration;
            mask_sum_out[count] = mask_sum;
            used_fallback[count] = use_clean ? 0 : 1;
            reuse_of[count] = reused;
            std::copy(mask.begin(), mask.end(), frame_weights + (long long)count * frames);
            std::copy(resampled.begin(), resampled.end(), model_weights + (long long)count * weight_frames);
            ++count;
        }
        if (++in_batch == fbank_batch) {   // flushFbankBatch: the cache does not outlive the batch (:632-639)
            in_batch = 0;
            std::fill(cache_entry.begin(), cache_entry.end(), -1);
        }
    }
    return count;
}

// The fbank input of the listed chunks (:663-691, 807-832): out [count x audio_sample_count]
void oracle_embed_windows(const float *audio, long long total_samples, const double *chunk_offsets, int offsets_count,
                          const int *chunks, int count, int sample_rate, double window_duration, int audio_sample_count,
                          float *out) {
    const long long chunk_size = samples_per_window(sample_rate, window_duration);
    for (int i = 0; i < count; ++i) {
        const int c = chunks[i];
        const double given = c < offsets_count ? chunk_offsets[c] : (double)c * window_duration;
        const double offset = std::isfinite(given) ? given : (double)c * window_duration;
        const double estimated = std::round(offset * (double)sample_rate);
        const long long est = estimated <= -9e18 ? LLONG_MIN / 2 : (estimated >= 9e18 ? LLONG_MAX / 2 : (long long)estimated);
        const long long start = std::max(0LL, std::min(est, total_samples));
        const long long end = std::min(start + chunk_size, total_samples);
        float *dst = out + (long long)i * audio_sample_count;
        for (int k = 0; k < audio_sample_count; ++k) dst[k] = 0;
        const long long copy = std::min<long long>(std::max(0LL, end - start), audio_sample_count);
        for (long long k = 0; k < copy; ++k) dst[k] = audio[start + k];
    }
}

} // extern "C"
