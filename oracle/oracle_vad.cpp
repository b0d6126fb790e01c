// ORACLE — TEST INFRASTRUCTURE ONLY.  Sequential CPU restatement of voice activity detection around the Silero and
// FSMN-VAD models, written from the reference's behaviour (Sources/FluidAudio/VAD/): VadSegmentationConfig's checks
// and thresholds, VadManager.processChunk's staging, streamingStateMachine, detectSpeechSampleRanges with its whole
// possibleEnds list and a separate padding pass, and FsmnVadManager.decide with its window array.
#include <cmath>
#include <cstdint>
#include <vector>

namespace {

struct Config {   // fa_vad_config's layout
    float default_threshold;
    double min_speech, min_silence, max_speech, pad;
    float split;
    int32_t has_negative;
    float negative, offset;
    double min_silence_at_max;
    int32_t use_max;
};

struct Resolved {   // fa_vad_resolved's layout
    float threshold, negative, split;
    int32_t use_max;
    int64_t min_speech, min_silence, max_speech, pad, min_silence_at_max;
};

template <typename T> T smin(T x, T y) { return y < x ? y : x; }   // Swift.min
template <typename T> T smax(T x, T y) { return y >= x ? y : x; }  // Swift.max

bool to_samples(double seconds, int64_t &out) {
    if (std::isnan(seconds) || std::isinf(seconds) || seconds < 0) return false;
    const double x = seconds * 16000.0;
    if (x >= 4611686018427387904.0) return false;   // 2^62 samples or more
    out = (int64_t)x;
    return true;
}

const int kChunk = 4096, kContext = 64;

} // namespace

extern "C" {

// 0 and *out, or 1 when the config is refused
int oracle_vad_resolve(const Config *c, Resolved *out) {
    Resolved r{};
    if (std::isnan(c->min_speech) || c->min_speech < 0) return 1;
    if (std::isnan(c->min_silence) || c->min_silence < 0) return 1;
    if (std::isnan(c->max_speech) || c->max_speech <= 0) return 1;
    if (std::isnan(c->pad) || c->pad < 0) return 1;
    if (std::isnan(c->split) || c->split < 0 || c->split > 1) return 1;
    if (std::isnan(c->offset) || c->offset < 0) return 1;
    if (std::isnan(c->min_silence_at_max) || c->min_silence_at_max < 0) return 1;
    if (c->has_negative && (std::isnan(c->negative) || c->negative < 0 || c->negative > 1)) return 1;
    if (!to_samples(c->min_speech, r.min_speech) || !to_samples(c->min_silence, r.min_silence) ||
        !to_samples(c->pad, r.pad) || !to_samples(c->min_silence_at_max, r.min_silence_at_max))
        return 1;
    if (std::isinf(c->max_speech)) {
        r.max_speech = INT64_MAX;
    } else {
        int64_t m;
        if (!to_samples(c->max_speech, m)) return 1;
        const __int128 raw = (__int128)m - kChunk - 2 * (__int128)r.pad;
        if (raw < (__int128)INT64_MIN) return 1;   // Swift's subtraction traps
        r.max_speech = raw > 0 ? (int64_t)raw : 0;
    }
    if (c->has_negative) {
        const float sum = c->negative + c->offset;
        r.threshold = smin(1.0f, sum);
        r.negative = c->negative;
    } else {
        r.threshold = c->default_threshold;
        const float diff = r.threshold - c->offset;
        r.negative = smax(diff, 0.01f);
    }
    r.split = c->split;
    r.use_max = c->use_max != 0;
    *out = r;
    return 0;
}

// processChunk's model input [context | chunk padded or truncated to 4096] and the next context
void oracle_vad_model_input(const float *context, const float *chunk, int64_t n, float *input, float *next_context) {
    std::vector<float> processed(chunk, chunk + n);
    if ((int64_t)processed.size() < kChunk) {
        const float last = processed.empty() ? 0.0f : processed.back();
        processed.resize(kChunk, last);
    } else {
        processed.resize(kChunk);
    }
    for (int k = 0; k < kContext; ++k) input[k] = context[k];
    for (int k = 0; k < kChunk; ++k) input[kContext + k] = processed[(size_t)k];
    for (int k = 0; k < kContext; ++k) next_context[k] = processed[(size_t)(kChunk - kContext + k)];
}

// streamingStateMachine: state = {processedSamples, triggered, tempEndSample (-1 nil)}; returns the event kind (0 none,
// 1 start, 2 end) and its sample in *sample (-1 none)
int oracle_vad_stream_step(int64_t *state, float probability, int64_t chunk_count, const Resolved *r,
                           int64_t *sample) {
    int64_t processed = state[0] + chunk_count;
    bool triggered = state[1] != 0;
    bool has_temp = state[2] >= 0;
    int64_t temp = state[2];
    int kind = 0;
    *sample = -1;
    if (probability >= r->threshold) {
        has_temp = false;
        if (!triggered) {
            triggered = true;
            kind = 1;
            *sample = smax<int64_t>(0, processed - r->pad - chunk_count);
        }
    } else if (probability < r->negative && triggered) {
        if (!has_temp) {
            has_temp = true;
            temp = processed;
        }
        if (processed - temp >= r->min_silence) {
            kind = 2;
            *sample = smax<int64_t>(0, temp + r->pad - chunk_count);
            triggered = false;
            has_temp = false;
        }
    }
    state[0] = processed;
    state[1] = triggered;
    state[2] = has_temp ? temp : -1;
    return kind;
}

// segmentSpeech(from:totalSamples:config:)'s sample ranges into out (pairs, at most cap); returns their count
int64_t oracle_vad_segment(const float *probs, int64_t count, int64_t total_samples, const Resolved *r, int64_t *out,
                           int64_t cap) {
    struct Candidate {
        int64_t start, duration;
        float min_probability;
    };
    struct Range {
        int64_t start, end;
    };
    if (count == 0 || total_samples <= 0) return 0;
    const int64_t L = total_samples;
    bool triggered = false;
    int64_t current = 0;
    bool has_temp = false, has_min = false;
    int64_t temp_end = 0;
    float temp_min = 0;
    std::vector<Candidate> ends;
    std::vector<Range> speeches;
    auto flush = [&](int64_t end) {
        if (!(end > current)) return;
        if (end - current >= r->min_speech) speeches.push_back(Range{current, smin(end, L)});
    };
    auto longest = [](const std::vector<Candidate> &v) -> const Candidate * {   // Sequence.max(by:): first maximum
        const Candidate *best = nullptr;
        for (const Candidate &c : v)
            if (!best || best->duration < c.duration) best = &c;
        return best;
    };
    for (int64_t index = 0; index < count; ++index) {
        const int64_t frame = index * kChunk;
        const float p = probs[index];
        if (p >= r->threshold) {
            if (has_temp) {
                const int64_t d = frame - temp_end;
                if (d > r->min_silence_at_max) ends.push_back(Candidate{temp_end, d, has_min ? temp_min : 1.0f});
            }
            has_temp = has_min = false;
            if (!triggered) {
                triggered = true;
                current = frame;
                continue;
            }
        }
        if (triggered && r->max_speech < INT64_MAX && frame - current > r->max_speech) {
            bool chosen = false;
            Candidate split{};
            if (!ends.empty()) {
                std::vector<Candidate> below;
                for (const Candidate &c : ends)
                    if (c.min_probability <= r->split) below.push_back(c);
                if (const Candidate *b = longest(below)) {
                    split = *b;
                } else if (r->use_max) {
                    split = *longest(ends);
                } else {
                    split = ends.back();
                }
                chosen = true;
            }
            flush(chosen ? split.start : frame);
            if (chosen) {
                const int64_t next = split.start + split.duration;
                if (next < frame) {
                    current = next;
                    triggered = true;
                } else {
                    triggered = false;
                }
            } else {
                triggered = false;
            }
            ends.clear();
            has_temp = has_min = false;
            if (!triggered) continue;
        }
        if (p < r->negative && triggered) {
            if (!has_temp) {
                has_temp = true;
                temp_end = frame;
            }
            temp_min = has_min ? smin(temp_min, p) : smin(p, p);
            has_min = true;
            if (frame - temp_end >= r->min_silence) {
                flush(temp_end);
                triggered = false;
                has_temp = has_min = false;
                ends.clear();
                continue;
            }
        }
    }
    if (triggered) flush(L);
    std::vector<Range> a = speeches;
    const int64_t pad = r->pad;
    for (size_t i = 0; i < a.size(); ++i) {
        if (i == 0) a[i].start = smax<int64_t>(0, a[i].start - pad);
        if (i + 1 < a.size()) {
            const int64_t silence = a[i + 1].start - a[i].end;
            if (silence < 2 * pad) {
                const int64_t half = silence / 2;
                a[i].end = smin(L, a[i].end + half);
                a[i + 1].start = smax<int64_t>(0, a[i + 1].start - half);
            } else {
                a[i].end = smin(L, a[i].end + pad);
                a[i + 1].start = smax<int64_t>(0, a[i + 1].start - pad);
            }
        } else {
            a[i].end = smin(L, a[i].end + pad);
        }
    }
    int64_t n = 0;
    for (const Range &x : a) {
        const int64_t s = smax<int64_t>(0, smin(x.start, L)), e = smax(s, smin(x.end, L));
        if (e > s) {
            if (n < cap) {
                out[2 * n] = s;
                out[2 * n + 1] = e;
            }
            ++n;
        }
    }
    return n;
}

// One tick of S sessions the way the reference runs them, one after another, for timing the restatement without a
// foreign call per session: session i stages audio[offsets[i] .. offsets[i+1]) into inputs [S x 4160] and hands its
// state to hidden_out / cell_out [S x 128], then commits new_hidden / new_cell and probability[i] through
// streamingStateMachine (events [S x 2]).  states [S x 3] as oracle_vad_stream_step's, contexts [S x 64], hidden and
// cell [S x 128] are each session's carried state.
void oracle_vad_tick(int64_t S, int64_t *states, float *contexts, float *hidden, float *cell, const float *audio,
                     const int64_t *offsets, const float *probability, const float *new_hidden,
                     const float *new_cell, const Resolved *r, float *inputs, float *hidden_out, float *cell_out,
                     int64_t *events) {
    const int kState = 128;
    for (int64_t i = 0; i < S; ++i) {
        float next[kContext];
        const int64_t n = offsets[i + 1] - offsets[i];
        oracle_vad_model_input(contexts + i * kContext, audio + offsets[i], n, inputs + i * (kChunk + kContext), next);
        for (int k = 0; k < kState; ++k) {
            hidden_out[i * kState + k] = hidden[i * kState + k];
            cell_out[i * kState + k] = cell[i * kState + k];
            hidden[i * kState + k] = new_hidden[i * kState + k];
            cell[i * kState + k] = new_cell[i * kState + k];
        }
        for (int k = 0; k < kContext; ++k) contexts[i * kContext + k] = next[k];
        events[2 * i] = oracle_vad_stream_step(states + 3 * i, probability[i], n, r, events + 2 * i + 1);
    }
}

// oracle_vad_segment over many clips, one after another: clip b is probs[offsets[b] .. offsets[b+1]) of totals[b]
// samples; its counts[b] pairs go to out back to back (out holds offsets[clips] pairs); returns the total
int64_t oracle_vad_segment_batch(const float *probs, const int64_t *offsets, int64_t clips, const int64_t *totals,
                                 const Resolved *r, int64_t *out, int64_t *counts) {
    int64_t at = 0;
    for (int64_t b = 0; b < clips; ++b) {
        const int64_t P = offsets[b + 1] - offsets[b];
        counts[b] = oracle_vad_segment(probs + offsets[b], P, totals[b], r, out + 2 * at, P);
        at += counts[b];
    }
    return at;
}

// FsmnVadManager.decide(silence:): (startMs, endMs) pairs into out (at most cap); returns their count
int64_t oracle_fsmn_decide(const float *silence, int64_t T, int64_t *out, int64_t cap) {
    const int window = 20, sil_to_speech = 15, speech_to_sil = 15, max_end_sil = 80, lookback = 20, lookahead = 10,
              max_seg = 6000, frame_ms = 10;
    std::vector<int> win(window, 0);
    int pos = 0, win_sum = 0, cont = 0;
    bool pre = false, in = false;
    int64_t seg_start = 0, n = 0;
    auto close = [&](int64_t frame) {
        if (n < cap) {
            out[2 * n] = seg_start * frame_ms;
            out[2 * n + 1] = frame * frame_ms;
        }
        ++n;
        in = false;
    };
    for (int64_t t = 0; t < T; ++t) {
        const int cur = silence[t] <= 0.2f ? 1 : 0;
        win_sum -= win[pos];
        win_sum += cur;
        win[pos] = cur;
        pos = (pos + 1) % window;
        if (!pre && win_sum >= sil_to_speech) {
            pre = true;
            if (!in) {
                in = true;
                seg_start = smax<int64_t>(0, t - sil_to_speech - lookback);
                cont = 0;
            }
        } else if (pre && win_sum <= speech_to_sil) {
            pre = false;
        }
        if (in && !pre) cont += 1;
        else cont = 0;
        if (in && cont >= max_end_sil) {
            close(t - max_end_sil + lookahead);
        } else if (in && (t - seg_start) >= max_seg) {
            close(t);
            pre = false;
        }
    }
    if (in) close(T);
    return n;
}

} // extern "C"
