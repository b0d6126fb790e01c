// ORACLE — TEST INFRASTRUCTURE ONLY.  Not part of the shipped product path.
//
// A sequential CPU restatement of DiarizerTimeline's numeric core (Sources/FluidAudio/Diarizer/DiarizerTimeline.swift),
// one timeline per object: the stored and tentative predictions, the finalized cursor and the per-speaker
// SegmentScratch, driven by addChunk (:827-872), finalize (:883-891), reset (:921-934), rebuild (:945-1003) and the
// scratch clearing of removeSpeaker / upsertSpeaker (:1108-1111, :1134-1136).  updateSegments (:1169-1294) and
// commitSegment (:1297-1336) are stated as the Swift states them; the speakers' segment storage is left to the caller.
//
// Built with the pinned flags (-O2 -ffp-contract=off, baseline x86-64): every float operation is one IEEE single
// operation in the order written.  Swift's Int is int64_t, `.min` is INT64_MIN, and `log` on Float is the correctly
// rounded float32 log of oracle_float.h (the library's definition; DESIGN §4.8).  maxStoredFrames < 0 stands for nil (unlimited).
#include <cmath>
#include <cstdint>
#include <cstring>
#include <vector>

#include "oracle_float.h"

namespace {

struct Segment {   // fa_diarizer_timeline_segment
    int64_t start_frame, end_frame;
    float activity;
    int32_t speaker;
};

struct SegmentScratch {   // fa_diarizer_timeline_scratch
    int64_t startFrame = INT64_MIN, endFrame = INT64_MIN, unmergedStartFrame = INT64_MIN;
    int64_t activeFrameCount = 0, unmergedActiveFrameCount = 0;
    float activitySum = 0, unmergedActivitySum = 0;
    int32_t speaking = 0, hasSegment = 0;
};
static_assert(sizeof(SegmentScratch) == 56, "scratch layout");

struct Config {
    int64_t numSpeakers, onsetPadFrames, offsetPadFrames, minFramesOn, minFramesOff, maxStoredFrames;
    float frameDurationSeconds, onsetThreshold, offsetThreshold;
    bool logits;
};

float swiftMin(float x, float y) { return y < x ? y : x; }
float swiftMax(float x, float y) { return y >= x ? y : x; }

float evaluate(const Config &c, float p) {
    if (!c.logits) return p;
    const float eps = 1e-6f;
    const float clamped = swiftMin(swiftMax(p, eps), 1 - eps);
    return oracle_float::log32(clamped / (1 - clamped));
}

struct Timeline {
    Config config;
    std::vector<float> finalizedPredictions, tentativePredictions;
    int64_t finalizedCursorFrame = 0;
    std::vector<SegmentScratch> scratches;
    std::vector<Segment> *finalizedResult = nullptr, *tentativeResult = nullptr;

    explicit Timeline(const Config &c) : config(c), scratches(c.numSpeakers) {}

    void trimPredictions() {
        if (config.maxStoredFrames < 0) return;
        const int64_t numToRemove = (int64_t)finalizedPredictions.size() - config.maxStoredFrames * config.numSpeakers;
        if (numToRemove > 0) finalizedPredictions.erase(finalizedPredictions.begin(), finalizedPredictions.begin() + numToRemove);
    }

    void commitSegment(SegmentScratch &aux, int64_t slot, bool isFinalized) {
        if (!aux.hasSegment) return;
        const Segment segment{aux.startFrame, aux.endFrame,
                              aux.activeFrameCount > 0 ? aux.activitySum / (float)aux.activeFrameCount : 0.0f,
                              (int32_t)slot};
        (isFinalized ? finalizedResult : tentativeResult)->push_back(segment);
        aux.hasSegment = 0;
        aux.activitySum = 0;
        aux.activeFrameCount = 0;
    }

    void updateSegments(const std::vector<float> &predictions, bool isFinalized, bool addTrailingTentative) {
        if (predictions.empty() && !addTrailingTentative) return;
        const int64_t frameOffset = finalizedCursorFrame;
        const float onset = config.onsetThreshold, offset = config.offsetThreshold;
        const int64_t padOnset = config.onsetPadFrames, padOffset = config.offsetPadFrames;
        const int64_t minFramesOn = config.minFramesOn, minFramesOff = config.minFramesOff;
        const int64_t speakerCapacity = config.numSpeakers;
        const int64_t numNewFrames = (int64_t)predictions.size() / speakerCapacity;
        const int64_t endFrame = frameOffset + numNewFrames;
        const int64_t pad = padOnset + padOffset;
        const int64_t minSegmentLength = pad + minFramesOn;
        const int64_t finalizedEndFrame = isFinalized ? endFrame - minFramesOff - pad : INT64_MIN;

        for (int64_t speakerIndex = 0; speakerIndex < speakerCapacity; ++speakerIndex) {
            SegmentScratch aux = scratches[speakerIndex];
            for (int64_t i = 0; i < numNewFrames; ++i) {
                const float activity = predictions[i * speakerCapacity + speakerIndex];
                const int64_t frame = frameOffset + i;
                if (aux.speaking) {
                    if (activity >= offset) {
                        aux.unmergedActivitySum += evaluate(config, activity);
                        aux.unmergedActiveFrameCount += 1;
                        continue;
                    }
                    aux.speaking = 0;
                    const int64_t end = frame + padOffset;
                    if (!(end >= aux.unmergedStartFrame + minSegmentLength)) {
                        aux.hasSegment = aux.endFrame >= aux.startFrame + minSegmentLength;
                        continue;
                    }
                    aux.endFrame = end;
                    aux.activitySum += aux.unmergedActivitySum;
                    aux.activeFrameCount += aux.unmergedActiveFrameCount;
                    aux.hasSegment = 1;
                } else if (activity > onset) {
                    const int64_t start = frame - padOnset;
                    aux.speaking = 1;
                    aux.unmergedStartFrame = start;
                    aux.unmergedActivitySum = evaluate(config, activity);
                    aux.unmergedActiveFrameCount = 1;
                    if (!(!aux.hasSegment || start > aux.endFrame + minFramesOff)) {
                        aux.hasSegment = 0;
                        continue;
                    }
                    commitSegment(aux, speakerIndex, isFinalized);
                    aux.startFrame = start;
                }
            }
            if (aux.hasSegment && (!isFinalized || aux.endFrame < finalizedEndFrame))
                commitSegment(aux, speakerIndex, isFinalized && aux.endFrame < finalizedEndFrame);
            if (isFinalized) {
                scratches[speakerIndex] = aux;
                continue;
            }
            if (!(addTrailingTentative && aux.speaking)) continue;
            const int64_t paddedEnd = endFrame + padOffset;
            if (!(paddedEnd >= aux.startFrame + minSegmentLength)) continue;
            aux.hasSegment = 1;
            if (paddedEnd >= aux.unmergedStartFrame + minSegmentLength) {
                aux.endFrame = paddedEnd;
                aux.activitySum += aux.unmergedActivitySum;
                aux.activeFrameCount += aux.unmergedActiveFrameCount;
            }
            commitSegment(aux, speakerIndex, false);
        }
    }

    void addChunk(const std::vector<float> &fin, const std::vector<float> &ten) {
        if (config.maxStoredFrames != 0) {
            finalizedPredictions.insert(finalizedPredictions.end(), fin.begin(), fin.end());
            trimPredictions();
        }
        tentativePredictions = ten;
        updateSegments(fin, true, false);
        finalizedCursorFrame += (int64_t)fin.size() / config.numSpeakers;
        updateSegments(ten, false, true);
    }

    void finalize() {
        finalizedPredictions.insert(finalizedPredictions.end(), tentativePredictions.begin(), tentativePredictions.end());
        finalizedCursorFrame += (int64_t)tentativePredictions.size() / config.numSpeakers;
        tentativePredictions.clear();
        trimPredictions();
    }

    void reset() {
        finalizedPredictions.clear();
        tentativePredictions.clear();
        finalizedCursorFrame = 0;
        scratches.assign(config.numSpeakers, SegmentScratch());
    }

    void rebuild(const std::vector<float> &fin, const std::vector<float> &ten, bool isComplete) {
        reset();
        finalizedPredictions = fin;
        tentativePredictions = ten;
        updateSegments(fin, true, false);
        finalizedCursorFrame = (int64_t)fin.size() / config.numSpeakers;
        updateSegments(ten, false, true);
        if (isComplete) finalize();
        else trimPredictions();
    }
};

std::vector<float> rows(const float *p, int64_t n, int64_t S) { return n > 0 ? std::vector<float>(p, p + n * S) : std::vector<float>(); }

void emit(const std::vector<Segment> &v, Segment *out, int64_t *count) {
    if (!v.empty()) std::memcpy(out, v.data(), v.size() * sizeof(Segment));
    *count = (int64_t)v.size();
}

} // namespace

extern "C" {

// ints = {numSpeakers, onsetPad, offsetPad, minFramesOn, minFramesOff, logits, maxStoredFrames (< 0: unlimited)},
// floats = {frameDurationSeconds, onsetThreshold, offsetThreshold}
void *oracle_tl_create(const int64_t *ints, const float *floats) {
    Config c{ints[0], ints[1], ints[2], ints[3], ints[4], ints[6], floats[0], floats[1], floats[2], ints[5] != 0};
    return new Timeline(c);
}

void oracle_tl_destroy(void *h) { delete static_cast<Timeline *>(h); }

// addChunk (or rebuild when rebuild >= 0, isComplete = rebuild): the segments of each list and their counts[2]
void oracle_tl_push(void *h, const float *fin, int64_t n, const float *ten, int64_t m, int32_t rebuild, Segment *fin_out,
                    Segment *ten_out, int64_t *counts) {
    Timeline &t = *static_cast<Timeline *>(h);
    std::vector<Segment> f, g;
    t.finalizedResult = &f;
    t.tentativeResult = &g;
    const int64_t S = t.config.numSpeakers;
    if (rebuild >= 0) t.rebuild(rows(fin, n, S), rows(ten, m, S), rebuild != 0);
    else t.addChunk(rows(fin, n, S), rows(ten, m, S));
    emit(f, fin_out, counts);
    emit(g, ten_out, counts + 1);
}

void oracle_tl_finalize(void *h) { static_cast<Timeline *>(h)->finalize(); }
void oracle_tl_reset(void *h) { static_cast<Timeline *>(h)->reset(); }
void oracle_tl_clear_speaker(void *h, int64_t k) { static_cast<Timeline *>(h)->scratches[k] = SegmentScratch(); }

// {finalizedCursorFrame, stored rows, tentative rows}
void oracle_tl_lengths(void *h, int64_t *out) {
    const Timeline &t = *static_cast<Timeline *>(h);
    out[0] = t.finalizedCursorFrame;
    out[1] = (int64_t)t.finalizedPredictions.size() / t.config.numSpeakers;
    out[2] = (int64_t)t.tentativePredictions.size() / t.config.numSpeakers;
}

void oracle_tl_state(void *h, float *stored, float *tentative, SegmentScratch *scratch) {
    const Timeline &t = *static_cast<Timeline *>(h);
    if (stored && !t.finalizedPredictions.empty())
        std::memcpy(stored, t.finalizedPredictions.data(), t.finalizedPredictions.size() * sizeof(float));
    if (tentative && !t.tentativePredictions.empty())
        std::memcpy(tentative, t.tentativePredictions.data(), t.tentativePredictions.size() * sizeof(float));
    if (scratch) std::memcpy(scratch, t.scratches.data(), t.scratches.size() * sizeof(SegmentScratch));
}

} // extern "C"
