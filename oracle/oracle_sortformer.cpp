// ORACLE — TEST INFRASTRUCTURE ONLY.  Not part of the shipped product path.
//
// Sequential CPU restatement of Sortformer's streaming state update, written from the Swift sources (paths under
// Sources/FluidAudio/Diarizer/Sortformer):
//   SortformerTypes.swift:219-255, 270-327    configuration clamps, SortformerStreamingState
//   SortformerStateUpdater.swift:31-578       streamingUpdate, updateSilenceProfile, compressSpkcache and its helpers
// The state is held as the reference holds it (growing arrays, optional prediction arrays), and both top-k selections
// are the reference's insertion sorts as written, so this file shares nothing with the GPU's rank counting.
// vForce.log / log1p (Accelerate, closed) are computed as (float)log((double)x) / (float)log1p((double)x).
// Compiled with -O2 -ffp-contract=off on baseline x86-64: every float32 operation is rounded as written.
//
// C interface (one session per handle):
//   oracle_sf_create(ints[7], floats[6]) -> handle   ints: chunkLen, left, right, fifoLen, spkcacheLen, period, sil
//   oracle_sf_destroy(h)
//   oracle_sf_config(h, ints[7])                       the clamped configuration
//   oracle_sf_update(h, chunk, chunk_count, preds, preds_count, lc, rc, confirmed, tentative, counts[2]) -> 0 ok,
//                    1 insufficientPredsLength, 2 insufficientChunkLength
//   oracle_sf_lengths(h, out[5])                       spkcacheLength, fifoLength, spkcachePreds?, fifoPreds?, silence count
//   oracle_sf_state(h, spkcache, spkcache_preds, fifo, fifo_preds, mean)
//   oracle_sf_last_pop(h, embs, preds) -> rows the last update popped into the silence profile and the cache
//   oracle_sf_last_compression(h, preds, scores, disabled_scores, strong, weak, indices, is_disabled) -> frame count L
//                    of the last update's compression (0: none); its input spkcachePreds and its scores at each stage
//                    [L x 4], the gathered indices / is_disabled [spkcacheLen]
#include <algorithm>
#include <cmath>
#include <cstring>
#include <limits>
#include <vector>

namespace {

constexpr int kNumSpeakers = 4;
constexpr int kPreEncoderDims = 512;
constexpr int kMaxIndex = 99999;

struct SfConfig {
    int chunkLen, chunkLeftContext, chunkRightContext, fifoLen, spkcacheLen, spkcacheUpdatePeriod, spkcacheSilFramesPerSpk;
    float silenceThreshold, predScoreThreshold, scoresBoostLatest, strongBoostRate, weakBoostRate, minPosScoresRate;
};

struct SfState {
    std::vector<float> spkcache;
    int spkcacheLength = 0;
    bool hasSpkcachePreds = false;
    std::vector<float> spkcachePreds;
    std::vector<float> fifo;
    int fifoLength = 0;
    bool hasFifoPreds = false;
    std::vector<float> fifoPreds;
    std::vector<float> meanSilenceEmbedding = std::vector<float>(kPreEncoderDims, 0.0f);
    long long silenceFrameCount = 0;
};

struct Session {
    SfConfig config;
    SfState state;
    // the last update's compression, stage by stage
    int lastFrames = 0;
    std::vector<float> lastScores, lastDisabled, lastStrong, lastWeak;
    std::vector<int> lastIndices, lastIsDisabled;
    std::vector<float> lastPreds;              // spkcachePreds the compression started from
    std::vector<float> lastPopEmbs, lastPopPreds;   // the rows the last update popped (none: empty)
};

float vlog(float x) { return (float)std::log((double)x); }
float vlog1p(float x) { return (float)std::log1p((double)x); }
float clipf(float x, float lo, float hi) { return x < lo ? lo : (x > hi ? hi : x); }
int swiftInt(float v) { return (int)v; }

std::vector<float> getLogPredScores(const SfConfig &cfg, const std::vector<float> &preds, int frameCount) {
    const int S = kNumSpeakers;
    const float threshold = cfg.predScoreThreshold;
    std::vector<float> scores(frameCount * S), log1P(preds.size());
    for (size_t i = 0; i < (size_t)frameCount * S; ++i)
        scores[i] = vlog(clipf(preds[i], threshold, std::numeric_limits<float>::max()));
    const float hi = 1 - threshold;
    for (size_t i = 0; i < preds.size(); ++i) log1P[i] = vlog1p(-clipf(preds[i], 0, hi));
    for (size_t i = 0; i < scores.size(); ++i) scores[i] = scores[i] - log1P[i];
    const float ln2 = std::log(2.0f);
    for (size_t i = 0; i < scores.size(); ++i) scores[i] = ln2 + scores[i];
    for (int frame = 0; frame < frameCount; ++frame) {
        float sum = 0;
        for (int spk = 0; spk < S; ++spk) sum += log1P[frame * S + spk];
        for (int spk = 0; spk < S; ++spk) scores[frame * S + spk] += sum;
    }
    return scores;
}

std::vector<float> disableLowScores(const std::vector<float> &preds, const std::vector<float> &scores, int frameCount,
                                    int minPosScores) {
    const int S = kNumSpeakers;
    std::vector<float> result = scores;
    int posScoreCounts[kNumSpeakers] = {0, 0, 0, 0};
    for (int frame = 0; frame < frameCount; ++frame)
        for (int spk = 0; spk < S; ++spk) {
            const int index = frame * S + spk;
            if (preds[index] > 0.5f && scores[index] > 0) posScoreCounts[spk] += 1;
        }
    for (int spk = 0; spk < S; ++spk)
        for (int frame = 0; frame < frameCount; ++frame) {
            const int idx = frame * S + spk;
            const float p = preds[idx];
            if (p <= 0.5f) {
                result[idx] = -INFINITY;
                continue;
            }
            if (result[idx] <= 0 && posScoreCounts[spk] >= minPosScores) result[idx] = -INFINITY;
        }
    return result;
}

std::vector<float> boostTopKScores(const std::vector<float> &scores, int frameCount, int k, float scaleFactor) {
    const int S = kNumSpeakers;
    if (frameCount <= 0 || k <= 0) return scores;
    const float boostDelta = -scaleFactor * std::log(0.5f);
    std::vector<float> result = scores;
    const int kEff = std::min(k, frameCount);
    for (int spk = 0; spk < S; ++spk) {
        std::vector<int> topFrames(kEff, 0);
        std::vector<float> topScores(kEff, -std::numeric_limits<float>::max());
        int count = 0;
        for (int frame = 0; frame < frameCount; ++frame) {
            const float v = result[frame * S + spk];
            if (v == -INFINITY) continue;
            if (count < kEff) {
                int pos = count;
                while (pos > 0 && v > topScores[pos - 1]) {
                    topScores[pos] = topScores[pos - 1];
                    topFrames[pos] = topFrames[pos - 1];
                    pos -= 1;
                }
                topScores[pos] = v;
                topFrames[pos] = frame;
                count += 1;
            } else {
                if (v <= topScores[count - 1]) continue;
                int pos = count - 1;
                while (pos > 0 && v > topScores[pos - 1]) {
                    topScores[pos] = topScores[pos - 1];
                    topFrames[pos] = topFrames[pos - 1];
                    pos -= 1;
                }
                topScores[pos] = v;
                topFrames[pos] = frame;
            }
        }
        for (int i = 0; i < count; ++i) result[topFrames[i] * S + spk] += boostDelta;
    }
    return result;
}

void getTopKIndices(const SfConfig &cfg, const std::vector<float> &scores, int frameCount, int k, std::vector<int> &indices,
                    std::vector<int> &isDisabled) {
    const int S = kNumSpeakers;
    const int nFramesNoSil = frameCount - cfg.spkcacheSilFramesPerSpk;
    const int N = frameCount * S;
    indices.assign(k > 0 ? k : 0, kMaxIndex);
    isDisabled.assign(k > 0 ? k : 0, 0);
    if (k <= 0) return;
    const int kEff = std::min(k, N);
    std::vector<int> bestIdx(kEff, 0);
    std::vector<float> bestVal(kEff, -INFINITY);
    int count = 0;
    for (int spk = 0; spk < S; ++spk)
        for (int frame = 0; frame < frameCount; ++frame) {
            const int permutedIdx = spk * frameCount + frame;
            const float v = scores[frame * S + spk];
            if (count < kEff) {
                int pos = count;
                while (pos > 0) {
                    const float pv = bestVal[pos - 1];
                    const int pi = bestIdx[pos - 1];
                    if (v > pv || (v == pv && permutedIdx < pi)) {
                        bestVal[pos] = pv;
                        bestIdx[pos] = pi;
                        pos -= 1;
                    } else {
                        break;
                    }
                }
                bestVal[pos] = v;
                bestIdx[pos] = permutedIdx;
                count += 1;
            } else {
                const float worstV = bestVal[kEff - 1];
                const int worstI = bestIdx[kEff - 1];
                if (v < worstV || (v == worstV && permutedIdx >= worstI)) continue;
                int pos = kEff - 1;
                while (pos > 0) {
                    const float pv = bestVal[pos - 1];
                    const int pi = bestIdx[pos - 1];
                    if (v > pv || (v == pv && permutedIdx < pi)) {
                        bestVal[pos] = pv;
                        bestIdx[pos] = pi;
                        pos -= 1;
                    } else {
                        break;
                    }
                }
                bestVal[pos] = v;
                bestIdx[pos] = permutedIdx;
            }
        }
    for (int i = 0; i < kEff; ++i) indices[i] = bestVal[i] == -INFINITY ? kMaxIndex : bestIdx[i];
    std::sort(indices.begin(), indices.end());
    for (int i = 0; i < k; ++i)
        if (indices[i] == kMaxIndex) isDisabled[i] = 1;
    for (int i = 0; i < k; ++i)
        if (!isDisabled[i]) indices[i] = indices[i] % frameCount;
    for (int i = 0; i < k; ++i)
        if (!isDisabled[i] && indices[i] >= nFramesNoSil) isDisabled[i] = 1;
    for (int i = 0; i < k; ++i)
        if (isDisabled[i]) indices[i] = 0;
}

void updateSilenceProfile(const SfConfig &cfg, SfState &state, const std::vector<float> &embs,
                          const std::vector<float> &preds, int frameCount) {
    for (int frame = 0; frame < frameCount; ++frame) {
        float probSum = 0.0f;
        for (int spk = 0; spk < kNumSpeakers; ++spk) {
            const size_t idx = (size_t)frame * kNumSpeakers + spk;
            if (idx < preds.size()) probSum += preds[idx];
        }
        if (probSum < cfg.silenceThreshold) {
            const float n = (float)state.silenceFrameCount;
            const float newN = n + 1.0f;
            for (int d = 0; d < kPreEncoderDims; ++d) {
                const size_t embIdx = (size_t)frame * kPreEncoderDims + d;
                if (embIdx < embs.size()) {
                    const float oldMean = state.meanSilenceEmbedding[d];
                    const float newVal = embs[embIdx];
                    state.meanSilenceEmbedding[d] = (oldMean * n + newVal) / newN;
                }
            }
            state.silenceFrameCount += 1;
        }
    }
}

void compressSpkcache(Session &s) {
    SfState &state = s.state;
    const SfConfig &cfg = s.config;
    if (!state.hasSpkcachePreds) return;
    const std::vector<float> spkcachePreds = state.spkcachePreds;
    s.lastPreds = spkcachePreds;
    const int spkcacheCapacity = cfg.spkcacheLen, sil = cfg.spkcacheSilFramesPerSpk;
    const int currentLength = state.spkcacheLength;
    const int spkcacheLenPerSpk = spkcacheCapacity / kNumSpeakers - sil;
    const int strongBoostPerSpk = swiftInt((float)spkcacheLenPerSpk * cfg.strongBoostRate);
    const int weakBoostPerSpk = swiftInt((float)spkcacheLenPerSpk * cfg.weakBoostRate);
    const int minPosScoresPerSpk = swiftInt((float)spkcacheLenPerSpk * cfg.minPosScoresRate);

    std::vector<float> scores = getLogPredScores(cfg, spkcachePreds, currentLength);
    s.lastScores = scores;
    scores = disableLowScores(spkcachePreds, scores, currentLength, minPosScoresPerSpk);
    if (currentLength > spkcacheCapacity)
        for (int frame = spkcacheCapacity; frame < currentLength; ++frame)
            for (int spk = 0; spk < kNumSpeakers; ++spk) scores[frame * kNumSpeakers + spk] += cfg.scoresBoostLatest;
    s.lastDisabled = scores;
    scores = boostTopKScores(scores, currentLength, strongBoostPerSpk, 2.0f);
    s.lastStrong = scores;
    scores = boostTopKScores(scores, currentLength, weakBoostPerSpk, 1.0f);
    s.lastWeak = scores;
    const int totalFrames = currentLength + sil;
    for (int i = 0; i < sil * kNumSpeakers; ++i) scores.push_back(INFINITY);
    std::vector<int> topKIndices, isDisabled;
    getTopKIndices(cfg, scores, totalFrames, spkcacheCapacity, topKIndices, isDisabled);
    s.lastIndices = topKIndices;
    s.lastIsDisabled = isDisabled;
    s.lastFrames = currentLength;

    std::vector<float> newSpkcache((size_t)spkcacheCapacity * kPreEncoderDims, 0.0f);
    std::vector<float> newSpkcachePreds((size_t)spkcacheCapacity * kNumSpeakers, 0.0f);
    for (size_t i = 0; i < topKIndices.size(); ++i) {
        const int frameIdx = topKIndices[i];
        if (isDisabled[i]) {
            for (int d = 0; d < kPreEncoderDims; ++d) newSpkcache[i * kPreEncoderDims + d] = state.meanSilenceEmbedding[d];
        } else if (frameIdx < currentLength) {
            for (int d = 0; d < kPreEncoderDims; ++d) {
                const size_t srcIdx = (size_t)frameIdx * kPreEncoderDims + d;
                if (srcIdx < state.spkcache.size()) newSpkcache[i * kPreEncoderDims + d] = state.spkcache[srcIdx];
            }
            for (int k = 0; k < kNumSpeakers; ++k) {
                const size_t srcIdx = (size_t)frameIdx * kNumSpeakers + k;
                if (srcIdx < spkcachePreds.size()) newSpkcachePreds[i * kNumSpeakers + k] = spkcachePreds[srcIdx];
            }
        }
    }
    state.spkcache = newSpkcache;
    state.spkcacheLength = spkcacheCapacity;
    state.spkcachePreds = newSpkcachePreds;
}

int streamingUpdate(Session &s, const std::vector<float> &chunk, const std::vector<float> &preds, int leftContext,
                    int rightContext, std::vector<float> &confirmed, std::vector<float> &tentative) {
    SfState &state = s.state;
    const SfConfig &cfg = s.config;
    const int S = kNumSpeakers, D = kPreEncoderDims;
    const int currentSpkcacheLength = state.spkcacheLength, currentFifoLength = state.fifoLength;
    s.lastFrames = 0;
    s.lastPopEmbs.clear();
    s.lastPopPreds.clear();
    if (currentFifoLength > 0) {
        const size_t start = (size_t)currentSpkcacheLength * S, end = (size_t)(currentSpkcacheLength + currentFifoLength) * S;
        if (end > preds.size()) return 1;
        state.fifoPreds.assign(preds.begin() + start, preds.begin() + end);
        state.hasFifoPreds = true;
    }
    const int lc = leftContext, rc = rightContext;
    const int coreFrames = (int)(chunk.size() / D) - lc - rc;
    const long long embsStart = (long long)lc * D, embsEnd = (long long)(lc + coreFrames) * D;
    if (embsEnd > (long long)chunk.size()) return 2;
    std::vector<float> chunkEmbs(chunk.begin() + embsStart, chunk.begin() + embsEnd);
    const long long chunkStart = currentSpkcacheLength + currentFifoLength + lc, chunkEnd = chunkStart + coreFrames;
    const long long tentativeEnd = (chunkEnd + rc) * S;
    if (tentativeEnd > (long long)preds.size()) return 1;
    std::vector<float> chunkPreds(preds.begin() + chunkStart * S, preds.begin() + chunkEnd * S);
    tentative.assign(preds.begin() + chunkEnd * S, preds.begin() + tentativeEnd);
    confirmed = chunkPreds;

    state.fifo.insert(state.fifo.end(), chunkEmbs.begin(), chunkEmbs.end());
    state.fifoLength += coreFrames;
    if (state.hasFifoPreds) {
        state.fifoPreds.insert(state.fifoPreds.end(), chunkPreds.begin(), chunkPreds.end());
    } else {
        state.fifoPreds = chunkPreds;
        state.hasFifoPreds = true;
    }
    const int contextLength = coreFrames + currentFifoLength;
    if (contextLength > cfg.fifoLen) {
        const std::vector<float> currentFifoPreds = state.fifoPreds;
        int popOutLength = cfg.spkcacheUpdatePeriod;
        popOutLength = std::max(popOutLength, contextLength - cfg.fifoLen);
        popOutLength = std::min(popOutLength, contextLength);
        std::vector<float> popOutEmbs(state.fifo.begin(), state.fifo.begin() + (size_t)popOutLength * D);
        std::vector<float> popOutPreds(currentFifoPreds.begin(), currentFifoPreds.begin() + (size_t)popOutLength * S);
        s.lastPopEmbs = popOutEmbs;
        s.lastPopPreds = popOutPreds;
        updateSilenceProfile(cfg, state, popOutEmbs, popOutPreds, popOutLength);
        state.fifo.erase(state.fifo.begin(), state.fifo.begin() + (size_t)popOutLength * D);
        state.fifoLength -= popOutLength;
        state.fifoPreds.erase(state.fifoPreds.begin(), state.fifoPreds.begin() + (size_t)popOutLength * S);
        state.spkcache.insert(state.spkcache.end(), popOutEmbs.begin(), popOutEmbs.end());
        state.spkcacheLength += popOutLength;
        if (state.hasSpkcachePreds) state.spkcachePreds.insert(state.spkcachePreds.end(), popOutPreds.begin(), popOutPreds.end());
        if (state.spkcacheLength > cfg.spkcacheLen) {
            if (!state.hasSpkcachePreds) {
                if (currentSpkcacheLength > 0) {
                    state.spkcachePreds.assign(preds.begin(), preds.begin() + (size_t)currentSpkcacheLength * S);
                    state.spkcachePreds.insert(state.spkcachePreds.end(), popOutPreds.begin(), popOutPreds.end());
                } else {
                    state.spkcachePreds = popOutPreds;
                }
                state.hasSpkcachePreds = true;
            }
            compressSpkcache(s);
        }
    }
    return 0;
}

void copy_out(float *dst, const std::vector<float> &v) {
    if (dst && !v.empty()) std::memcpy(dst, v.data(), v.size() * sizeof(float));
}

} // namespace

extern "C" {

void *oracle_sf_create(const int *ints, const float *floats) {
    auto *s = new Session();
    SfConfig &c = s->config;
    // SortformerConfig.init (SortformerTypes.swift:219-255)
    c.chunkLen = std::max(1, ints[0]);
    c.chunkLeftContext = ints[1];
    c.chunkRightContext = ints[2];
    c.fifoLen = ints[3];
    c.spkcacheSilFramesPerSpk = ints[6];
    c.silenceThreshold = floats[0];
    c.predScoreThreshold = floats[1];
    c.scoresBoostLatest = floats[2];
    c.strongBoostRate = floats[3];
    c.weakBoostRate = floats[4];
    c.minPosScoresRate = floats[5];
    c.spkcacheLen = std::max(ints[4], (1 + c.spkcacheSilFramesPerSpk) * kNumSpeakers);
    c.spkcacheUpdatePeriod = std::max(std::min(ints[5], c.fifoLen + c.chunkLen), c.chunkLen);
    return s;
}

void oracle_sf_destroy(void *h) { delete static_cast<Session *>(h); }

void oracle_sf_config(void *h, int *ints) {
    const SfConfig &c = static_cast<Session *>(h)->config;
    const int v[7] = {c.chunkLen, c.chunkLeftContext, c.chunkRightContext, c.fifoLen, c.spkcacheLen,
                      c.spkcacheUpdatePeriod, c.spkcacheSilFramesPerSpk};
    std::memcpy(ints, v, sizeof(v));
}

int oracle_sf_update(void *h, const float *chunk, long long chunk_count, const float *preds, long long preds_count, int lc,
                     int rc, float *confirmed, float *tentative, long long *counts) {
    auto *s = static_cast<Session *>(h);
    std::vector<float> ch(chunk, chunk + chunk_count), pr(preds, preds + preds_count), conf, tent;
    const int st = streamingUpdate(*s, ch, pr, lc, rc, conf, tent);
    counts[0] = (long long)conf.size();
    counts[1] = (long long)tent.size();
    if (st == 0) {
        copy_out(confirmed, conf);
        copy_out(tentative, tent);
    }
    return st;
}

void oracle_sf_lengths(void *h, long long *out) {
    const SfState &st = static_cast<Session *>(h)->state;
    out[0] = st.spkcacheLength;
    out[1] = st.fifoLength;
    out[2] = st.hasSpkcachePreds;
    out[3] = st.hasFifoPreds;
    out[4] = st.silenceFrameCount;
}

void oracle_sf_state(void *h, float *spkcache, float *spkcache_preds, float *fifo, float *fifo_preds, float *mean) {
    const SfState &st = static_cast<Session *>(h)->state;
    copy_out(spkcache, st.spkcache);
    if (st.hasSpkcachePreds) copy_out(spkcache_preds, st.spkcachePreds);
    copy_out(fifo, st.fifo);
    if (st.hasFifoPreds) copy_out(fifo_preds, st.fifoPreds);
    copy_out(mean, st.meanSilenceEmbedding);
}

int oracle_sf_last_pop(void *h, float *embs, float *preds) {
    const Session &s = *static_cast<Session *>(h);
    copy_out(embs, s.lastPopEmbs);
    copy_out(preds, s.lastPopPreds);
    return (int)(s.lastPopPreds.size() / kNumSpeakers);
}

int oracle_sf_last_compression(void *h, float *preds, float *scores, float *disabled, float *strong, float *weak, int *indices,
                               int *is_disabled) {
    const Session &s = *static_cast<Session *>(h);
    if (s.lastFrames == 0) return 0;
    copy_out(preds, s.lastPreds);
    copy_out(scores, s.lastScores);
    copy_out(disabled, s.lastDisabled);
    copy_out(strong, s.lastStrong);
    copy_out(weak, s.lastWeak);
    if (indices) std::memcpy(indices, s.lastIndices.data(), s.lastIndices.size() * sizeof(int));
    if (is_disabled) std::memcpy(is_disabled, s.lastIsDisabled.data(), s.lastIsDisabled.size() * sizeof(int));
    return s.lastFrames;
}

} // extern "C"
