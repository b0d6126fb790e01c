"""A plain Python restatement of SortformerStateUpdater.swift (Sources/FluidAudio/Diarizer/Sortformer), written from the
Swift alone, to check ``oracle/oracle_sortformer.cpp`` independently (tests/test_sortformer_restated.py).

It is meant to be read beside the Swift: line numbers in the comments are SortformerStateUpdater.swift's unless a
comment names SortformerTypes.swift.  The state is held as the Swift holds it: flat Python lists that grow by
``append(contentsOf:)`` and shrink by ``removeFirst``, and optional prediction arrays (None for nil).  Both top-k
selections are the Swift's insertion sorts as written.  Every arithmetic step is one np.float32 scalar operation in the
Swift's order.  The one deviation is the documented one (DESIGN §4.7): vForce.log / log1p are (float)log((double)x) and
(float)log1p((double)x).
"""
from __future__ import annotations

from types import SimpleNamespace

import numpy as np

F32 = np.float32
S, D = 4, 512                  # numSpeakers, preEncoderDims (SortformerTypes.swift:23-26)
MAX_INDEX = 99999              # maxIndex (SortformerTypes.swift:97)
INF, NEG_INF = F32(np.inf), F32(-np.inf)
GREATEST = F32(np.finfo(np.float32).max)    # Float.greatestFiniteMagnitude
LOGF_2 = F32(np.log(2.0))      # logf(2), correctly rounded
LOGF_HALF = F32(np.log(0.5))   # logf(0.5) = -logf(2)


def vlog(x):
    with np.errstate(all="ignore"):
        return F32(np.log(np.float64(x)))


def vlog1p(x):
    with np.errstate(all="ignore"):
        return F32(np.log1p(np.float64(x)))


def clip(x, lo, hi):
    """vDSP.clip of one element: lo below the range, hi above it, else x itself"""
    return lo if x < lo else (hi if x > hi else x)


def swift_int(v):
    """Int(Float): truncation toward zero (the Swift traps outside Int's range; the configs here stay inside)"""
    return int(v)


class Config:
    """SortformerConfig.init (SortformerTypes.swift:219-255) from fa_sortformer_config field names."""

    def __init__(self, fields):
        get = (lambda k: fields[k]) if isinstance(fields, dict) else (lambda k: getattr(fields, k))
        self.chunkLen = max(1, int(get("chunk_len")))                                        # :239
        self.chunkLeftContext = int(get("chunk_left_context"))
        self.chunkRightContext = int(get("chunk_right_context"))
        self.fifoLen = int(get("fifo_len"))
        self.silenceThreshold = F32(get("silence_threshold"))
        self.spkcacheSilFramesPerSpk = int(get("spkcache_sil_frames_per_spk"))
        self.predScoreThreshold = F32(get("pred_score_threshold"))
        self.scoresBoostLatest = F32(get("scores_boost_latest"))
        self.strongBoostRate = F32(get("strong_boost_rate"))
        self.weakBoostRate = F32(get("weak_boost_rate"))
        self.minPosScoresRate = F32(get("min_pos_scores_rate"))
        self.spkcacheLen = max(int(get("spkcache_len")), (1 + self.spkcacheSilFramesPerSpk) * S)       # :253
        self.spkcacheUpdatePeriod = max(min(int(get("spkcache_update_period")), self.fifoLen + self.chunkLen),
                                        self.chunkLen)                                                  # :254


class InsufficientLength(Exception):
    """SortformerError.insufficientPredsLength / insufficientChunkLength"""

    def __init__(self, kind):
        super().__init__(kind)
        self.kind = kind


class State:
    """SortformerStreamingState.init (SortformerTypes.swift:301-315)"""

    def __init__(self):
        self.spkcache, self.spkcacheLength, self.spkcachePreds = [], 0, None
        self.fifo, self.fifoLength, self.fifoPreds = [], 0, None
        self.meanSilenceEmbedding = [F32(0.0)] * D
        self.silenceFrameCount = 0


class Updater:
    """One session: SortformerStateUpdater over one SortformerStreamingState.  After each update, ``last_pop`` holds
    the popped rows (or None) and ``last_compression`` the compression's stages (or None)."""

    def __init__(self, fields):
        self.config = Config(fields)
        self.state = State()
        self.last_pop = None
        self.last_compression = None

    # ---- streamingUpdate (:31-165)
    def streaming_update(self, chunk, preds, leftContext, rightContext):
        """chunk [rows x 512], preds [pred rows x 4] -> (confirmed [core*4], tentative [rc*4]) as flat lists; raises
        InsufficientLength where the Swift throws, leaving the state as the Swift leaves it."""
        chunk = list(np.asarray(chunk, F32).reshape(-1))
        preds = list(np.asarray(preds, F32).reshape(-1))
        cfg, state = self.config, self.state
        self.last_pop = self.last_compression = None
        fcDModel, numSpeakers = D, S
        fifoCapacity = cfg.fifoLen
        spkcacheCapacity = cfg.spkcacheLen
        currentSpkcacheLength = state.spkcacheLength
        currentFifoLength = state.fifoLength

        if currentFifoLength > 0:                                                      # :47-55
            fifoPredsStart = currentSpkcacheLength * numSpeakers
            fifoPredsEnd = (currentSpkcacheLength + currentFifoLength) * numSpeakers
            if not fifoPredsEnd <= len(preds):
                raise InsufficientLength("preds")
            state.fifoPreds = preds[fifoPredsStart:fifoPredsEnd]

        lc, rc = leftContext, rightContext                                             # :60-71
        coreFrames = len(chunk) // fcDModel - lc - rc
        embsStartIdx = lc * fcDModel
        embsEndIdx = (lc + coreFrames) * fcDModel
        if not embsEndIdx <= len(chunk):
            raise InsufficientLength("chunk")
        chunkEmbs = chunk[embsStartIdx:embsEndIdx]

        chunkStart = currentSpkcacheLength + currentFifoLength + lc                    # :75-94
        chunkEnd = chunkStart + coreFrames
        chunkPredsStart, chunkPredsEnd = chunkStart * numSpeakers, chunkEnd * numSpeakers
        tentativePredsStart, tentativePredsEnd = chunkPredsEnd, (chunkEnd + rc) * numSpeakers
        if not tentativePredsEnd <= len(preds):
            raise InsufficientLength("preds")
        chunkPreds = preds[chunkPredsStart:chunkPredsEnd]
        tentativePreds = preds[tentativePredsStart:tentativePredsEnd]

        state.fifo.extend(chunkEmbs)                                                   # :97-104
        state.fifoLength += coreFrames
        if state.fifoPreds is not None:
            state.fifoPreds.extend(chunkPreds)
        else:
            state.fifoPreds = list(chunkPreds)

        contextLength = coreFrames + currentFifoLength                                 # :108
        if contextLength > fifoCapacity:
            currentFifoPreds = list(state.fifoPreds)
            popOutLength = cfg.spkcacheUpdatePeriod                                    # :119-121
            popOutLength = max(popOutLength, contextLength - fifoCapacity)
            popOutLength = min(popOutLength, contextLength)
            popOutEmbs = state.fifo[:popOutLength * fcDModel]
            popOutPreds = currentFifoPreds[:popOutLength * numSpeakers]
            self.last_pop = (popOutEmbs, popOutPreds)
            self.update_silence_profile(popOutEmbs, popOutPreds, popOutLength)        # :128-133
            del state.fifo[:popOutLength * fcDModel]                                   # :136-138
            state.fifoLength -= popOutLength
            del state.fifoPreds[:popOutLength * numSpeakers]
            state.spkcache.extend(popOutEmbs)                                          # :141-142
            state.spkcacheLength += popOutLength
            if state.spkcachePreds is not None:                                        # :145-147
                state.spkcachePreds.extend(popOutPreds)
            if state.spkcacheLength > spkcacheCapacity:                                # :150-161
                if state.spkcachePreds is None:
                    if currentSpkcacheLength > 0:
                        state.spkcachePreds = preds[:currentSpkcacheLength * numSpeakers] + popOutPreds
                    else:
                        state.spkcachePreds = list(popOutPreds)
                self.compress_spkcache()
        return chunkPreds, tentativePreds

    # ---- updateSilenceProfile (:175-212)
    def update_silence_profile(self, embs, preds, frameCount):
        cfg, state = self.config, self.state
        for frame in range(frameCount):
            probSum = F32(0.0)
            for spk in range(S):
                idx = frame * S + spk
                if idx < len(preds):
                    probSum = probSum + preds[idx]
            if probSum < cfg.silenceThreshold:
                n = F32(state.silenceFrameCount)
                newN = n + F32(1.0)
                for d in range(D):
                    embIdx = frame * D + d
                    if embIdx < len(embs):
                        oldMean = state.meanSilenceEmbedding[d]
                        newVal = embs[embIdx]
                        state.meanSilenceEmbedding[d] = (oldMean * n + newVal) / newN
                state.silenceFrameCount += 1

    # ---- compressSpkcache (:220-305)
    def compress_spkcache(self):
        cfg, state = self.config, self.state
        if state.spkcachePreds is None:
            return
        spkcachePreds = list(state.spkcachePreds)
        spkcacheCapacity = cfg.spkcacheLen
        silFramesPerSpk = cfg.spkcacheSilFramesPerSpk
        currentLength = state.spkcacheLength

        spkcacheLenPerSpk = spkcacheCapacity // S - silFramesPerSpk                    # :229-232
        strongBoostPerSpk = swift_int(F32(spkcacheLenPerSpk) * cfg.strongBoostRate)
        weakBoostPerSpk = swift_int(F32(spkcacheLenPerSpk) * cfg.weakBoostRate)
        minPosScoresPerSpk = swift_int(F32(spkcacheLenPerSpk) * cfg.minPosScoresRate)

        rec = SimpleNamespace(frames=currentLength, preds=list(spkcachePreds), strong_k=strongBoostPerSpk,
                              weak_k=weakBoostPerSpk, min_pos=minPosScoresPerSpk)
        scores = self.get_log_pred_scores(spkcachePreds, currentLength)               # :235
        rec.scores = list(scores)
        scores = self.disable_low_scores(spkcachePreds, scores, currentLength, minPosScoresPerSpk)   # :238-243
        if currentLength > spkcacheCapacity:                                           # :246-252
            for frame in range(spkcacheCapacity, currentLength):
                for spk in range(S):
                    scores[frame * S + spk] = scores[frame * S + spk] + cfg.scoresBoostLatest
        rec.disabled = list(scores)
        scores = self.boost_top_k_scores(scores, currentLength, strongBoostPerSpk, F32(2.0))   # :255
        rec.strong = list(scores)
        scores = self.boost_top_k_scores(scores, currentLength, weakBoostPerSpk, F32(1.0))     # :258
        rec.weak = list(scores)

        totalFrames = currentLength + silFramesPerSpk                                  # :261-264
        for _ in range(silFramesPerSpk * S):
            scores.append(INF)
        topKIndices, isDisabled = self.get_top_k_indices(scores, totalFrames, spkcacheCapacity)   # :267-271
        rec.indices, rec.is_disabled = list(topKIndices), list(isDisabled)

        newSpkcache = [F32(0.0)] * (spkcacheCapacity * D)                              # :274-300
        newSpkcachePreds = [F32(0.0)] * (spkcacheCapacity * S)
        for i, frameIdx in enumerate(topKIndices):
            if isDisabled[i]:
                for d in range(D):
                    newSpkcache[i * D + d] = state.meanSilenceEmbedding[d]
            elif frameIdx < currentLength:
                for d in range(D):
                    srcIdx = frameIdx * D + d
                    if srcIdx < len(state.spkcache):
                        newSpkcache[i * D + d] = state.spkcache[srcIdx]
                for s in range(S):
                    srcIdx = frameIdx * S + s
                    if srcIdx < len(spkcachePreds):
                        newSpkcachePreds[i * S + s] = spkcachePreds[srcIdx]
        state.spkcache = newSpkcache                                                   # :302-304
        state.spkcacheLength = spkcacheCapacity
        state.spkcachePreds = newSpkcachePreds
        self.last_compression = rec

    # ---- getLogPredScores (:311-348)
    def get_log_pred_scores(self, preds, frameCount):
        threshold = self.config.predScoreThreshold
        scores = [F32(0.0)] * (frameCount * S)
        # :320-321 scores <- log(clip(preds, threshold...greatestFiniteMagnitude))
        for i in range(len(scores)):
            scores[i] = vlog(clip(preds[i], threshold, GREATEST))
        # :324-327 log1P <- log1p(-clip(preds, 0...(1 - threshold))); scores <- scores - log1P
        hi = F32(1) - threshold
        log1P = [vlog1p(-clip(p, F32(0), hi)) for p in preds]
        for i in range(len(scores)):
            scores[i] = scores[i] - log1P[i]
        # :330 scores <- logf(2) + scores
        for i in range(len(scores)):
            scores[i] = LOGF_2 + scores[i]
        # :338-343 each frame's scores gain the sum of its log1P, summed in speaker order
        for frame in range(frameCount):
            base = frame * S
            total = F32(0)
            for spk in range(S):
                total = total + log1P[base + spk]
            for spk in range(S):
                scores[base + spk] = scores[base + spk] + total
        return scores

    # ---- disableLowScores (:351-390)
    def disable_low_scores(self, preds, scores, frameCount, minPosScores):
        result = list(scores)
        posScoreCounts = [0] * S
        for frame in range(frameCount):
            for spk in range(S):
                index = frame * S + spk
                if preds[index] > 0.5 and scores[index] > 0:
                    posScoreCounts[spk] += 1
        for spk in range(S):
            for frame in range(frameCount):
                idx = frame * S + spk
                p = preds[idx]
                if p <= 0.5:                                                           # :377-380
                    result[idx] = NEG_INF
                    continue
                if result[idx] <= 0 and posScoreCounts[spk] >= minPosScores:           # :383-385
                    result[idx] = NEG_INF
        return result

    # ---- boostTopKScores (:393-457)
    def boost_top_k_scores(self, scores, frameCount, k, scaleFactor):
        if not (frameCount > 0 and S > 0 and k > 0):                                   # :400
            return scores
        boostDelta = -scaleFactor * LOGF_HALF                                          # :402
        result = list(scores)
        kEff = min(k, frameCount)
        for spk in range(S):
            topFrames = [0] * kEff
            topScores = [-GREATEST] * kEff
            count = 0
            for frame in range(frameCount):
                idx = frame * S + spk
                v = result[idx]
                if v == NEG_INF:                                                       # :419
                    continue
                if count < kEff:                                                       # :421-431
                    pos = count
                    while pos > 0 and v > topScores[pos - 1]:
                        topScores[pos] = topScores[pos - 1]
                        topFrames[pos] = topFrames[pos - 1]
                        pos -= 1
                    topScores[pos] = v
                    topFrames[pos] = frame
                    count += 1
                else:                                                                  # :432-445
                    if v <= topScores[count - 1]:
                        continue
                    pos = count - 1
                    while pos > 0 and v > topScores[pos - 1]:
                        topScores[pos] = topScores[pos - 1]
                        topFrames[pos] = topFrames[pos - 1]
                        pos -= 1
                    topScores[pos] = v
                    topFrames[pos] = frame
            for i in range(count):                                                     # :449-452
                idx = topFrames[i] * S + spk
                result[idx] = result[idx] + boostDelta
        return result

    # ---- getTopKIndices (:465-578)
    def get_top_k_indices(self, scores, frameCount, k):
        silFramesPerSpk = self.config.spkcacheSilFramesPerSpk
        nFramesNoSil = frameCount - silFramesPerSpk
        N = frameCount * S
        if k <= 0:
            return [], []
        kEff = min(k, N)
        bestIdx = [0] * kEff
        bestVal = [NEG_INF] * kEff
        count = 0
        for spk in range(S):                                                           # :494-541
            for frame in range(frameCount):
                permutedIdx = spk * frameCount + frame
                v = scores[frame * S + spk]
                if count < kEff:
                    pos = count
                    while pos > 0:
                        pv, pi = bestVal[pos - 1], bestIdx[pos - 1]
                        if v > pv or (v == pv and permutedIdx < pi):
                            bestVal[pos], bestIdx[pos] = pv, pi
                            pos -= 1
                        else:
                            break
                    bestVal[pos], bestIdx[pos] = v, permutedIdx
                    count += 1
                else:
                    worstV, worstI = bestVal[kEff - 1], bestIdx[kEff - 1]
                    if v < worstV or (v == worstV and permutedIdx >= worstI):
                        continue
                    pos = kEff - 1
                    while pos > 0:
                        pv, pi = bestVal[pos - 1], bestIdx[pos - 1]
                        if v > pv or (v == pv and permutedIdx < pi):
                            bestVal[pos], bestIdx[pos] = pv, pi
                            pos -= 1
                        else:
                            break
                    bestVal[pos], bestIdx[pos] = v, permutedIdx
        topKIndices = [MAX_INDEX] * k                                                  # :544-547
        for i in range(kEff):
            topKIndices[i] = MAX_INDEX if bestVal[i] == NEG_INF else bestIdx[i]
        # :550 topKIndices.sort(): ascending; any sort of these integers gives the same list, insertion sort here
        for i in range(1, k):
            v, j = topKIndices[i], i
            while j > 0 and topKIndices[j - 1] > v:
                topKIndices[j] = topKIndices[j - 1]
                j -= 1
            topKIndices[j] = v
        isDisabled = [False] * k                                                       # :553-558
        for i in range(k):
            if topKIndices[i] == MAX_INDEX:
                isDisabled[i] = True
        for i in range(k):                                                             # :561-563
            if not isDisabled[i]:
                topKIndices[i] = topKIndices[i] % frameCount
        for i in range(k):                                                             # :566-570
            if not isDisabled[i] and topKIndices[i] >= nFramesNoSil:
                isDisabled[i] = True
        for i in range(k):                                                             # :573-575
            if isDisabled[i]:
                topKIndices[i] = 0
        return topKIndices, isDisabled


def frame_scores(preds_row, threshold):
    """getLogPredScores (:311-348) of one frame [4] under ``threshold``: the CPU search for exact-zero scores uses it"""
    u = Updater.__new__(Updater)
    u.config = SimpleNamespace(predScoreThreshold=F32(threshold))
    return u.get_log_pred_scores([F32(p) for p in preds_row], 1)
