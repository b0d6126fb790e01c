"""A literal pure-Python restatement of the reference's VAD logic (Sources/FluidAudio/VAD/), line for line with the
Swift: VadSegmentationConfig's checks and thresholds, streamingStateMachine, detectSpeechSampleRanges with its whole
possibleEnds list, and FsmnVadManager.decide.  Float values are numpy float32, as Swift's Float; sample counts are
Python ints, as Swift's Int.  It holds the C++ oracle to the reference's behaviour in the CPU suite."""
import math

import numpy as np

F = np.float32
CHUNK = 4096
RATE = 16000


def swift_min(x, y):
    return y if y < x else x


def swift_max(x, y):
    return y if y >= x else x


def trunc_div(a, b):
    """Swift's Int division: truncation toward zero"""
    q = abs(a) // abs(b)
    return q if (a >= 0) == (b > 0) else -q


def to_int(x):
    """Int(Double) for a value the reference does not trap on; None where it traps (or beyond 2^62, the library's
    sample-arithmetic bound: 2^62 and above)"""
    if math.isnan(x) or math.isinf(x) or x >= 2.0 ** 62:
        return None
    return int(x)


def resolve(c):
    """the oracle's Config -> dict, or None when refused"""
    d = {k: getattr(c, k) for k, _ in c._fields_}
    if not (d["min_speech_duration"] >= 0 and d["min_silence_duration"] >= 0 and d["max_speech_duration"] > 0 and
            d["speech_padding"] >= 0 and 0 <= F(d["silence_threshold_for_split"]) <= 1 and
            F(d["negative_threshold_offset"]) >= 0 and d["min_silence_at_max_speech"] >= 0):
        return None
    if d["has_negative_threshold"] and not (0 <= F(d["negative_threshold"]) <= 1):
        return None
    r = {}
    for key, name in (("min_speech", "min_speech_duration"), ("min_silence", "min_silence_duration"),
                      ("pad", "speech_padding"), ("min_silence_at_max", "min_silence_at_max_speech")):
        r[key] = to_int(d[name] * float(RATE))
        if r[key] is None:
            return None
    if math.isinf(d["max_speech_duration"]):
        r["max_speech"] = 2 ** 63 - 1
    else:
        m = to_int(d["max_speech_duration"] * float(RATE))
        if m is None:
            return None
        raw = m - CHUNK - 2 * r["pad"]
        if raw < -2 ** 63:   # Swift's subtraction traps
            return None
        r["max_speech"] = max(0, raw)
    off = F(d["negative_threshold_offset"])
    if d["has_negative_threshold"]:
        neg = F(d["negative_threshold"])
        r["threshold"] = swift_min(F(1.0), F(neg + off))
        r["negative"] = neg
    else:
        r["threshold"] = F(d["default_threshold"])
        r["negative"] = swift_max(F(r["threshold"] - off), F(0.01))
    r["split"] = F(d["silence_threshold_for_split"])
    r["use_max"] = bool(d["use_max_possible_silence_at_max_speech"])
    return r


class StreamState:
    def __init__(self):
        self.processed, self.triggered, self.temp_end = 0, False, None


def stream_step(s, probability, chunk_count, r):
    """streamingStateMachine: (kind, sample), kind 0 none (sample -1), 1 start, 2 end"""
    p = F(probability)
    s.processed += chunk_count
    if p >= r["threshold"]:
        s.temp_end = None
        if not s.triggered:
            s.triggered = True
            return 1, max(0, s.processed - r["pad"] - chunk_count)
    elif p < r["negative"] and s.triggered:
        if s.temp_end is None:
            s.temp_end = s.processed
        if s.processed - s.temp_end >= r["min_silence"]:
            end = max(0, s.temp_end + r["pad"] - chunk_count)
            s.triggered = False
            s.temp_end = None
            return 2, end
    return 0, -1


def _max_by_duration(cands):
    """Sequence.max(by: { $0.duration < $1.duration }): the first of equal maxima"""
    best = None
    for c in cands:
        if best is None or best[1] < c[1]:
            best = c
    return best


def segment(probabilities, total_samples, r):
    """segmentSpeech(from:totalSamples:config:) as [(start, end)] samples"""
    probs = [F(p) for p in probabilities]
    if not probs or total_samples <= 0:
        return []
    L = total_samples
    triggered, current, temp_end, temp_min = False, 0, None, None
    possible_ends, speeches = [], []

    def flush(end):
        if not end > current:
            return
        if end - current >= r["min_speech"]:
            speeches.append([current, min(end, L)])

    for index, prob in enumerate(probs):
        frame = index * CHUNK
        if prob >= r["threshold"]:
            if temp_end is not None:
                d = frame - temp_end
                if d > r["min_silence_at_max"]:
                    possible_ends.append((temp_end, d, temp_min if temp_min is not None else F(1.0)))
            temp_end, temp_min = None, None
            if not triggered:
                triggered, current = True, frame
                continue
        if triggered and r["max_speech"] < 2 ** 63 - 1:
            if frame - current > r["max_speech"]:
                chosen = None
                if possible_ends:
                    below = _max_by_duration([c for c in possible_ends if c[2] <= r["split"]])
                    if below is not None:
                        chosen = below
                    elif r["use_max"]:
                        chosen = _max_by_duration(possible_ends)
                    else:
                        chosen = possible_ends[-1]
                flush(chosen[0] if chosen is not None else frame)
                if chosen is not None:
                    new_start = chosen[0] + chosen[1]
                    if new_start < frame:
                        current, triggered = new_start, True
                    else:
                        triggered = False
                else:
                    triggered = False
                possible_ends = []
                temp_end, temp_min = None, None
                if not triggered:
                    continue
        if prob < r["negative"] and triggered:
            if temp_end is None:
                temp_end = frame
            temp_min = swift_min(temp_min if temp_min is not None else prob, prob)
            if frame - temp_end >= r["min_silence"]:
                flush(temp_end)
                triggered, temp_end, temp_min, possible_ends = False, None, None, []
                continue
    if triggered:
        flush(L)
    if not speeches:
        return []
    pad = r["pad"]
    a = [list(s) for s in speeches]
    for i in range(len(a)):
        if i == 0:
            a[i][0] = max(0, a[i][0] - pad)
        if i < len(a) - 1:
            silence = a[i + 1][0] - a[i][1]
            if silence < 2 * pad:
                half = trunc_div(silence, 2)
                a[i][1] = min(L, a[i][1] + half)
                a[i + 1][0] = max(0, a[i + 1][0] - half)
            else:
                a[i][1] = min(L, a[i][1] + pad)
                a[i + 1][0] = max(0, a[i + 1][0] - pad)
        else:
            a[i][1] = min(L, a[i][1] + pad)
    out = []
    for s, e in a:
        s2 = max(0, min(s, L))
        e2 = max(s2, min(e, L))
        if e2 > s2:
            out.append((s2, e2))
    return out


def fsmn_decide(silence):
    """FsmnVadManager.decide(silence:) as [(startMs, endMs)]"""
    win = [0] * 20
    pos = win_sum = 0
    pre = in_seg = False
    seg_start = cont = 0
    segs = []
    T = len(silence)
    for t in range(T):
        cur = 1 if F(silence[t]) <= F(0.2) else 0
        win_sum -= win[pos]
        win_sum += cur
        win[pos] = cur
        pos = (pos + 1) % 20
        if not pre and win_sum >= 15:
            pre = True
            if not in_seg:
                in_seg = True
                seg_start = max(0, t - 15 - 20)
                cont = 0
        elif pre and win_sum <= 15:
            pre = False
        cont = cont + 1 if in_seg and not pre else 0
        if in_seg and cont >= 80:
            segs.append((seg_start * 10, (t - 80 + 10) * 10))
            in_seg = False
        elif in_seg and t - seg_start >= 6000:
            segs.append((seg_start * 10, t * 10))
            in_seg = False
            pre = False
    if in_seg:
        segs.append((seg_start * 10, T * 10))
    return segs


def make_vad_results(pattern):
    """makeVadResults (TestHelpers/VadTestHelpers.swift): ([probability], totalSamples) of 256 ms chunks, 0.95 for
    active runs and 0.05 for silent ones; a run of s seconds is (s / 0.256).rounded() chunks"""
    chunk_duration = CHUNK / float(RATE)
    probs = []
    for active, seconds in pattern:
        x = seconds / chunk_duration
        f = math.floor(abs(x))
        n = max(0, int(math.copysign(f + 1 if abs(x) - f >= 0.5 else f, x)))
        probs += [F(0.95) if active else F(0.05)] * n
    return np.array(probs, np.float32), len(probs) * CHUNK
