"""A literal Python restatement of streaming speaker tracking, written from the Swift source and independent of the C++
oracle: SpeakerManager (Clustering/SpeakerManager.swift), Speaker and RawEmbedding (SpeakerTypes.swift),
SpeakerUtilities.cosineDistance (SpeakerOperations.swift), VDSPOperations.l2Normalize, AudioValidation and
DiarizerManager's chunk step and segments (Core/DiarizerManager.swift).  numpy float32 scalars and arrays round every
operation, as Swift's Float does.  The reference's open points take the library's pins: the Dictionary is a list in
insertion order, Date() timestamps are a counter, and vDSP_dotpr / vDSP_svesq reduce in the documented order (32 left
folds over elements l, l + 32, ..., then an xor butterfly at 16, 8, 4, 2, 1)."""
from __future__ import annotations

import math

import numpy as np

f32 = np.float32
LANE = np.arange(32)


def vdsp_dot(a, b):
    p = (np.asarray(a, f32) * np.asarray(b, f32)).astype(f32)
    s = p[:32].copy()
    for k in range(1, 8):
        s = (s + p[32 * k:32 * k + 32]).astype(f32)
    for o in (16, 8, 4, 2, 1):
        s = (s + s[LANE ^ o]).astype(f32)
    return f32(s[0])


def swift_max(x, y):
    return y if y >= x else x


def swift_min(x, y):
    return y if y < x else x


def l2_normalize(x):
    x = np.asarray(x, f32)
    norm = swift_max(f32(np.sqrt(vdsp_dot(x, x))), f32(1e-12))
    scale = f32(f32(1) / norm)
    return (x * scale).astype(f32)


def cosine_distance(a, b):
    dot, sa, sb = vdsp_dot(a, b), vdsp_dot(a, a), vdsp_dot(b, b)
    if not (sa > 0 and sb > 0):
        return f32(np.inf)
    if abs(f32(sa - f32(1))) <= f32(1e-3) and abs(f32(sb - f32(1))) <= f32(1e-3):
        sim = dot
    else:
        ma, mb = f32(np.sqrt(sa)), f32(np.sqrt(sb))
        if not (ma > 0 and mb > 0):
            return f32(np.inf)
        sim = f32(dot / f32(ma * mb))
    return f32(f32(1) - swift_min(swift_max(sim, f32(-1)), f32(1)))


def validate_embedding(e):
    if not all(math.isfinite(float(v)) for v in e):
        return False
    acc = f32(0)
    for v in np.asarray(e, f32):
        acc = f32(acc + f32(v * v))
    return f32(np.sqrt(acc)) > f32(0.1)


class Speaker:
    def __init__(self, sid, current, duration=0.0, permanent=False):
        self.id = sid
        self.current = l2_normalize(current)
        self.duration = f32(duration)
        self.update_count = 1
        self.raws = []   # (timestamp, row)
        self.permanent = permanent

    def recalculate(self):
        if not self.raws:
            return
        avg = np.zeros(256, f32)
        for _, r in self.raws:
            avg = (avg + r).astype(f32)
        avg = (avg / f32(len(self.raws))).astype(f32)
        self.current = l2_normalize(avg)

    def add_raw(self, ts, row):
        if not vdsp_dot(row, row) > f32(0.01):
            return
        if len(self.raws) >= 50:
            self.raws.pop(0)
        self.raws.append((ts, row))
        self.recalculate()

    def update_main(self, duration, e, ts):
        if not vdsp_dot(e, e) > f32(0.01):
            return
        ne = l2_normalize(e)
        self.add_raw(ts, l2_normalize(ne))   # the raw goes in (and the mean is recomputed) before the EMA
        alpha = f32(0.9)
        self.current = l2_normalize((alpha * self.current + f32(f32(1) - alpha) * ne).astype(f32))
        self.duration = f32(self.duration + duration)
        self.update_count += 1

    def merge_with(self, other):
        all_ = self.raws + other.raws
        if len(all_) > 50:
            all_ = sorted(all_, key=lambda t: -t[0])[:50]
        self.raws = all_
        self.duration = f32(self.duration + other.duration)
        self.recalculate()
        self.update_count += other.update_count


def swift_int(s):
    import re
    if not re.fullmatch(r"[+-]?[0-9]+", s):
        return None
    v = int(s)
    return v if -(1 << 63) <= v < (1 << 63) else None


class SpeakerManager:
    def __init__(self, speaker_threshold, embedding_threshold, min_speech):
        self.db = {}   # insertion-ordered
        self.next_id = 1
        self.clock = 0
        self.speaker_threshold, self.embedding_threshold, self.min_speech = speaker_threshold, embedding_threshold, min_speech

    def tick(self):
        self.clock += 1
        return self.clock

    def known(self, sid, current, raws=(), duration=0.0, update_count=1, permanent=False):
        s = Speaker(sid, current, duration, permanent)
        s.update_count = update_count
        s.raws = [(self.tick(), l2_normalize(r)) for r in raws]
        return s

    def initialize_known_speakers(self, speakers, mode="skip", preserve=True):
        if mode == "reset":
            self.reset(preserve)
        most = 0
        for s in speakers:
            if s.id in self.db:
                old = self.db[s.id]
                if mode == "skip" or (old.permanent and preserve):
                    continue
                if mode == "merge":
                    old.merge_with(s)
                else:
                    self.db[s.id] = s
            else:
                self.db[s.id] = s
            v = swift_int(s.id)
            if v is not None:
                most = max(most, v)
        self.next_id = most + 1

    def closest(self, e):
        best, at = f32(np.inf), None
        for sid, s in self.db.items():
            d = cosine_distance(e, s.current)
            if d < best:
                best, at = d, sid
        return at, best

    def assign_speaker(self, e, duration):
        n = l2_normalize(e)
        sid, d = self.closest(n)
        if sid is not None and d < self.speaker_threshold:
            s = self.db[sid]
            if d < self.embedding_threshold:
                if vdsp_dot(n, n) > f32(0.01):
                    s.update_main(duration, n, self.tick())
            else:
                s.duration = f32(s.duration + duration)
            return sid
        if not duration >= self.min_speech:
            return None
        ne = l2_normalize(n)
        new = str(self.next_id)
        self.next_id += 1
        sp = Speaker(new, ne, duration)
        sp.add_raw(self.tick(), l2_normalize(ne))
        self.db[new] = sp   # an existing id keeps its place
        return new

    def upsert(self, sid, current, duration, raws=(), update_count=1, permanent=False):
        rows = [(self.tick(), l2_normalize(r)) for r in raws]
        if sid in self.db:
            s = self.db[sid]
            s.current = np.asarray(current, f32).copy()
            s.duration, s.raws, s.update_count = f32(duration), rows, update_count
            if permanent:
                s.permanent = True
            return
        s = Speaker(sid, current, duration, permanent)
        s.raws, s.update_count = rows, update_count
        self.db[sid] = s
        v = swift_int(sid)
        if v is not None:
            self.next_id = max(self.next_id, v + 1)

    def remove(self, sid, keep=True):
        if sid not in self.db or (keep and self.db[sid].permanent):
            return False
        del self.db[sid]
        return True

    def merge(self, src, dst, stop=True):
        if src == dst or src not in self.db or dst not in self.db or (stop and self.db[src].permanent):
            return False
        self.db[dst].merge_with(self.db[src])
        del self.db[src]
        return True

    def reset(self, keep=False):
        if not keep:
            self.db, self.next_id = {}, 1
            return
        self.db = {k: v for k, v in self.db.items() if v.permanent}
        most = 0
        for k in self.db:
            v = swift_int(k)
            if v is not None:
                most = max(most, v)
        self.next_id = most + 1

    def find_speaker(self, e, threshold):
        sid, d = self.closest(e)
        return (sid, d) if sid is not None and d <= threshold else (None, f32(np.inf))

    def find_matching_speakers(self, e, threshold):
        hits = [(sid, cosine_distance(e, s.current)) for sid, s in self.db.items()]
        return sorted([h for h in hits if h[1] <= threshold], key=lambda h: h[1])

    def find_mergeable_pairs(self, threshold, exclude_both_permanent=True):
        ids, pairs = list(self.db), []
        for i in range(len(ids)):
            for j in range(i + 1, len(ids)):
                a, b = self.db[ids[i]], self.db[ids[j]]
                if exclude_both_permanent and a.permanent and b.permanent:
                    continue
                if not cosine_distance(a.current, b.current) < threshold:
                    continue
                pairs.append((b.id, a.id) if not b.permanent else (a.id, b.id))
        return pairs


POWERSET = [[], [0], [1], [2], [0, 1], [0, 2], [1, 2]]


def chunk(mgr, logits, chunk_size, emb, offset, min_active, min_speech):
    """processChunkWithSpeakerTracking after the two models: (masks, need, ids, segments)"""
    F = len(logits)
    bin_ = np.zeros((F, 3), f32)
    for f in range(F):
        m, mi = logits[f][0], 0
        for c in range(1, 7):
            if logits[f][c] > m:
                m, mi = logits[f][c], c
        for s in POWERSET[mi]:
            bin_[f, s] = 1
    masks = [[bin_[f, s] * (f32(1) if bin_[f].sum() < 2 else f32(0)) for f in range(F)] for s in range(3)]
    nm = min((F * chunk_size + 80000) // 160000, F)
    rows = np.array([[masks[s][f % nm] if nm > 0 else 0 for f in range(F)] for s in range(3)], f32)
    need = [int(not sum(masks[s]) < min_active) for s in range(3)]
    embs = [np.asarray(emb[s], f32) if need[s] else np.zeros(256, f32) for s in range(3)]
    activity = [f32(bin_[:, s].sum()) for s in range(3)]
    ids = []
    for s in range(3):
        if activity[s] > min_active and validate_embedding(embs[s]):
            ids.append(mgr.assign_speaker(embs[s], f32(activity[s] * f32(0.016875))) or "")
        else:
            ids.append("")
    segs = []
    for s in range(3):
        if activity[s] < min_active:
            continue
        quality = swift_min(f32(1), f32(f32(np.sqrt(vdsp_dot(embs[s], embs[s]))) / f32(10)))

        def emit(a, b):
            if not ids[s]:
                return
            t0, t1 = offset + a * 0.016875, offset + b * 0.016875
            if f32(t1 - t0) < min_speech:
                return
            segs.append((ids[s], f32(t0), f32(t1), f32(quality * f32(activity[s] / f32(b - a)))))
        on, start = False, 0
        for f in range(F):
            th = f32(0.3)
            for o in range(3):
                if o != s and bin_[f, o] > f32(0.3):
                    th = f32(0.15)
                    break
            if bin_[f, s] > th and not on:
                on, start = True, f
            elif bin_[f, s] <= th and on:
                emit(start, f)
                on = False
        if on:
            emit(start, F)
    segs.sort(key=lambda t: t[1])   # stable: equal starts keep local-speaker order
    return rows, need, ids, segs
