"""The C++ oracle (oracle/oracle_online_diar.cpp) against the independent Python restatement
(tests/online_diar_restated.py), bit for bit, on scenarios restated from the reference's SpeakerManagerTests,
SpeakerTests and SpeakerOperationsTests, and on seeded multi-chunk sessions."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import online_diar_restated as P  # noqa: E402
from oracle import oracle_online_diar as O  # noqa: E402

D = 256
NAMES = ["alice", "bob", "carol"]   # named ids: key = index


def sid_of(named, key):
    return "" if named < 0 else NAMES[key] if named else str(key)


def key_of(sid):
    return (1, NAMES.index(sid)) if sid in NAMES else (0, int(sid))


def unit(rng, n):
    x = rng.normal(size=(n, D)).astype(np.float32)
    return (x / np.linalg.norm(x, axis=1, keepdims=True)).astype(np.float32)


class Pair:
    """the oracle session and the restated manager, driven alike"""

    def __init__(self, thr=0.7, min_speech=1.0, min_active=10.0):
        self.r = O.resolved(thr, min_speech, min_active)
        self.o = O.Session()
        self.p = P.SpeakerManager(self.r[0], self.r[1], self.r[2])

    def chunk(self, logits, emb, offset, chunk_size=160000):
        om, on, oa, oi, ov = self.o.chunk(logits, chunk_size, emb, offset, self.r)
        pm, pn, pi, ps = P.chunk(self.p, logits, chunk_size, emb, offset, self.r[3], self.r[2])
        assert om.tobytes() == pm.tobytes() and list(on) == pn
        assert [sid_of(*a) for a in oa] == pi
        assert [(sid_of(*i), v[0], v[1], v[2]) for i, v in zip(oi, ov)] == \
            [(s, np.float32(a), np.float32(b), np.float32(q)) for s, a, b, q in ps]
        assert all(np.float32(v[k]).tobytes() == np.float32(t[k + 1]).tobytes() for v, t in zip(ov, ps) for k in range(3))
        self.same()
        return pi, ps

    def known(self, speakers, mode, preserve=True):
        """speakers: (id, current, raws, duration, update_count, permanent)"""
        sp = np.zeros(len(speakers), O.SPEAKER)
        for i, (sid, _, raws, dur, uc, perm) in enumerate(speakers):
            named, key = key_of(sid)
            sp[i] = (key, 0 if named else key, uc, dur, named, 0 if named else 1, perm, len(raws))
        cur = np.array([s[1] for s in speakers], np.float32).reshape(-1, D)
        raws = np.concatenate([np.asarray(s[2], np.float32).reshape(-1, D) for s in speakers]) if speakers else \
            np.zeros((0, D), np.float32)
        self.o.initialize(sp, cur, raws, {"reset": 0, "merge": 1, "overwrite": 2, "skip": 3}[mode], preserve)
        self.p.initialize_known_speakers([self.p.known(s[0], s[1], s[2], s[3], s[4], bool(s[5])) for s in speakers],
                                         mode, preserve)
        self.same()

    def same(self):
        sp, cur, raws = self.o.read()
        assert self.o.count() == (len(self.p.db), self.p.next_id)
        for i, (sid, s) in enumerate(self.p.db.items()):
            assert sid_of(int(sp[i]["named"]), int(sp[i]["key"])) == sid
            assert cur[i].tobytes() == s.current.tobytes()
            assert np.float32(sp[i]["duration"]).tobytes() == np.float32(s.duration).tobytes()
            assert sp[i]["update_count"] == s.update_count and bool(sp[i]["permanent"]) == s.permanent
            assert sp[i]["raw_count"] == len(s.raws)
            assert raws[i, :len(s.raws)].tobytes() == np.array([r for _, r in s.raws], np.float32).reshape(-1, D).tobytes()


def logits_for(pattern):
    lg = np.zeros((len(pattern), 7), np.float32)
    lg[np.arange(len(pattern)), pattern] = 5.0
    return lg


SOLO0 = [1] * 300 + [0] * 289


def emb_rows(*rows):
    e = np.zeros((3, D), np.float32)
    for i, r in enumerate(rows):
        e[i] = r
    return e


def test_new_and_existing_assignment_fifo_and_update_then_ema():
    rng = np.random.default_rng(1)
    v = unit(rng, 2)
    t = Pair()
    ids, _ = t.chunk(logits_for(SOLO0), emb_rows(v[0] * 3), 0.0)
    assert ids == ["1", "", ""]
    for k in range(55):   # the FIFO reaches 50 and then drops the oldest
        t.chunk(logits_for(SOLO0), emb_rows(v[0] + rng.normal(0, 0.05, D).astype(np.float32)), 10.0 * (k + 1))
    s = t.p.db["1"]
    assert len(s.raws) == 50 and s.update_count == 56
    # updateMainEmbedding appends the raw (recomputing the mean) before the EMA: the other order differs
    e = P.l2_normalize(v[0] + rng.normal(0, 0.05, D).astype(np.float32))
    before = P.Speaker("x", s.current)
    before.current, before.raws = s.current.copy(), list(s.raws)
    ema_first = P.l2_normalize((np.float32(0.9) * before.current + np.float32(0.1) * P.l2_normalize(e)).astype(np.float32))
    t.chunk(logits_for(SOLO0), emb_rows(e), 600.0)
    assert t.p.db["1"].current.tobytes() != ema_first.tobytes()


def test_threshold_boundaries_and_min_duration():
    rng = np.random.default_rng(2)
    v = unit(rng, 1)[0]
    for delta in (-1, 0, 1):
        t = Pair()
        t.chunk(logits_for(SOLO0), emb_rows(v), 0.0)
        q = (v + rng.normal(0, 0.5, D)).astype(np.float32)
        d = P.cosine_distance(P.l2_normalize(q), t.p.db["1"].current)
        t.r[0] = d if delta == 0 else np.nextafter(d, np.float32(np.inf * delta))
        t.p.speaker_threshold = t.r[0]
        ids, _ = t.chunk(logits_for(SOLO0), emb_rows(q), 10.0)
        assert (ids[0] == "1") == (delta > 0)   # strict <
    t = Pair()
    ids, segs = t.chunk(logits_for([1] * 59 + [0] * 530), emb_rows(v), 0.0)   # 0.995625 s < 1.0
    assert ids == ["", "", ""] and segs == []
    ids, segs = t.chunk(logits_for([1] * 60 + [0] * 529), emb_rows(v), 10.0)   # 1.0125 s
    assert ids[0] == "1" and len(segs) == 1


def test_gates_ties_nan_and_short_embeddings():
    rng = np.random.default_rng(3)
    t = Pair(min_speech=0.0)
    lg = logits_for([1] * 10 + [4] * 5 + [2] * 40 + [0] * 534)
    lg[:3, 0] = np.nan
    lg[20:25, 3] = lg[20:25, 2]   # a tie: the lower class wins
    t.chunk(lg, emb_rows(unit(rng, 1)[0], unit(rng, 1)[0]), 0.0)
    short = np.full(D, 0.006, np.float32)   # magnitude 0.096 < 0.1
    t.chunk(logits_for([1] * 300 + [0] * 289), emb_rows(short), 10.0)
    nan = unit(rng, 1)[0]
    nan[7] = np.nan
    t.chunk(logits_for([1] * 300 + [0] * 289), emb_rows(nan), 20.0)
    assert len(t.p.db) <= 2


def test_known_speaker_modes_permanence_merge_and_reset():
    rng = np.random.default_rng(4)
    v = unit(rng, 6)
    raws = rng.normal(size=(70, D)).astype(np.float32)
    t = Pair()
    t.known([("1", v[0], raws[:40], 3.0, 2, 1), ("alice", v[1], raws[40:70], 4.0, 3, 0)], "skip")
    t.known([("1", v[2], [], 1.0, 1, 0), ("alice", v[3], raws[:30], 2.0, 1, 0)], "overwrite", True)
    t.known([("1", v[4], raws[:25], 1.0, 1, 0), ("alice", v[5], raws[30:60], 2.0, 4, 0)], "merge", False)
    t.known([("bob", v[5], [], 1.0, 1, 1)], "reset", True)
    assert list(t.p.db) == ["1", "bob"] and t.p.next_id == 1
    t.known([("carol", v[3], raws[:50], 1.0, 1, 0)], "skip")
    assert t.o.merge((1, 2), (0, 1), True) == t.p.merge("carol", "1", True)   # merge truncates to the newest 50
    t.same()
    assert t.o.merge((1, 1), (0, 1), True) == t.p.merge("bob", "1", True) is False   # a permanent source stays
    assert t.o.remove(1, 1, True) == t.p.remove("bob", True) is False
    assert t.o.set_permanent(0, 1, True) == (t.p.db["1"].__setattr__("permanent", True) or True)
    t.o.reset(True)
    t.p.reset(True)
    t.same()


def test_next_speaker_id_reset_overwrites_an_existing_speaker():
    rng = np.random.default_rng(5)
    v = unit(rng, 3)
    t = Pair()
    t.known([("1", v[0], [], 2.0, 1, 0), ("2", v[1], [], 2.0, 1, 0)], "skip")
    t.known([("alice", v[2], [], 2.0, 1, 0)], "skip")
    assert t.p.next_id == 1
    ids, _ = t.chunk(logits_for(SOLO0), emb_rows(-v[0] - v[1] - v[2]), 0.0)
    assert ids[0] == "1" and list(t.p.db) == ["1", "2", "alice"] and t.p.next_id == 2


def test_upsert_queries_and_mergeable_pairs():
    rng = np.random.default_rng(6)
    v = unit(rng, 4)
    t = Pair()
    for sid, cur, perm in (("7", v[0], 0), ("alice", v[0], 1), ("3", v[1], 0), ("7", v[2] * 2, 1)):
        named, key = key_of(sid)
        sp = np.zeros(1, O.SPEAKER)
        sp[0] = (key, 0 if named else key, 2, 1.5, named, 0 if named else 1, perm, 2)
        rows = rng.normal(size=(2, D)).astype(np.float32)
        t.o.upsert(sp, cur, rows)
        t.p.upsert(sid, cur, 1.5, rows, 2, bool(perm))
        t.same()
    assert t.p.next_id == 8
    q = np.stack([v[0], v[0] * 2, v[3]])
    dist = t.o.query(q)
    for i, e in enumerate(q):
        for j, s in enumerate(t.p.db.values()):
            assert dist[i, j].tobytes() == P.cosine_distance(e, s.current).tobytes()
    thr = t.r[0]
    # "7" (unnormalised v[2] * 2 after its upsert) and "alice" (v[0]): findMatchingSpeakers ties keep database order
    assert t.p.find_matching_speakers(v[0], thr) == sorted(
        [(sid, dist[0, j]) for j, sid in enumerate(t.p.db) if dist[0, j] <= thr], key=lambda h: h[1])
    pairs = t.p.find_mergeable_pairs(np.float32(2.0))
    assert pairs and all(not (t.p.db[a].permanent and t.p.db[b].permanent) for a, b in pairs)


@pytest.mark.parametrize("seed,F,chunk", [(0, 589, 160000), (1, 101, 80000), (2, 589, 320000)])
def test_seeded_sessions(seed, F, chunk):
    rng = np.random.default_rng(seed)
    voices = unit(rng, 5)
    t = Pair(min_speech=0.3)
    for k in range(25):
        classes = np.repeat(rng.integers(0, 7, size=F // 20 + 1), 20)[:F]
        lg = rng.normal(size=(F, 7)).astype(np.float32)
        lg[np.arange(F), classes] += 4
        emb = np.empty((3, D), np.float32)
        for s in range(3):
            kind = rng.integers(0, 8)
            emb[s] = 0 if kind == 0 else voices[rng.integers(0, 5)] if kind == 1 else \
                (voices[rng.integers(0, 5)] + rng.normal(0, 0.4, D).astype(np.float32)) * 2
        t.chunk(lg, emb, 10.0 * k, chunk)
    assert len(t.p.db) >= 2
