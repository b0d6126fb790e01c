"""Diarizer timelines on the CPU: DiarizerTimeline's numeric core (Diarizer/DiarizerTimeline.swift).

* the reference's DiarizerTimelineMergeTests (all five) and the numeric cases of SortformerTimelineTests, with their
  exact numbers, on the oracle (``oracle/oracle_timeline.cpp``) and on a pure-Python restatement below;
* the oracle against that restatement over seeded streams: both activity types, 1 / 4 / 7 / 32 speakers, pads and
  minimum durations, empty and tentative-only pushes, finalize mid-stream, clearing a speaker, maxStoredFrames 0 /
  small / large / unlimited, predictions exactly at the thresholds and NaN;
* ``timeline_core.cuh`` — the arithmetic the kernel runs — compiled for the host (``tests/emul/timeline_emul.cpp``)
  against the oracle bit for bit, segments, activity bits and scratches, push by push;
* the per-push segment bound: never exceeded, and reached exactly by alternating 0/1 input;
* the seconds initialiser's rounding at the .5 boundaries, through the C ABI (no device needed).
"""
import ctypes as C
import math
import os
import subprocess
import zlib

import numpy as np
import pytest

import float_exact
from fluidaudio_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F = np.float32
MIN = -2 ** 63


@pytest.fixture(scope="module")
def O():
    from oracle import oracle_timeline
    oracle_timeline.build()
    oracle_timeline.lib()
    return oracle_timeline


@pytest.fixture(scope="module")
def emul(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("timeline") / "libtimeline_emul.so")
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-fPIC", "-shared", "-o", out,
                           os.path.join(ROOT, "tests", "emul", "timeline_emul.cpp")])
    L = C.CDLL(out)
    L.timeline_emul_push.argtypes = [C.c_void_p] * 4 + [C.c_void_p, C.c_longlong, C.c_void_p, C.c_longlong] + \
        [C.c_void_p] * 4
    L.timeline_emul_push.restype = None
    return L


@pytest.fixture(scope="module")
def lib():
    if not os.path.exists(_lib.LIB_PATH):
        import __graft_entry__
        __graft_entry__.build()
    return _lib.load()


def config(S=4, fd=0.08, onset=0.5, offset=0.5, pad_on=0, pad_off=0, min_on=0, min_off=0, logits=False,
           max_stored=None):
    return dict(num_speakers=S, frame_duration_seconds=fd, onset_threshold=onset, offset_threshold=offset,
                onset_pad_frames=pad_on, offset_pad_frames=pad_off, min_frames_on=min_on, min_frames_off=min_off,
                activity_type=int(logits), max_stored_frames=max_stored)


MERGE = config(S=1, fd=0.1, pad_on=2, pad_off=2, min_on=4, min_off=3)


# ---- an independent restatement in Python, float32 operations one at a time -----------------------------------------
class PyScratch:
    def __init__(self):
        self.speaking = self.has_segment = False
        self.start = self.end = self.unmerged_start = MIN
        self.sum, self.count, self.unmerged_sum, self.unmerged_count = F(0), 0, F(0), 0

    def copy(self):
        s = PyScratch()
        s.__dict__.update(self.__dict__)
        return s

    def record(self):
        return (self.start, self.end, self.unmerged_start, self.count, self.unmerged_count, F(self.sum),
                F(self.unmerged_sum), int(self.speaking), int(self.has_segment))


class PyTimeline:
    def __init__(self, cfg):
        self.c = cfg
        self.S = cfg["num_speakers"]
        self.stored, self.tentative, self.cursor = [], [], 0
        self.scratch = [PyScratch() for _ in range(self.S)]

    def act(self, p):
        if not self.c["activity_type"]:
            return p
        eps = F(1e-6)
        lo = eps if eps >= p else p                     # Swift.max(p, eps) = eps >= p ? eps : p
        hi = F(1) - eps
        c = hi if hi < lo else lo                       # Swift.min(lo, hi) = hi < lo ? hi : lo
        return float_exact.log(F(c / (F(1) - c)))

    def commit(self, a, spk, finalized, out):
        if not a.has_segment:
            return
        act = F(a.sum / F(a.count)) if a.count > 0 else F(0)
        out[0 if finalized else 1].append((a.start, a.end, act, spk))
        a.has_segment, a.sum, a.count = False, F(0), 0

    def update(self, rows, finalized, trailing, out):
        if len(rows) == 0 and not trailing:
            return
        c = self.c
        on, off = F(c["onset_threshold"]), F(c["offset_threshold"])
        pad_on, pad_off = c["onset_pad_frames"], c["offset_pad_frames"]
        n = len(rows)
        end_frame = self.cursor + n
        min_len = pad_on + pad_off + c["min_frames_on"]
        fin_end = end_frame - c["min_frames_off"] - pad_on - pad_off if finalized else MIN
        for k in range(self.S):
            a = self.scratch[k].copy()
            for i in range(n):
                p, frame = F(rows[i][k]), self.cursor + i
                if a.speaking:
                    if p >= off:
                        a.unmerged_sum = F(a.unmerged_sum + self.act(p))
                        a.unmerged_count += 1
                        continue
                    a.speaking = False
                    end = frame + pad_off
                    if not end >= a.unmerged_start + min_len:
                        a.has_segment = a.end >= a.start + min_len
                        continue
                    a.end = end
                    a.sum = F(a.sum + a.unmerged_sum)
                    a.count += a.unmerged_count
                    a.has_segment = True
                elif p > on:
                    start = frame - pad_on
                    a.speaking = True
                    a.unmerged_start, a.unmerged_sum, a.unmerged_count = start, self.act(p), 1
                    if a.has_segment and not start > a.end + c["min_frames_off"]:
                        a.has_segment = False
                        continue
                    self.commit(a, k, finalized, out)
                    a.start = start
            if a.has_segment and (not finalized or a.end < fin_end):
                self.commit(a, k, finalized and a.end < fin_end, out)
            if finalized:
                self.scratch[k] = a
                continue
            if not (trailing and a.speaking):
                continue
            padded = end_frame + pad_off
            if not padded >= a.start + min_len:
                continue
            a.has_segment = True
            if padded >= a.unmerged_start + min_len:
                a.end = padded
                a.sum = F(a.sum + a.unmerged_sum)
                a.count += a.unmerged_count
            self.commit(a, k, False, out)

    def trim(self):
        ms = self.c["max_stored_frames"]
        if ms is not None and len(self.stored) > ms:
            del self.stored[:len(self.stored) - ms]

    def add_chunk(self, fin, ten):
        fin, ten = [list(r) for r in np.asarray(fin, F).reshape(-1, self.S)], \
            [list(r) for r in np.asarray(ten, F).reshape(-1, self.S)]
        if self.c["max_stored_frames"] != 0:
            self.stored += fin
            self.trim()
        self.tentative = ten
        out = ([], [])
        self.update(fin, True, False, out)
        self.cursor += len(fin)
        self.update(ten, False, True, out)
        return out

    def finalize(self):
        self.stored += self.tentative
        self.cursor += len(self.tentative)
        self.tentative = []
        self.trim()

    def clear_speaker(self, k):
        self.scratch[k] = PyScratch()


def records(segs):
    return [(int(s["start_frame"]), int(s["end_frame"]), F(s["activity"]), int(s["speaker"])) for s in segs]


def bits(x):
    return np.asarray(x, F).view(np.uint32)


def same_segments(a, b):
    """(start, end, activity, speaker) lists equal, the activity bit for bit"""
    assert len(a) == len(b), (a, b)
    for x, y in zip(a, b):
        assert x[0] == y[0] and x[1] == y[1] and x[3] == y[3] and bits(x[2]) == bits(y[2]), (x, y)


def same_scratch(rec, py):
    got = tuple(rec[k] for k in rec.dtype.names)
    want = py.record()
    assert got[:5] == want[:5] and got[7:] == want[7:], (got, want)
    assert bits(got[5]) == bits(want[5]) and bits(got[6]) == bits(want[6]), (got, want)


# ---- the reference's tests ------------------------------------------------------------------------------------------
class Both:
    """The oracle and the Python restatement side by side: every push must agree before it is returned."""

    def __init__(self, O, cfg):
        self.o, self.p, self.S = O.Timeline(cfg), PyTimeline(cfg), cfg["num_speakers"]
        self.speakers = {}   # host store of DiarizerSpeaker segments: slot -> ([finalized], [tentative])

    def add_chunk(self, fin, ten=()):
        f, t = self.o.add_chunk(fin, ten)
        pf, pt = self.p.add_chunk(fin, ten)
        same_segments(records(f), pf)
        same_segments(records(t), pt)
        for sp in self.speakers.values():
            sp[1].clear()
        for s in records(f):
            self.speakers.setdefault(s[3], ([], []))[0].append(s)
        for s in records(t):
            self.speakers.setdefault(s[3], ([], []))[1].append(s)
        return records(f), records(t)

    def finalize(self):
        self.o.finalize()
        self.p.finalize()
        for fin, ten in self.speakers.values():
            fin.extend(ten)
            ten.clear()

    def finalized(self, k):
        return self.speakers.get(k, ([], []))[0]


def merge_preds(n, *spans):
    p = np.zeros(n, F)
    for a, b in spans:
        p[a:b + 1] = 0.9
    return p


def test_short_segment_after_small_gap_does_not_drop_prior_segment(O):
    t = Both(O, MERGE)
    t.add_chunk(merge_preds(30, (5, 14), (19, 20)))
    t.finalize()
    assert [(s[0], s[1]) for s in t.finalized(0)] == [(3, 17)]


def test_small_gap_merges_two_long_segments(O):
    t = Both(O, MERGE)
    t.add_chunk(merge_preds(40, (5, 14), (19, 28)))
    t.finalize()
    assert [(s[0], s[1]) for s in t.finalized(0)] == [(3, 31)]


def test_trailing_tentative_short_tail_emits_held_segment_alone(O):
    _, ten = Both(O, MERGE).add_chunk(np.zeros(0, F), merge_preds(22, (5, 14), (19, 21)))
    assert [(s[0], s[1]) for s in ten] == [(3, 17)]
    assert abs(ten[0][2] - 0.9) <= 1e-5


def test_segment_in_buffer_zone_survives_next_chunk(O):
    t = Both(O, MERGE)
    t.add_chunk(merge_preds(22, (5, 14)))
    assert t.o.state().scratch[0]["has_segment"] == 1   # A.endFrame 17 > finalizedEndFrame 15: held
    t.add_chunk(np.zeros(22, F))
    t.finalize()
    assert [(s[0], s[1]) for s in t.finalized(0)] == [(3, 17)]


def test_trailing_tentative_long_tail_emits_merged_span(O):
    _, ten = Both(O, MERGE).add_chunk(np.zeros(0, F), merge_preds(29, (5, 14), (19, 28)))
    assert [(s[0], s[1]) for s in ten] == [(3, 31)]
    assert abs(ten[0][2] - 0.9) <= 1e-5


def test_chunks_accumulate_frames_finalize_and_reset(O):
    t = Both(O, config())
    for _ in range(3):
        t.add_chunk(np.zeros((6, 4), F))
    assert t.o.state().finalized_frames == 18 == t.p.cursor
    t.add_chunk(np.zeros((6, 4), F), np.zeros((4, 4), F))
    st = t.o.state()
    assert (st.finalized_frames, st.tentative.shape[0]) == (24, 4)
    t.finalize()
    st = t.o.state()
    assert (st.finalized_frames, st.tentative.shape[0], st.stored.shape[0]) == (28, 0, 28)
    t.add_chunk(np.full((6, 4), 0.9, F))
    t.o.reset()
    st = t.o.state()
    assert st.finalized_frames == 0 and st.stored.size == 0 and st.tentative.size == 0
    assert all(r["start_frame"] == MIN and not r["speaking"] for r in st.scratch)


def test_segment_activity_excludes_padding_frames(O):
    t = Both(O, config(S=1, pad_on=1, pad_off=2))
    t.add_chunk(np.array([0.0, 0.8, 0.6, 0.0], F))
    t.finalize()
    (s,) = t.finalized(0)
    assert (s[0], s[1]) == (0, 5) and abs(s[2] - 0.7) <= 1e-6


def test_segment_activity_excludes_bridged_gap_frames(O):
    t = Both(O, config(S=1, min_off=1))
    t.add_chunk(np.array([0.9, 0.0, 0.7, 0.7, 0.0], F))
    t.finalize()
    (s,) = t.finalized(0)
    assert (s[0], s[1]) == (0, 4) and abs(s[2] - F(F(F(0.9) + F(0.7)) + F(0.7)) / F(3)) <= 1e-6


def test_probability_access_after_rebuild(O):
    t = O.Timeline(config())
    t.rebuild(np.array([0.1, 0.2, 0.3, 0.4, 0.5, 0.6, 0.7, 0.8], F), is_complete=True)
    st = t.state()
    assert st.stored[0, 0] == F(0.1) and st.stored[0, 3] == F(0.4) and st.stored[1, 0] == F(0.5)
    assert st.finalized_frames == 2   # frame 999 lies outside the stored frames: NaN in the façade


def test_segment_time_conversion():
    from fluidaudio_b200.diarizer_timeline import DiarizerSegment
    s = DiarizerSegment(0, 10, 20, True, 0.08)
    assert abs(s.start_time - 0.8) <= 1e-5 and abs(s.end_time - 1.6) <= 1e-5 and abs(s.duration - 0.8) <= 1e-5
    assert s.length == 10


def half_speaker0(frames, S=4):
    p = np.zeros((frames, S), F)
    p[:frames // 2, 0] = 0.9
    return p


def test_emit_only_updates_equal_storing_updates_across_chunks(O):
    """storeSegments only decides whether the speakers keep the segments: the updates are the same"""
    storing, emitting = Both(O, config()), O.Timeline(config())
    total = 0
    for _ in range(3):
        f, t = storing.add_chunk(half_speaker0(12))
        g, u = emitting.add_chunk(half_speaker0(12))
        same_segments(f, records(g))
        same_segments(t, records(u))
        total += len(f)
    assert total > 0 and storing.speakers


def test_rebuild_equals_reset_push_finalize(O):
    rng = np.random.default_rng(7)
    for cfg in (config(), config(S=3, pad_on=1, pad_off=2, min_on=2, min_off=3, max_stored=9)):
        S = cfg["num_speakers"]
        fin, ten = rng.uniform(size=(40, S)).astype(F), rng.uniform(size=(5, S)).astype(F)
        for complete in (True, False):
            a, b = O.Timeline(cfg), O.Timeline(cfg)
            a.add_chunk(rng.uniform(size=(13, S)).astype(F))
            b.add_chunk(rng.uniform(size=(7, S)).astype(F), rng.uniform(size=(2, S)).astype(F))
            ra = a.rebuild(fin, ten, is_complete=complete)
            b.reset()
            rb = b.add_chunk(fin, ten)
            if complete:
                b.finalize()
            for x, y in zip(ra, rb):
                same_segments(records(x), records(y))
            sa, sb = a.state(), b.state()
            assert sa.finalized_frames == sb.finalized_frames
            assert np.array_equal(sa.stored, sb.stored) and np.array_equal(sa.tentative, sb.tentative)
            assert sa.scratch.tobytes() == sb.scratch.tobytes()


# ---- seeded streams: oracle, Python restatement and the kernel's arithmetic -------------------------------------------
def draw(rng, rows, S, kind):
    if kind == "levels":   # exact thresholds, 0 / 1, and NaN
        return rng.choice(np.array([0.0, 0.25, 0.5, 0.5, 0.75, 1.0, np.nan], F), size=(rows, S))
    if kind == "turns":
        on = (rng.uniform(size=(rows // 4 + 1, S)) < 0.4).repeat(4, 0)[:rows]
        return np.where(on, rng.uniform(0.45, 1.0, (rows, S)), rng.uniform(0.0, 0.55, (rows, S))).astype(F)
    return rng.uniform(size=(rows, S)).astype(F)


STREAM_CASES = [
    config(S=1),
    config(S=4, pad_on=1, pad_off=2, min_on=2, min_off=3, max_stored=0),
    config(S=4, logits=True, max_stored=5),
    config(S=7, onset=0.6, offset=0.4, pad_on=3, min_off=1, logits=True, max_stored=1000),
    config(S=32, pad_off=1, min_on=1, max_stored=64),
    config(S=4, onset=0.5, offset=0.5, pad_on=2, pad_off=2, min_on=4, min_off=3, max_stored=None),
]


def emul_push(emul, cfg, scratch, cursor, fin, ten):
    S = cfg["num_speakers"]
    ints = np.array([S, cfg["onset_pad_frames"], cfg["offset_pad_frames"], cfg["min_frames_on"], cfg["min_frames_off"],
                     cfg["activity_type"]], np.int32)
    floats = np.array([cfg["onset_threshold"], cfg["offset_threshold"]], F)
    fin, ten = np.ascontiguousarray(fin, F).reshape(-1, S), np.ascontiguousarray(ten, F).reshape(-1, S)
    n, m = fin.shape[0], ten.shape[0]
    from oracle.oracle_timeline import SEGMENT
    fo = np.zeros(S * (n // 2 + 2), SEGMENT)
    to = np.zeros(S * ((m + 1) // 2 + 2), SEGMENT)
    counts, lanes = np.zeros(2, np.int64), np.zeros(S, np.int64)
    emul.timeline_emul_push(ints.ctypes.data, floats.ctypes.data, scratch.ctypes.data, cursor, fin.ctypes.data, n,
                            ten.ctypes.data, m, fo.ctypes.data, to.ctypes.data, counts.ctypes.data, lanes.ctypes.data)
    return fo[:counts[0]], to[:counts[1]], lanes


@pytest.mark.parametrize("case", range(len(STREAM_CASES)))
@pytest.mark.parametrize("kind", ["levels", "turns", "uniform"])
def test_oracle_restatement_and_emulation_agree(O, emul, case, kind):
    cfg = STREAM_CASES[case]
    S = cfg["num_speakers"]
    rng = np.random.default_rng(zlib.crc32(f"{case}/{kind}".encode()))
    o, p = O.Timeline(cfg), PyTimeline(cfg)
    scratch = o.state().scratch   # fresh: INT64_MIN frames
    cursor = 0
    for step in range(30):
        shape = rng.integers(0, 5)
        n = 0 if shape == 0 else int(rng.integers(1, 40))          # shape 0: a tentative-only (or empty) push
        m = 0 if shape == 1 else int(rng.integers(0, 12))
        fin, ten = draw(rng, n, S, kind), draw(rng, m, S, kind)
        f, t = o.add_chunk(fin, ten)
        pf, pt = p.add_chunk(fin, ten)
        same_segments(records(f), pf)
        same_segments(records(t), pt)
        ef, et, lanes = emul_push(emul, cfg, scratch, cursor, fin, ten)
        assert ef.tobytes() == f.tobytes() and et.tobytes() == t.tobytes()
        assert (lanes <= (n + m + 1) // 2 + 1).all()
        st = o.state()
        assert scratch.tobytes() == st.scratch.tobytes()
        for k in range(S):
            same_scratch(st.scratch[k], p.scratch[k])
        cursor += n
        assert st.finalized_frames == cursor == p.cursor
        assert np.array_equal(bits(st.stored), bits(np.array(p.stored, F).reshape(-1, S)))
        assert np.array_equal(bits(st.tentative), bits(np.array(p.tentative, F).reshape(-1, S)))
        if step % 7 == 6:
            o.finalize()
            p.finalize()
            cursor += m
        if step % 11 == 10:
            k = int(rng.integers(0, S))
            o.clear_speaker(k)
            p.clear_speaker(k)
            scratch[k] = o.state().scratch[k]


# ---- the per-push segment bound ------------------------------------------------------------------------------------
def test_alternating_input_reaches_the_segment_bound(O, emul):
    """ceil((n + m) / 2) + 1 segments per speaker: alternating input from a speaking lane, n and m odd"""
    cfg = config(S=2)
    for n, m in ((1, 1), (3, 5), (45, 7), (101, 3)):
        o = O.Timeline(cfg)
        scratch = o.state().scratch
        first = np.ones((1, 2), F)
        o.add_chunk(first)
        emul_push(emul, cfg, scratch, 0, first, np.zeros((0, 2), F))
        fin = (np.arange(n) % 2 == 1).astype(F)[:, None].repeat(2, 1)    # 0, 1, 0, ... from speaking
        ten = (np.arange(m) % 2 == 0).astype(F)[:, None].repeat(2, 1)    # 1, 0, 1, ...
        f, t = o.add_chunk(fin, ten)
        _, _, lanes = emul_push(emul, cfg, scratch, 1, fin, ten)
        assert (lanes == (n + m + 1) // 2 + 1).all(), (n, m, lanes)
        assert len(f) + len(t) == 2 * ((n + m + 1) // 2 + 1)


def test_segment_bound_holds_for_every_short_binary_stream():
    """Every 0/1 stream of up to 9 frames, split into a prior push, finalized and tentative rows, under several
    configurations: no lane ever exceeds the bound, and for odd n and m some stream reaches it."""
    cfgs = [config(S=1), config(S=1, pad_off=1), config(S=1, pad_on=1, pad_off=1, min_off=1), config(S=1, min_on=1)]
    reached = {}
    for bitsn in range(1, 10):
        for v in range(2 ** bitsn):
            seq = [F((v >> i) & 1) for i in range(bitsn)]
            for pre in range(0, bitsn):
                for n in range(0, bitsn - pre + 1):
                    m = bitsn - pre - n
                    for ci, cfg in enumerate(cfgs):
                        t = PyTimeline(cfg)
                        if pre:
                            t.add_chunk(np.array(seq[:pre], F), np.zeros(0, F))
                        f, g = t.add_chunk(np.array(seq[pre:pre + n], F), np.array(seq[pre + n:], F))
                        got = len(f) + len(g)
                        assert got <= (n + m + 1) // 2 + 1, (seq, pre, n, m, ci)
                        assert len(f) <= (n // 2 + 1 if n else 0) and len(g) <= (m + 1) // 2 + 1
                        reached[(n, m)] = max(reached.get((n, m), 0), got)
    for (n, m), best in reached.items():
        if n % 2 == 1 and m % 2 == 1:   # both odd: the bound is the exact maximum
            assert best == (n + m + 1) // 2 + 1, (n, m, best)


# ---- configuration through the C ABI (no device) ----------------------------------------------------------------------
def test_presets(lib):
    from fluidaudio_b200.diarizer_timeline import DiarizerTimelineConfig
    s = DiarizerTimelineConfig.sortformer_default()
    assert (s.num_speakers, F(s.frame_duration_seconds)) == (4, F(0.08))
    d = DiarizerTimelineConfig.default(7, 0.1)
    assert (d.num_speakers, F(d.frame_duration_seconds), d.onset_threshold, d.offset_threshold) == (7, F(0.1), 0.5, 0.5)
    assert (d.onset_pad_frames, d.offset_pad_frames, d.min_frames_on, d.min_frames_off, d.activity_type) == (0,) * 5
    assert d.store_segments


def test_seconds_initialiser_rounds_half_away_from_zero(lib):
    from fluidaudio_b200.diarizer_timeline import DiarizerTimelineConfig
    # frame 0.5 s: every quotient is exact in float32, so the .5 cases are true ties
    c = DiarizerTimelineConfig.from_seconds(0.25, 0.75, 1.25, -0.25, frame_duration_seconds=0.5)
    assert (c.onset_pad_frames, c.offset_pad_frames, c.min_frames_on, c.min_frames_off) == (1, 2, 3, -1)
    c = DiarizerTimelineConfig.from_seconds(0.2, 0.12, 0.04, 0.36, frame_duration_seconds=0.08)
    want = [int(math.copysign(math.floor(abs(float(F(F(x) / F(0.08)))) + 0.5), x)) for x in (0.2, 0.12, 0.04, 0.36)]
    assert [c.onset_pad_frames, c.offset_pad_frames, c.min_frames_on, c.min_frames_off] == want
    cfg = DiarizerTimelineConfig(frame_duration_seconds=0.0).to_c()
    assert lib.fa_diarizer_timeline_config_from_seconds(C.byref(cfg), 1.0, 0.0, 0.0, 0.0) == 1   # inf: Swift traps


def test_create_rejects_invalid_configs(lib):
    from fluidaudio_b200.diarizer_timeline import DiarizerTimelineConfig
    bad = [dict(num_speakers=0), dict(num_speakers=33), dict(onset_pad_frames=-1), dict(min_frames_off=-1),
           dict(onset_threshold=float("nan")), dict(frame_duration_seconds=float("inf")), dict(activity_type=2),
           dict(max_stored_frames=-1)]
    for kw in bad:
        h = C.c_void_p()
        assert lib.fa_diarizer_timeline_create(C.byref(DiarizerTimelineConfig(**kw).to_c()), 8, C.byref(h)) == 1, kw
        assert not h.value
    h = C.c_void_p()
    assert lib.fa_diarizer_timeline_create(C.byref(DiarizerTimelineConfig().to_c()), -1, C.byref(h)) == 1


def test_segment_bound_entry(lib):
    f, t = C.c_int64(), C.c_int64()
    fr, tr = np.array([0, 1, 4, 45000], np.int64), np.array([7, 0, 3, 0], np.int64)
    assert lib.fa_diarizer_timeline_segment_bound(4, 4, fr.ctypes.data, tr.ctypes.data, C.byref(f), C.byref(t)) == 0
    assert f.value == 4 * (0 + 1 + 3 + 22501) and t.value == 4 * (5 + 1 + 3 + 1)
