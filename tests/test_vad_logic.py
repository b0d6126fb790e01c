"""Voice activity detection's logic on the CPU: the reference's model-free VAD tests on the oracle, the oracle held to
a literal Python restatement (tests/vad_restated.py), the host build of vad_core.cuh (tests/emul/vad_emul.cpp) held to
the oracle bit for bit with the segment bound checked exhaustively on short streams, fa_vad_resolve against the
oracle, and FsmnVadManager's chunk schedule."""
import ctypes as C
import itertools
import math
import os
import subprocess

import numpy as np
import pytest

import vad_restated as R
from fluidaudio_b200 import _lib
from fluidaudio_b200 import vad as V
from oracle import oracle_vad as O

CHUNK_S = 4096 / 16000.0


def _cfg(**kw):
    return O.config(**kw)


def _seconds(ranges):
    return [(a / 16000.0, b / 16000.0) for a, b in ranges]


# ---------------------------------------------------------------- the reference's segmentation tests, on the oracle
def _segments(pattern, **kw):
    p, total = R.make_vad_results(pattern)
    return _seconds(O.segment(p, total, _cfg(**kw)))


def _durations(segs):
    return [b - a for a, b in segs]


def test_silence_produces_no_segments():
    assert _segments([(False, 2.0)]) == []


def test_continuous_speech_produces_segment():
    s = _segments([(True, 5.0)])
    assert len(s) == 1 and sum(_durations(s)) > 4.5


def test_single_segment_amid_silence():
    s = _segments([(False, 1.0), (True, 3.0), (False, 1.0)], min_speech_duration=0.15)
    assert len(s) == 1 and 2.7 < _durations(s)[0] < 3.4


@pytest.mark.parametrize("pattern,count", [
    ([(False, 1.0), (True, 2.0), (False, 1.0), (True, 2.0), (False, 1.0)], 2),
    ([(True, 1.0), (False, 0.5), (True, 1.0)], 1),
    ([(True, 1.0), (False, 1.0), (True, 1.0)], 2),
])
def test_merging_and_separation(pattern, count):
    s = _segments(pattern, min_speech_duration=0.15, min_silence_duration=0.75)
    assert len(s) == count
    if count == 1:
        assert 2.4 < _durations(s)[0] < 2.6
    if pattern[1] == (False, 1.0):
        assert all(0.9 < d < 1.3 for d in _durations(s))
    assert all(d < 15.0 for d in _durations(s))


def test_min_speech_duration_filter():
    s = _segments([(True, 0.2), (False, 1.0), (True, 0.8), (False, 1.0), (True, 0.1)], min_speech_duration=0.5,
                  min_silence_duration=0.75)
    assert len(s) == 1 and 0.7 < _durations(s)[0] < 1.1


@pytest.mark.parametrize("seconds,max_speech,least", [(30.0, 15.0, 2), (25.0, 10.0, 3), (16.0, 15.0, 2)])
def test_long_speech_splits(seconds, max_speech, least):
    s = _segments([(True, seconds)], min_speech_duration=0.15, max_speech_duration=max_speech)
    assert len(s) >= least and all(d < max_speech + 0.1 for d in _durations(s))


def test_exactly_max_duration_segment():
    p, total = R.make_vad_results([(True, 5.0)])
    exact = CHUNK_S * len(p)
    s = _seconds(O.segment(p, total, _cfg(min_speech_duration=0.15, max_speech_duration=exact)))
    assert len(s) == 1 and abs(_durations(s)[0] - exact) <= CHUNK_S
    s = _segments([(True, 5.0)], min_speech_duration=0.15, max_speech_duration=5.0)
    assert s and all(d <= 5.1 for d in _durations(s))


def test_alternating_speech_silence():
    assert len(_segments([(True, 0.3), (False, 0.3)] * 5, min_speech_duration=0.1, min_silence_duration=0.2)) >= 1


def test_custom_segmentation_config():
    s = _segments([(True, 20.0)], min_speech_duration=1.0, min_silence_duration=2.0, max_speech_duration=8.0,
                  speech_padding=0.2, silence_threshold_for_split=0.5)
    assert len(s) >= 3 and all(d < 8.1 for d in _durations(s))


def test_real_world_pattern():
    s = _segments([(True, 5.0), (False, 85.0), (True, 30.0)], min_speech_duration=0.15, min_silence_duration=0.75,
                  max_speech_duration=15.0)
    assert 3 <= len(s) <= 4 and all(d < 15.1 for d in _durations(s))
    # VadTests.swift:547 reads `first?.endTime ?? 0 - (...)`: `??` binds looser than `-`, so it checks the end time
    assert s[0][1] > 4.9


def test_speech_padding_application():
    s = _segments([(False, 1.0), (True, 2.0), (False, 1.0)], min_speech_duration=0.25, speech_padding=0.2)
    assert len(s) == 1 and 2.0 < _durations(s)[0] < 2.0 + 0.2 * 2 + 0.1


def test_empty_input_and_very_short_speech():
    assert O.segment([], 0, _cfg()) == []
    assert _segments([(True, 0.05)], min_speech_duration=0.15) == []


# ---------------------------------------------------------------- the reference's streaming tests, on the oracle
def _drive(probs, cfg, n=4096):
    s = O.Stream()
    return [s.step(p, n, cfg) for p in probs], s


def test_streaming_emits_start_and_end_events():
    ev, s = _drive([0.9] + [0.05] * 5, _cfg())
    assert ev[0] == (1, 0)
    ends = [e for e in ev[1:] if e[0]]
    assert ends and ends[0][0] == 2 and ends[0][1] > 0 and s.state[1] == 0


def test_streaming_returns_seconds_when_requested():
    ev, _ = _drive([0.9] + [0.05] * 5, _cfg())
    kind, sample = next(e for e in ev[1:] if e[0])
    e = V.stream_event(kind, sample, True, 2)
    assert e.is_end and e.time == V.swift_rounded(sample / 16000.0 * 100) / 100


@pytest.mark.parametrize("default,kw,below,above", [(0.8, dict(negative_threshold=0.2, negative_threshold_offset=0.05),
                                                     0.24, 0.3), (0.6, {}, 0.59, 0.7)])
def test_streaming_threshold_override_and_default(default, kw, below, above):
    ev, _ = _drive([below, above], _cfg(default_threshold=default, **kw))
    assert ev[0] == (0, -1) and ev[1] == (1, max(0, 4096 - int(0.1 * 16000)))


def test_swift_rounding_ties_away_from_zero():
    assert V.swift_rounded(2.5) == 3.0 and V.swift_rounded(-2.5) == -3.0 and V.swift_rounded(0.49999999999999994) == 0


# ---------------------------------------------------------------- FsmnVadChunkingTests on the Python helpers
def _absolute(a, b):
    return np.arange(V.FsmnVadManager.lfr_frame_count(b - a), dtype=np.float32) + a // V.FsmnVadManager.HOP_SAMPLES


def test_fsmn_full_chunk_frame_count():
    assert V.FsmnVadManager.lfr_frame_count(488_320) == 3048 and V.FsmnVadManager.lfr_frame_count(399) == 0


@pytest.mark.parametrize("total", [100 * 60 * 16_000, 488_320 + 7_213])
def test_fsmn_chunks_tile_the_absolute_grid(total):
    starts = []

    def score(a, b):
        starts.append(a)
        assert a % V.FsmnVadManager.HOP_SAMPLES == 0
        return _absolute(a, b)

    sil = V.FsmnVadManager.concatenate_chunks(total, score)
    assert np.array_equal(sil, np.arange(sil.size, dtype=np.float32))
    whole = V.FsmnVadManager.lfr_frame_count(total)
    assert whole - V.FsmnVadManager.LFR_PAD_FRAMES <= sil.size <= whole
    if total > 10 ** 7:
        assert len(starts) > 100


def test_fsmn_hour_has_no_cumulative_drift():
    sil = V.FsmnVadManager.concatenate_chunks(60 * 60 * 16_000, _absolute)
    assert 360_000 - 5 <= sil.size <= 360_000


def test_fsmn_short_audio_single_chunk_and_too_short():
    calls = []
    sil = V.FsmnVadManager.concatenate_chunks(20 * 16_000, lambda a, b: calls.append((a, b)) or _absolute(a, b))
    assert calls == [(0, 20 * 16_000)] and sil.size == V.FsmnVadManager.lfr_frame_count(20 * 16_000)
    assert V.FsmnVadManager.concatenate_chunks(300, lambda a, b: []).size == 0


# ---------------------------------------------------------------- seeded streams: oracle vs restatement vs emulation
LEVELS = [np.float32(v) for v in (0.1, 0.5, 0.8, 0.9)]   # below split, below negative, below threshold, above

CONFIGS = [
    dict(),
    dict(max_speech_duration=math.inf),
    dict(max_speech_duration=0.9, min_silence_duration=0.3, min_silence_at_max_speech=0.0),
    dict(max_speech_duration=0.3, min_silence_duration=0.0, min_silence_at_max_speech=0.0, speech_padding=0.0),
    dict(max_speech_duration=1.2, use_max_possible_silence_at_max_speech=False, min_silence_duration=0.5,
         min_silence_at_max_speech=0.0),
    dict(negative_threshold=0.6, negative_threshold_offset=0.25, max_speech_duration=1.0, min_silence_duration=0.2),
    dict(speech_padding=0.0, min_speech_duration=0.0, min_silence_duration=0.0),
    dict(speech_padding=0.7, min_silence_duration=0.26, max_speech_duration=2.0, min_silence_at_max_speech=0.1),
    dict(default_threshold=0.005),
]


def _streams(seed, count):
    rng = np.random.default_rng(seed)
    for _ in range(count):
        P = int(rng.integers(0, 120))
        kind = rng.integers(0, 3)
        if kind == 0:
            p = rng.choice(LEVELS, size=P)
        elif kind == 1:
            p = rng.uniform(0, 1, size=P).astype(np.float32)
        else:   # runs, so candidate silences of equal length tie
            p = np.repeat(rng.choice(LEVELS, size=P), rng.integers(1, 6, size=P))[:P]
        if P and rng.random() < 0.1:
            p[rng.integers(0, P)] = np.float32("nan")
        total = int(P * 4096 + rng.integers(-3 * 4096, 3 * 4096)) if rng.random() < 0.5 else P * 4096
        yield p.astype(np.float32), total


@pytest.fixture(scope="module")
def emul(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("vad") / "libvad_emul.so")
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-fPIC", "-shared", "-o", out,
                           os.path.join(os.path.dirname(os.path.abspath(__file__)), "emul", "vad_emul.cpp")])
    L = C.CDLL(out)
    vp, i64 = C.c_void_p, C.c_int64
    L.vad_emul_chunk_sample.argtypes = [vp, i64, C.c_int]
    L.vad_emul_chunk_sample.restype = C.c_float
    L.vad_emul_stream_step.argtypes = [vp, C.c_float, i64, C.POINTER(O.Resolved), C.POINTER(i64)]
    L.vad_emul_stream_step.restype = C.c_int
    L.vad_emul_segment.argtypes = [vp, i64, i64, C.POINTER(O.Resolved), vp]
    L.vad_emul_segment.restype = i64
    L.vad_emul_fsmn.argtypes = [vp, i64, vp]
    L.vad_emul_fsmn.restype = i64
    return L


def _emul_segment(L, p, total, r):
    p = np.ascontiguousarray(p, np.float32)
    out = np.zeros(2 * max(1, p.size), np.int64)
    n = L.vad_emul_segment(p.ctypes.data, p.size, total, C.byref(r), out.ctypes.data)
    return [(int(out[2 * k]), int(out[2 * k + 1])) for k in range(n)]


def _emul_fsmn(L, s):
    s = np.ascontiguousarray(s, np.float32)
    out = np.zeros(2 * max(1, (s.size + 1) // 2), np.int64)
    n = L.vad_emul_fsmn(s.ctypes.data, s.size, out.ctypes.data)
    return [(int(out[2 * k]), int(out[2 * k + 1])) for k in range(n)]


@pytest.mark.parametrize("ci", range(len(CONFIGS)))
def test_segments_agree_oracle_restatement_emulation(emul, ci):
    cfg = _cfg(**CONFIGS[ci])
    r, rr = O.resolve(cfg), R.resolve(cfg)
    splits = 0
    for p, total in _streams(ci, 150):
        want = O.segment(p, total, cfg)
        assert R.segment(p, total, rr) == want
        assert _emul_segment(emul, p, total, r) == want
        splits += len(want)
    assert splits > 0


def test_segment_bound_holds_exhaustively_on_short_streams(emul):
    """every stream of 1..7 probabilities over the four levels, under every config: the emulation equals the oracle
    and never emits more segments than probabilities (the scratch bound the kernel is sized by)"""
    worst = 0
    for cfg_kw in CONFIGS:
        cfg = _cfg(**cfg_kw)
        r = O.resolve(cfg)
        for P in range(1, 8):
            for combo in itertools.product(LEVELS, repeat=P):
                p = np.array(combo, np.float32)
                want = O.segment(p, P * 4096, r)
                got = _emul_segment(emul, p, P * 4096, r)
                assert got == want, (cfg_kw, combo)
                worst = max(worst, len(got) - (P + 1) // 2)
                assert len(got) <= P
    assert worst <= 0   # the tighter ceil(P / 2) observation also holds here


def test_streaming_agrees_oracle_restatement_emulation(emul):
    rng = np.random.default_rng(11)
    for ci, kw in enumerate(CONFIGS):
        cfg = _cfg(**kw)
        r, rr = O.resolve(cfg), R.resolve(cfg)
        o, py, em = O.Stream(), R.StreamState(), np.array([0, 0, -1], np.int64)
        events = 0
        for _ in range(400):
            p = rng.choice(LEVELS + [np.float32(rng.uniform()), np.float32("nan")])
            n = int(rng.choice([0, 1, 63, 64, 4095, 4096, 5000]))
            want = o.step(p, n, cfg)
            assert R.stream_step(py, p, n, rr) == want
            sample = C.c_int64()
            kind = emul.vad_emul_stream_step(em.ctypes.data, p, n, C.byref(r), C.byref(sample))
            assert (kind, sample.value) == want and list(em) == list(o.state)
            assert [py.processed, int(py.triggered), -1 if py.temp_end is None else py.temp_end] == list(o.state)
            events += want[0] != 0
        assert events > 0


def test_fsmn_agrees_oracle_restatement_emulation(emul):
    rng = np.random.default_rng(12)
    for _ in range(60):
        T = int(rng.integers(0, 20000))
        runs = rng.integers(1, 400, size=T // 50 + 1)
        vals = rng.choice(np.array([0.05, 0.19, 0.2, 0.21, 0.9, np.nan], np.float32), size=runs.size)
        s = np.repeat(vals, runs)[:T].astype(np.float32)
        want = O.fsmn_decide(s)
        assert R.fsmn_decide(s) == want and _emul_fsmn(emul, s) == want
    long = np.full(20000, 0.05, np.float32)   # one long speech run: max-segment closes
    assert len(O.fsmn_decide(long)) >= 3 and _emul_fsmn(emul, long) == O.fsmn_decide(long)


def test_chunk_staging_agrees_with_the_oracle(emul):
    rng = np.random.default_rng(13)
    ctx = rng.normal(size=64).astype(np.float32)
    for n in (0, 1, 63, 64, 4095, 4096, 5000):
        x = rng.normal(size=n).astype(np.float32)
        if n > 2:
            x[1], x[-1] = np.float32("nan"), np.float32("inf")
        inp, nxt = O.model_input(ctx, x)
        got = np.array([emul.vad_emul_chunk_sample(x.ctypes.data if n else None, n, j) for j in range(4096)],
                       np.float32)
        assert got.tobytes() == inp[64:].tobytes() and nxt.tobytes() == inp[-64:].tobytes()
        assert inp[:64].tobytes() == ctx.tobytes()


# ---------------------------------------------------------------- fa_vad_resolve
VALID = CONFIGS + [dict(negative_threshold=0.0), dict(negative_threshold=1.0, negative_threshold_offset=0.5),
                   dict(negative_threshold_offset=math.inf), dict(default_threshold=float("nan")),
                   dict(min_speech_duration=0.0, speech_padding=3.3, max_speech_duration=0.01),
                   dict(max_speech_duration=2.0 ** 61 / 16000), dict(speech_padding=(2.0 ** 62 - 1024) / 16000),
                   dict(speech_padding=(2.0 ** 62 - 1024) / 16000, max_speech_duration=1.0)]
INVALID = [dict(min_speech_duration=-1e-9), dict(min_silence_duration=float("nan")), dict(max_speech_duration=0.0),
           dict(max_speech_duration=-math.inf), dict(speech_padding=math.inf), dict(silence_threshold_for_split=1.01),
           dict(silence_threshold_for_split=float("nan")), dict(negative_threshold=-0.1),
           dict(negative_threshold=float("nan")), dict(negative_threshold_offset=-1.0),
           dict(negative_threshold_offset=float("nan")), dict(min_silence_at_max_speech=math.inf),
           dict(max_speech_duration=2.0 ** 63 / 16000), dict(min_silence_duration=1e300),
           dict(max_speech_duration=2.0 ** 62 / 16000), dict(speech_padding=2.0 ** 62 / 16000),
           dict(speech_padding=(2.0 ** 62 - 1024) / 16000, max_speech_duration=0.1)]


def _lib_resolve(cfg):
    L = _lib.load()
    out = _lib.VadResolved()
    c = _lib.VadConfig(*[getattr(cfg, k) for k, _ in cfg._fields_])
    return out if L.fa_vad_resolve(C.byref(c), C.byref(out)) == 0 else None


def _fields(r):
    return [np.float32(getattr(r, k)).tobytes() if t is C.c_float else getattr(r, k) for k, t in r._fields_]


@pytest.mark.parametrize("kw", VALID)
def test_resolve_equals_the_oracle(kw):
    cfg = _cfg(**kw)
    want = O.resolve(cfg)
    assert want is not None and _fields(_lib_resolve(cfg)) == _fields(want)
    rr = R.resolve(cfg)
    assert [rr["threshold"].tobytes(), rr["negative"].tobytes(), rr["max_speech"], rr["pad"]] == \
        [np.float32(want.threshold).tobytes(), np.float32(want.negative_threshold).tobytes(), want.max_speech_samples,
         want.speech_pad_samples]


@pytest.mark.parametrize("kw", INVALID)
def test_resolve_refuses_what_the_reference_traps_on(kw):
    cfg = _cfg(**kw)
    assert O.resolve(cfg) is None and R.resolve(cfg) is None and _lib_resolve(cfg) is None
    assert _lib.load().fa_last_error()
    with pytest.raises(ValueError):
        V.VadSegmentationConfig(**{k: v for k, v in kw.items() if k != "default_threshold"})


def test_default_config_is_the_reference_defaults():
    c = _lib.VadConfig()
    _lib.load().fa_vad_default_config(C.byref(c))
    assert _fields(c) == _fields(_lib.VadConfig(*[getattr(_cfg(), k) for k, _ in _cfg()._fields_]))


def test_segment_speech_audio_slices_one_sample_short_like_the_reference():
    s = np.arange(0, 16000 * 3600, 7, dtype=np.int64)
    assert int(np.count_nonzero((s / 16000.0 * 16000.0).astype(np.int64) != s)) == 53_932
    seg = V.VadSegment(7 * 1 / 16000.0, 1.0)
    assert seg.start_sample() == int(7 / 16000.0 * 16000.0)


def test_the_oracles_batch_entries_equal_its_single_calls():
    """oracle_vad_tick and oracle_vad_segment_batch (the timing script's native oracle arms) run the same restatement"""
    rng = np.random.default_rng(14)
    cfg = _cfg(min_silence_duration=0.3)
    r = O.resolve(cfg)
    S = 9
    t, refs = O.Tick(S), [O.Stream() for _ in range(S)]
    for _ in range(12):
        chunks = [rng.normal(size=int(rng.choice([0, 1, 64, 4096, 5000]))).astype(np.float32) for _ in range(S)]
        off = np.concatenate([[0], np.cumsum([c.size for c in chunks])]).astype(np.int64)
        p = rng.uniform(size=S).astype(np.float32)
        nh, nc = rng.normal(size=(S, 128)).astype(np.float32), rng.normal(size=(S, 128)).astype(np.float32)
        ev = t.run(np.concatenate(chunks), off, p, nh, nc, r)
        for i, ref in enumerate(refs):
            inp, nxt = O.model_input(ref.context, chunks[i])
            assert t.inputs[i].tobytes() == inp.tobytes() and t.hidden_out[i].tobytes() == ref.hidden.tobytes()
            ref.context, ref.hidden, ref.cell = nxt, nh[i], nc[i]
            assert tuple(int(v) for v in ev[i]) == ref.step(p[i], chunks[i].size, r)
            assert list(t.states[i]) == list(ref.state)
    clips = [c for c, _ in _streams(15, 40)]
    totals = [c.size * 4096 for c in clips]
    off = np.concatenate([[0], np.cumsum([c.size for c in clips])]).astype(np.int64)
    counts, pairs = O.segment_batch(np.concatenate(clips), off, totals, r)
    want = [O.segment(c, n, r) for c, n in zip(clips, totals)]
    assert list(counts) == [len(w) for w in want] and [tuple(x) for x in pairs.tolist()] == [x for w in want for x in w]
