"""Voice activity detection on the H100 against the oracle, exactly: the Silero model inputs byte for byte, events and
whole session state after advances over many sessions, speech segments for many clips over the config corners, the
FSMN decision up to an hour, host and device variants, refused calls, launch counts and VadManager's chunk loop."""
import ctypes as C
import math

import numpy as np
import pytest

from fluidaudio_b200 import _lib
from fluidaudio_b200 import vad as V
from oracle import oracle_vad as O

pytestmark = pytest.mark.gpu

LENGTHS = (0, 1, 63, 64, 4095, 4096, 5000)


@pytest.fixture(scope="module", autouse=True)
def device():
    if _lib.device_count() < 1:
        pytest.skip("needs an H100")
    _lib.set_device(0)


def _cfg_pair(**kw):
    """(oracle config, library-side VadConfig + VadSegmentationConfig) of the same values"""
    default = kw.pop("default_threshold", 0.85)
    return O.config(default_threshold=default, **kw), V.VadConfig(default), V.VadSegmentationConfig(**kw)


def fake_model(inp, hid, cel):
    """deterministic and elementwise per row, so a batch equals its rows one by one"""
    inp, hid, cel = (np.asarray(a, np.float32) for a in (inp, hid, cel))
    a = np.nan_to_num(np.abs(inp[:, 100]) * np.float32(0.37) + np.abs(inp[:, 4100]), nan=0.5, posinf=0.25)
    p = np.mod((a + np.abs(hid[:, 0])) * np.float32(3.1), np.float32(1.0)).astype(np.float32)
    p[inp[:, 71] > np.float32(0.7)] = np.float32("nan")   # now and then a NaN probability
    nh = np.nan_to_num(hid * np.float32(0.5) + inp[:, 64:192] * np.float32(0.25), nan=0.1, posinf=0.2, neginf=-0.2)
    nc = np.nan_to_num(cel * np.float32(0.9) - hid * np.float32(0.1), nan=0.1, posinf=0.2, neginf=-0.2)
    return p, nh.astype(np.float32), nc.astype(np.float32)


def _chunk(rng, n):
    x = rng.normal(0, 0.3, size=n).astype(np.float32)
    if n > 3 and rng.random() < 0.3:
        x[rng.integers(0, n)] = np.float32("nan")
        x[rng.integers(0, n)] = np.float32("inf")
    return x


def _same_state(st, ref):
    assert st.context.tobytes() == ref.context.tobytes()
    assert st.hidden.tobytes() == ref.hidden.tobytes() and st.cell.tobytes() == ref.cell.tobytes()
    assert (st.processed_samples, int(st.triggered), -1 if st.temp_end_sample is None else st.temp_end_sample) == \
        tuple(int(v) for v in ref.state)


@pytest.mark.parametrize("S,steps,kw", [
    (1, 40, {}), (7, 30, dict(min_silence_duration=0.0, speech_padding=0.0)),
    (64, 20, dict(negative_threshold=0.3, negative_threshold_offset=0.1)), (4096, 4, dict(default_threshold=0.4)),
])
def test_streams_equal_the_oracle(S, steps, kw):
    rng = np.random.default_rng(S)
    ocfg, vcfg, scfg = _cfg_pair(**kw)
    streams = V.SileroVadStreams()
    ids = [streams.open() for _ in range(S)]
    assert ids == list(range(S))
    refs = [O.Stream() for _ in ids]
    events = 0
    for step in range(steps):
        live = [i for i in range(S) if rng.random() < 0.7] or [0]
        rng.shuffle(live)
        chunks = [_chunk(rng, int(rng.choice(LENGTHS))) for _ in live]
        inp, hid, cel = streams.model_inputs([ids[i] for i in live], chunks)
        for j, i in enumerate(live):
            want, nxt = O.model_input(refs[i].context, chunks[j])
            assert inp[j].tobytes() == want.tobytes(), (step, i, chunks[j].size)
            assert hid[j].tobytes() == refs[i].hidden.tobytes() and cel[j].tobytes() == refs[i].cell.tobytes()
        p, nh, nc = fake_model(inp, hid, cel)
        ev = streams.advance([ids[i] for i in live], p, nh, nc, vcfg, scfg)
        for j, i in enumerate(live):
            want, nxt = O.model_input(refs[i].context, chunks[j])
            refs[i].context, refs[i].hidden, refs[i].cell = nxt, nh[j].copy(), nc[j].copy()
            assert tuple(int(v) for v in ev[j]) == refs[i].step(p[j], chunks[j].size, ocfg), (step, i)
            events += int(ev[j, 0] != 0)
        check = live if S <= 64 else live[:16]
        for i in check:
            _same_state(streams.state(ids[i]), refs[i])
    assert events > 0
    for i in range(0, S, max(1, S // 64)):
        _same_state(streams.state(ids[i]), refs[i])
    streams.close_handle()


def test_refused_calls_change_nothing_and_launch_counts():
    streams = V.SileroVadStreams()
    a, b = streams.open(), streams.open()
    x = np.ones(4096, np.float32)
    before = _lib.kernel_launch_count()
    streams.model_inputs([a, b], [x, x * 2])
    assert _lib.kernel_launch_count() - before == 1
    snap = [streams.state(s) for s in (a, b)]
    for bad in ([a, a], [a, 9], [a, -1]):
        with pytest.raises(_lib.FluidAudioError):
            streams.model_inputs(bad, [x, x])
    L = _lib.load()
    ids, off = np.array([a, b], np.int32), np.array([0, 5, 3], np.int64)
    z = np.zeros((2, 4160), np.float32)
    h = np.zeros((2, 128), np.float32)
    assert L.fa_vad_stream_model_inputs(streams._h, 2, ids.ctypes.data, x.ctypes.data, off.ctypes.data, z.ctypes.data,
                                        h.ctypes.data, h.ctypes.data) == 1
    p, nh, nc = np.array([0.9, 0.9], np.float32), np.ones((2, 128), np.float32), np.ones((2, 128), np.float32)
    before = _lib.kernel_launch_count()
    streams.advance([a], p[:1], nh[:1], nc[:1])
    assert _lib.kernel_launch_count() - before == 1
    with pytest.raises(_lib.FluidAudioError):   # a has nothing staged any more: the whole call is refused
        streams.advance([b, a], p, nh, nc)
    with pytest.raises(ValueError):
        V.VadSegmentationConfig(max_speech_duration=0.0)
    after = streams.state(b)
    assert after.has_pending and after.processed_samples == 0 and after.hidden.tobytes() == snap[1].hidden.tobytes()
    before = _lib.kernel_launch_count()
    streams.model_inputs([], [])
    streams.advance([], [], np.zeros((0, 128)), np.zeros((0, 128)))
    assert _lib.kernel_launch_count() == before
    streams.close(a)
    assert streams.open() == a   # the lowest free id, fresh
    st = streams.state(a)
    assert st.processed_samples == 0 and st.temp_end_sample is None and not st.has_pending
    streams.close_handle()


def test_device_variants_equal_host_variants():
    rng = np.random.default_rng(5)
    S = 33
    host, dev = V.SileroVadStreams(), V.SileroVadStreams()
    hid_ = [host.open() for _ in range(S)]
    did_ = [dev.open() for _ in range(S)]
    for step in range(6):
        chunks = [_chunk(rng, int(rng.choice(LENGTHS))) for _ in range(S)]
        inp, hh, hc = host.model_inputs(hid_, chunks)
        audio = np.concatenate(chunks)
        off = np.concatenate([[0], np.cumsum([c.size for c in chunks])]).astype(np.int64)
        d_audio, d_inp = _lib.DeviceBuffer(max(4, audio.nbytes)), _lib.DeviceBuffer(S * 4160 * 4)
        d_h, d_c = _lib.DeviceBuffer(S * 512), _lib.DeviceBuffer(S * 512)
        if audio.size:
            d_audio.upload(audio)
        _lib.synchronize()   # the uploads ran on the legacy stream, the handle's stream does not wait for them
        dev.model_inputs_device(did_, d_audio, off, d_inp, d_h, d_c)
        _lib.synchronize()   # the call is asynchronous on the handle's non-blocking stream
        assert d_inp.download((S, 4160), np.float32).tobytes() == inp.tobytes()
        assert d_h.download((S, 128), np.float32).tobytes() == hh.tobytes()
        assert d_c.download((S, 128), np.float32).tobytes() == hc.tobytes()
        p, nh, nc = fake_model(inp, hh, hc)
        ev = host.advance(hid_, p, nh, nc)
        d_p, d_nh, d_nc, d_ev = (_lib.DeviceBuffer(a.nbytes) for a in (p, nh, nc, ev))
        d_p.upload(p), d_nh.upload(nh), d_nc.upload(nc)
        _lib.synchronize()
        dev.advance_device(did_, d_p, d_nh, d_nc, d_ev)
        _lib.synchronize()
        assert d_ev.download((S, 2), np.int64).tobytes() == ev.tobytes()
        for a, b in zip(hid_, did_):
            x, y = host.state(a), dev.state(b)
            assert x.context.tobytes() == y.context.tobytes() and x.hidden.tobytes() == y.hidden.tobytes()
            assert x.cell.tobytes() == y.cell.tobytes() and (x.triggered, x.temp_end_sample, x.processed_samples,
                                                              x.has_pending) == \
                (y.triggered, y.temp_end_sample, y.processed_samples, y.has_pending)
    host.close_handle()
    dev.close_handle()


SEG_CORNERS = [
    dict(), dict(max_speech_duration=math.inf), dict(use_max_possible_silence_at_max_speech=False,
                                                     max_speech_duration=3.0, min_silence_at_max_speech=0.0),
    dict(negative_threshold=0.4, negative_threshold_offset=0.2), dict(speech_padding=0.0),
    dict(min_silence_duration=0.0, max_speech_duration=1.0, min_silence_at_max_speech=0.0),
]


def _probs(rng, P):
    levels = np.array([0.05, 0.25, 0.6, 0.8, 0.95], np.float32)
    p = np.repeat(rng.choice(levels, size=P), rng.integers(1, 12, size=P))[:P].astype(np.float32)
    if P and rng.random() < 0.05:
        p[rng.integers(0, P)] = np.float32("nan")
    return p


@pytest.mark.parametrize("clips,max_chunks", [(1, 879), (17, 879), (1000, 300), (10000, 120)])
@pytest.mark.parametrize("ci", range(len(SEG_CORNERS)))
def test_segments_equal_the_oracle(clips, max_chunks, ci):
    rng = np.random.default_rng(clips * 10 + ci)
    ocfg, vcfg, scfg = _cfg_pair(**SEG_CORNERS[ci])
    probs = [_probs(rng, int(rng.integers(0, max_chunks + 1))) for _ in range(clips)]
    if clips == 1:
        probs = [_probs(rng, 879)]
    totals = [int(p.size * 4096 + rng.choice([0, -5000, -1, 3000, 0])) for p in probs]
    before = _lib.kernel_launch_count()
    got = V.segment_sample_ranges(probs, totals, vcfg, scfg)
    assert _lib.kernel_launch_count() - before <= 2
    n = 0
    for g, p, t in zip(got, probs, totals):
        assert [tuple(int(v) for v in r) for r in g] == O.segment(p, t, ocfg)
        n += len(g)
    assert clips < 100 or n > 0


def test_segment_capacity_device_variant_and_empty():
    rng = np.random.default_rng(3)
    ocfg, vcfg, scfg = _cfg_pair()
    probs = [_probs(rng, 400) for _ in range(9)]
    totals = [p.size * 4096 for p in probs]
    want = [O.segment(p, t, ocfg) for p, t in zip(probs, totals)]
    total = sum(map(len, want))
    assert total > 2
    L = _lib.load()
    data = np.concatenate(probs)
    off = np.concatenate([[0], np.cumsum([p.size for p in probs])]).astype(np.int64)
    ts = np.array(totals, np.int64)
    counts, seg, tot = np.zeros(9, np.int64), np.full((total, 2), -7, np.int64), C.c_int64()
    cfg = V._c_config(vcfg, scfg)
    st = L.fa_vad_segment(data.ctypes.data, off.ctypes.data, 9, ts.ctypes.data, C.byref(cfg), counts.ctypes.data,
                          seg.ctypes.data, total - 1, C.byref(tot))
    assert st == V.STATUS_OUTPUT_TOO_SMALL and tot.value == total and list(counts) == [len(w) for w in want]
    assert (seg == -7).all()
    d_in, d_out = _lib.DeviceBuffer(data.nbytes), _lib.DeviceBuffer(seg.nbytes)
    d_in.upload(data)
    _lib.synchronize()
    _lib.check(L.fa_vad_segment_device(d_in.ptr, off.ctypes.data, 9, ts.ctypes.data, C.byref(cfg), counts.ctypes.data,
                                       d_out.ptr, total, C.byref(tot)), "fa_vad_segment_device")
    _lib.synchronize()
    assert [tuple(r) for r in d_out.download((total, 2), np.int64).tolist()] == [r for w in want for r in w]
    assert V.segment_sample_ranges([], [], vcfg) == []
    with pytest.raises(ValueError):   # one total_samples per clip
        V.segment_sample_ranges(probs, totals[:-1], vcfg)
    assert [len(g) for g in V.segment_sample_ranges([np.zeros(0, np.float32), probs[0]], [0, 0], vcfg)] == [0, 0]


def _silence(rng, T):
    runs = rng.integers(1, 3000, size=T // 100 + 2)
    vals = rng.choice(np.array([0.02, 0.15, 0.2, 0.25, 0.9, np.nan], np.float32), size=runs.size)
    return np.repeat(vals, runs)[:T].astype(np.float32)


@pytest.mark.parametrize("clips,T", [(1, 360_000), (64, 20_000), (3000, 700)])
def test_fsmn_equals_the_oracle(clips, T):
    rng = np.random.default_rng(clips)
    sil = [_silence(rng, int(rng.integers(0, T + 1)) if clips > 1 else T) for _ in range(clips)]
    before = _lib.kernel_launch_count()
    got = V.fsmn_vad_decide(sil)
    assert _lib.kernel_launch_count() - before <= 2
    for g, s in zip(got, sil):
        assert [(x.start_ms, x.end_ms) for x in g] == O.fsmn_decide(s)
    total = sum(map(len, got))
    assert total > 0
    # the device variant: silence and segments in HBM
    data = np.concatenate(sil)
    off = np.concatenate([[0], np.cumsum([x.size for x in sil])]).astype(np.int64)
    d_in, d_out = _lib.DeviceBuffer(max(4, data.nbytes)), _lib.DeviceBuffer(total * 16)
    if data.size:
        d_in.upload(data)
    _lib.synchronize()
    counts, tot = np.zeros(clips, np.int64), C.c_int64()
    _lib.check(_lib.load().fa_fsmn_vad_decide_device(d_in.ptr, off.ctypes.data, clips, counts.ctypes.data, d_out.ptr,
                                                     total, C.byref(tot)), "fa_fsmn_vad_decide_device")
    _lib.synchronize()
    assert tot.value == total and list(counts) == [len(g) for g in got]
    assert [tuple(r) for r in d_out.download((total, 2), np.int64).tolist()] == \
        [(x.start_ms, x.end_ms) for g in got for x in g]


def test_vad_manager_process_equals_the_oracle_chunk_loop():
    rng = np.random.default_rng(21)
    clips = [rng.normal(0, 0.3, size=int(n)).astype(np.float32) for n in rng.integers(0, 4096 * 40, size=50)]
    clips += [np.zeros(0, np.float32), np.ones(4096, np.float32), np.ones(4097, np.float32)]
    m = V.VadManager(fake_model)
    got = m.process(clips)
    for g, c in zip(got, clips):
        assert g.tobytes() == O.process(c, fake_model).tobytes()
    x = clips[0]
    segs = m.segment_speech(x, V.VadSegmentationConfig(min_silence_duration=0.3))
    want = O.segment(O.process(x, fake_model), x.size, O.config(min_silence_duration=0.3))
    assert [(s.start_time, s.end_time) for s in segs] == [(a / 16000.0, b / 16000.0) for a, b in want]
    audio = m.segment_speech_audio(x, V.VadSegmentationConfig(min_silence_duration=0.3))
    assert [a.size for a in audio] == [int(e / 16000.0 * 16000.0) - int(s / 16000.0 * 16000.0) for s, e in want]
    sid = m.make_stream_state()
    ref = O.Stream()
    for k in range(12):
        chunk = x[k * 1000:(k + 1) * 1000 + 2000] if k % 3 else np.zeros(0, np.float32)
        r = m.process_streaming_chunk(chunk, sid, return_seconds=True, time_resolution=2)
        kind, sample, p = ref.chunk(chunk, fake_model, O.config())
        assert np.float32(r.probability).tobytes() == p.tobytes()
        assert (r.event is None) == (kind == 0) and (r.event is None or r.event.sample_index == sample)
    m.close_stream_state(sid)
