"""Live log-mel streams (``fa_mel_stream_*``, ``MelStreams``) against SortformerDiarizer's incremental mel stream.

``MelStreamSession`` below restates the reference's session (Diarizer/Sortformer/SortformerDiarizer.swift:204-217 reset,
:417-424 addAudio, :842-870 emit, :876-901 finish) on top of any per-call ``.prePadded`` log-mel: the oracle on the CPU,
``fa_mel_compute`` on the GPU.  The CPU tests port SortformerStreamingMelTests onto the restatement; the GPU tests (``-m gpu``)
hold the batched session layer to the restatement's call sequence bit for bit.
"""
import ctypes as C
import random

import numpy as np
import pytest

from fluidaudio_b200 import _lib, synth

PRE_PADDED, CENTER = 1, 0
OK, INVALID, TOO_SMALL = 0, 1, 3
FEEDS = (160, 1600, 4093, 16000, None)   # None: the whole clip in one push


# ================================================================================================ restatement
def stream_frames(cfg, received, emitted, finished, n, finish):
    """Rows a push of n samples (and finish) emits: addAudio's count, then finalizeSession's remaining."""
    if finished:
        return 0
    r, hw = received + n, cfg.win_length // 2
    first = max(0, (r - hw) // cfg.hop_length + 1 - emitted) if r >= hw else 0
    second = 0
    if finish and r > 0:
        second = max(0, 1 + (r + cfg.n_fft - cfg.win_length) // cfg.hop_length - emitted - first)
    return first + second


class MelStreamSession:
    """One session of SortformerDiarizer's mel stream.  ``mel_fn(buffer, last, count)`` is the per-call
    computeFlatTransposed(.prePadded, expectedFrameCount: count) -> [count x nMels]; ``calls`` records its arguments."""

    def __init__(self, cfg, mel_fn):
        self.cfg, self.mel_fn = cfg, mel_fn
        self.reset()

    def reset(self):
        self.buffer = np.zeros(self.cfg.n_fft // 2, np.float32)
        self.last = np.float32(0.0)
        self.received = self.emitted = 0
        self.finished = False
        self.calls = []

    def _emit(self, count):
        rows = self.mel_fn(self.buffer, self.last, count)
        self.calls.append((self.buffer.copy(), self.last, count))
        consumed = count * self.cfg.hop_length
        self.last = self.buffer[consumed - 1]
        self.buffer = self.buffer[consumed:]
        self.emitted += count
        return rows

    def push(self, x, finish=False):
        rows = []
        if not self.finished:
            x = np.asarray(x, np.float32).reshape(-1)
            self.buffer = np.concatenate([self.buffer, x])
            self.received += x.size
            hw, hop = self.cfg.win_length // 2, self.cfg.hop_length
            if self.received >= hw:
                count = (self.received - hw) // hop + 1 - self.emitted
                if count > 0:
                    rows.append(self._emit(count))
            if finish:
                self.finished = True
                if self.received > 0:
                    remaining = 1 + (self.received + self.cfg.n_fft - self.cfg.win_length) // hop - self.emitted
                    if remaining > 0:
                        tail = np.zeros(self.cfg.n_fft // 2, np.float32)
                        a = np.float32(self.cfg.preemph)
                        if a != 0 and self.buffer.size:
                            v = self.buffer[-1]
                            for i in range(tail.size):
                                v = np.float32(v * a)
                                tail[i] = v
                        self.buffer = np.concatenate([self.buffer, tail])
                        rows.append(self._emit(remaining))
        return np.concatenate(rows) if rows else np.zeros((0, self.cfg.n_mels), np.float32)


def oracle_mel_fn(O, cfg):
    def f(buf, last, count):
        out, ml, nf = O.mel_flat_transposed(cfg, buf, last=float(last), padding_mode=PRE_PADDED, expected_frames=count)
        assert ml == count == nf
        return out.reshape(count, cfg.n_mels)
    return f


def feed(session, audio, size, finish=True):
    size = size or max(1, audio.size)
    rows = [session.push(audio[i:i + size]) for i in range(0, audio.size, size)]
    if finish:
        rows.append(session.push(np.zeros(0, np.float32), finish=True))
    return np.concatenate(rows)


AUDIO_12S = 16000 * 12 + 137


# ================================================================================================ CPU: the restatement
def test_restated_stream_feeding_granularity_is_bit_exact(oracle):
    """SortformerStreamingMelTests.testFeedingGranularityDoesNotChangeFramesOrChunks and testFinalizedFrameCountIsBatchExact
    on the restatement: every feeding size gives the same frames, as many as batch .center."""
    cfg = oracle.mel_config()
    audio = synth.tone_noise_audio(AUDIO_12S)
    streams = [feed(MelStreamSession(cfg, oracle_mel_fn(oracle, cfg)), audio, s) for s in FEEDS]
    expected = 1 + (audio.size + cfg.n_fft - cfg.win_length) // cfg.hop_length
    for s, rows in zip(FEEDS, streams):
        assert rows.shape == (expected, cfg.n_mels), s
        assert np.array_equal(rows, streams[-1]), s


def test_restated_stream_matches_batch_center(oracle):
    """testStreamedMelMatchesBatchValues: every streamed frame within 1e-5 of the oracle's .center output."""
    cfg = oracle.mel_config()
    audio = synth.tone_noise_audio(AUDIO_12S)
    rows = feed(MelStreamSession(cfg, oracle_mel_fn(oracle, cfg)), audio, 1600)
    ref, ml, nf = oracle.mel_flat_transposed(cfg, audio)
    assert rows.shape[0] == ml == nf
    assert float(np.abs(rows - ref).max()) <= 1e-5


def test_restated_stream_drops_audio_after_finish_and_restarts(oracle):
    """testResetAfterExhaustionRestartsMelStream / testResetRestartsMelStream."""
    cfg = oracle.mel_config()
    audio = synth.tone_noise_audio(16000 * 6 + 137)
    s = MelStreamSession(cfg, oracle_mel_fn(oracle, cfg))
    first = s.push(audio)
    s.push(np.zeros(0, np.float32), finish=True)
    emitted = s.emitted
    assert s.push(audio).shape[0] == 0 and s.emitted == emitted
    s.reset()   # fa_mel_stream_close + fa_mel_stream_open
    assert np.array_equal(s.push(audio), first)


def test_frame_count_rule_matches_restatement(oracle):
    """stream_frames (the rule fa_mel_stream_frames implements) predicts every push of the restatement, over random
    chunkings with empty pushes, pushes below win/2 and finish without audio."""
    rng = random.Random(5)
    for cfg in (oracle.mel_config(), oracle.mel_config(n_fft=256, win_length=200, hop_length=80),
                oracle.mel_config(hop_length=400), oracle.mel_config(hop_length=161, preemph=0.0)):
        count_only = lambda buf, last, count: np.zeros((count, cfg.n_mels), np.float32)
        for trial in range(40):
            s = MelStreamSession(cfg, count_only)
            for _ in range(rng.randrange(0, 12)):
                n = rng.choice((0, 0, 1, 7, cfg.win_length // 2 - 1, cfg.win_length // 2, 159, 160, 161, 1600, 4093))
                fin = rng.random() < 0.1
                want = stream_frames(cfg, s.received, s.emitted, s.finished, n, fin)
                assert s.push(np.ones(n, np.float32), finish=fin).shape[0] == want
            want = stream_frames(cfg, s.received, s.emitted, s.finished, 0, True)
            assert s.push(np.zeros(0, np.float32), finish=True).shape[0] == want


def test_stream_entry_points_reject_null_handle():
    """The library loads without a GPU; the session entry points check the handle first."""
    L = _lib.load()
    sid = C.c_int32()
    assert L.fa_mel_stream_open(None, C.byref(sid)) == INVALID
    assert L.fa_mel_stream_close(None, 0) == INVALID
    assert L.fa_mel_stream_frames(None, 0, 160, 0) == -1
    frames = np.zeros(1, np.int64)
    for f in (L.fa_mel_stream_push, L.fa_mel_stream_push_device):
        assert f(None, 0, None, None, None, None, None, 0, frames.ctypes.data) == INVALID


# ================================================================================================ GPU
from fluidaudio_b200.mel import AudioMelSpectrogram, MelStreams, Precision   # noqa: E402

CONFIGS = {
    "default": {},
    "mels80": dict(n_mels=80),
    "preemph0": dict(preemph=0.0),
    "odd_hop": dict(hop_length=161),                               # mel_generic_kernel
    "nfft256": dict(n_fft=256, win_length=200, hop_length=80),     # mel_generic_kernel
    "hop_eq_win": dict(hop_length=400),
}
PRECISIONS = (Precision.f64, Precision.f32)


def gpu_mel_fn(m):
    def f(buf, last, count):
        out, ml, nf = m.compute_flat_transposed(buf, last_audio_sample=float(last), padding_mode=PRE_PADDED,
                                                expected_frame_count=count)
        assert ml == count == nf
        return out.reshape(count, m.n_mels).copy()
    return f


def chunking(n, seed):
    rng = random.Random(seed)
    sizes, at = [], 0
    while at < n:
        k = min(n - at, rng.choice((0, 1, 7, 159, 160, 161, 1600, 2560, 4093, 10080)))
        sizes.append(k)
        at += k
    return sizes


def run_pair(key, prec, seed=3, seconds=3):
    """The same audio through MelStreams and through the restatement driving fa_mel_compute; the last push carries samples
    and finishes.  Returns (per-push library rows, per-push restatement rows, the handle)."""
    m = AudioMelSpectrogram(**CONFIGS[key], precision=prec)
    streams = MelStreams(m)
    sid = streams.open()
    ref = MelStreamSession(m, gpu_mel_fn(m))
    audio = synth.tone_noise_audio(16000 * seconds + 137, seed=seed)
    got, want, at = [], [], 0
    sizes = chunking(audio.size, seed)
    for i, k in enumerate(sizes):
        fin = i == len(sizes) - 1
        x = audio[at:at + k]
        at += k
        assert streams.pending_frames(sid, k, fin) == stream_frames(m, ref.received, ref.emitted, ref.finished, k, fin)
        got.append(streams.push({sid: x}, finish=(sid,) if fin else ())[sid].copy())
        want.append(ref.push(x, finish=fin))
    return got, want, m


@pytest.mark.gpu
@pytest.mark.parametrize("prec", PRECISIONS, ids=lambda p: p.name)
@pytest.mark.parametrize("key", list(CONFIGS))
def test_stream_equals_swift_call_sequence(gpu_lib, key, prec):
    """Every push's rows equal fa_mel_compute(buffer, last, .prePadded, expected=count) on the restatement's buffer."""
    got, want, m = run_pair(key, prec)
    assert sum(g.shape[0] for g in got) == 1 + (16000 * 3 + 137 + m.n_fft - m.win_length) // m.hop_length
    for i, (g, w) in enumerate(zip(got, want)):
        assert g.shape == w.shape and np.array_equal(g, w), (key, prec, "push", i)


def fp64_bar(r, top):
    return 1e-5 + 4e-7 * np.abs(r)


def f32_bar(r, top):   # tests/test_gpu_mel_sweep.py: 1e-4, widened more than 12 nats below the frame's strongest mel
    return np.minimum(2e-3, 1e-4 * np.maximum(1.0, np.exp(top - r - 12.0)))


@pytest.mark.gpu
@pytest.mark.parametrize("prec", PRECISIONS, ids=lambda p: p.name)
@pytest.mark.parametrize("key", list(CONFIGS))
def test_stream_within_oracle_bars(gpu_lib, oracle, key, prec):
    got, _, m = run_pair(key, prec)
    cfg = oracle.mel_config(**CONFIGS[key])
    ref = MelStreamSession(cfg, oracle_mel_fn(oracle, cfg))
    audio = synth.tone_noise_audio(16000 * 3 + 137, seed=3)
    sizes = chunking(audio.size, 3)
    want = feed_sizes(ref, audio, sizes)
    g = np.concatenate(got)
    generic = m.n_fft != 512 or m.hop_length % 2
    bar = f32_bar if (prec == Precision.f32 and not generic) else fp64_bar
    top = np.broadcast_to(want.max(axis=1, keepdims=True), want.shape)
    d = np.abs(g - want)
    assert not (d > bar(want, top)).any(), (key, prec, float(d.max()))


def feed_sizes(session, audio, sizes):
    rows, at = [], 0
    for i, k in enumerate(sizes):
        rows.append(session.push(audio[at:at + k], finish=i == len(sizes) - 1))
        at += k
    return np.concatenate(rows)


@pytest.mark.gpu
@pytest.mark.parametrize("prec", PRECISIONS, ids=lambda p: p.name)
@pytest.mark.parametrize("key", ["default", "nfft256"])
def test_stream_granularity_and_batch_equivalence(gpu_lib, key, prec):
    m = AudioMelSpectrogram(**CONFIGS[key], precision=prec)
    assert (m.n_fft - m.win_length) // 2 >= 1
    streams = MelStreams(m)
    audio = synth.tone_noise_audio(AUDIO_12S)
    outs = []
    for size in FEEDS:
        sid = streams.open()
        size = size or audio.size
        rows = [streams.push({sid: audio[i:i + size]})[sid].copy() for i in range(0, audio.size, size)]
        rows.append(streams.push({}, finish=(sid,))[sid].copy())
        streams.close(sid)
        outs.append(np.concatenate(rows))
    for size, o in zip(FEEDS, outs):
        assert np.array_equal(o, outs[-1]), (key, prec, size)
    batch, ml, nf = m.compute_flat_transposed(audio)
    batch = batch.reshape(nf, m.n_mels)
    s = outs[-1]
    assert s.shape[0] == ml == nf
    # frame k's window ends (exclusive) at audio index k*hop + (nFFT - win)/2 + win - nFFT/2
    k = np.arange(nf)
    covered = k * m.hop_length + (m.n_fft - m.win_length) // 2 + m.win_length - m.n_fft // 2 <= audio.size
    assert covered.sum() > nf - 8
    assert np.array_equal(s[covered], batch[covered])
    d = np.abs(s[~covered] - batch[~covered])
    if prec == Precision.f64 or m.n_fft != 512:
        assert float(d.max()) <= 1e-5, float(d.max())
    else:
        top = np.broadcast_to(batch[~covered].max(axis=1, keepdims=True), d.shape)
        assert not (d > f32_bar(batch[~covered], top)).any(), float(d.max())


CHUNKS = (0, 1, 7, 159, 160, 161, 1600, 2560, 10080, 20480)


def replay_alone(m, events):
    """One logical session's pushes, run alone on its own handle."""
    streams = MelStreams(m)
    sid = streams.open()
    rows = [streams.push({sid: x}, finish=(sid,) if fin else ())[sid].copy() for x, fin in events]
    streams.close(sid)
    return rows


@pytest.mark.gpu
@pytest.mark.parametrize("prec", PRECISIONS, ids=lambda p: p.name)
def test_many_sessions_match_sessions_run_alone(gpu_lib, prec):
    """~1000 sessions, random subsets per push, interleaved finish / close / open with ids reused: every session's stream
    is bit-identical to the same session run alone."""
    rng = random.Random(11 if prec == Precision.f64 else 12)
    m = AudioMelSpectrogram(precision=prec)
    solo = AudioMelSpectrogram(precision=prec)
    streams = MelStreams(m)
    live = {}      # id -> logical stream index
    logs = []      # per logical stream: (events, rows)
    finished = set()
    for _ in range(1000):
        sid = streams.open()
        live[sid] = len(logs)
        logs.append(([], []))
    seed = 0
    reused = 0
    for tick in range(24):
        ids = [s for s in live if rng.random() < 0.4]
        chunks, fin = {}, []
        for s in ids:
            n = rng.choice(CHUNKS)
            seed += 1
            chunks[s] = synth.tone_noise_audio(n, seed=seed)
            if rng.random() < 0.05:
                fin.append(s)
        out = streams.push(chunks, finish=fin)
        for s in ids:
            logs[live[s]][0].append((chunks[s], s in fin))
            logs[live[s]][1].append(out[s].copy())
        finished.update(fin)
        for s in [s for s in live if s in finished and rng.random() < 0.5]:   # close some finished sessions, reopen
            streams.close(s)
            del live[s]
            finished.discard(s)
            nid = streams.open()
            assert nid == s   # the lowest free id: this one
            reused += 1
            live[nid] = len(logs)
            logs.append(([], []))
    assert reused > 10
    for events, rows in logs:
        if not events:
            continue
        alone = replay_alone(solo, events)
        for a, b in zip(rows, alone):
            assert a.shape == b.shape and np.array_equal(a, b)


@pytest.mark.gpu
@pytest.mark.parametrize("sessions", (1, 1000))
def test_launches_per_push(gpu_lib, sessions):
    m = AudioMelSpectrogram()
    streams = MelStreams(m)
    ids = [streams.open() for _ in range(sessions)]
    x = synth.tone_noise_audio(100)   # below win/2: no frame
    before = _lib.kernel_launch_count()
    out = streams.push({s: x for s in ids})
    assert all(v.shape[0] == 0 for v in out.values())
    assert _lib.kernel_launch_count() - before == 1
    y = synth.tone_noise_audio(1600)
    for _ in range(3):
        before = _lib.kernel_launch_count()
        out = streams.push({s: y for s in ids})
        assert all(v.shape[0] >= 9 for v in out.values())
        assert _lib.kernel_launch_count() - before <= 2


def _device_push(streams, dbufs, ids, chunks, fin, d_out, row):
    """Upload chunks into a fresh device buffer (kept alive in dbufs) and push them asynchronously."""
    audio = np.concatenate(chunks)
    offsets = np.zeros(len(ids) + 1, np.int64)
    offsets[1:] = np.cumsum([c.size for c in chunks])
    d = _lib.DeviceBuffer(max(4, audio.nbytes))
    d.upload(audio)
    dbufs.append(d)
    return streams.push_device(ids, d, offsets, d_out, finish=fin, out_offset=row * streams.n_mels)


@pytest.mark.gpu
def test_push_device_matches_push_and_back_to_back(gpu_lib):
    """push_device is bit-identical to push; three device pushes with no synchronisation in between, the first queued
    behind a one-hour fa_mel_compute_device on the same handle, give what synchronised pushes give."""
    S = 64
    host_m, dev_m = AudioMelSpectrogram(), AudioMelSpectrogram()
    hs, ds = MelStreams(host_m), MelStreams(dev_m)
    hid = [hs.open() for _ in range(S)]
    did = [ds.open() for _ in range(S)]
    rng = np.random.default_rng(2)
    hour = 16000 * 3600
    d_hour = _lib.DeviceBuffer(hour * 4)
    d_hour.upload(np.zeros(hour, np.float32))
    d_hour_out = _lib.DeviceBuffer(dev_m.frame_count(hour) * dev_m.n_mels * 4)
    d_out = _lib.DeviceBuffer(4 * 128 * 300 * S)
    dbufs, want, rows, counts = [], [], 0, []
    for p in range(4):
        sizes = rng.choice([0, 160, 1601, 10080], S)
        chunks = [synth.tone_noise_audio(int(n), seed=100 * p + i) for i, n in enumerate(sizes)]
        fin = [1 if (p == 3 and i % 2) else 0 for i in range(S)]
        h = hs.push({s: c for s, c in zip(hid, chunks)}, finish=[s for s, f in zip(hid, fin) if f])
        want.append(np.concatenate([h[s] for s in hid]))
        if p == 1:   # the next three device pushes run back to back behind the hour
            dev_m.compute_device(d_hour, hour, d_hour_out, padding_mode=PRE_PADDED)
        fr = _device_push(ds, dbufs, did, chunks, fin, d_out, rows)
        counts.append(int(fr.sum()))
        assert counts[-1] == want[-1].shape[0]
        rows += counts[-1]
        if p == 0:
            _lib.synchronize()
    _lib.synchronize()
    got = d_out.download((rows, 128), np.float32)
    assert np.array_equal(got, np.concatenate(want))


@pytest.mark.gpu
def test_failed_pushes_change_nothing(gpu_lib):
    m, twin = AudioMelSpectrogram(), AudioMelSpectrogram()
    a, b = MelStreams(m), MelStreams(twin)
    ids = [a.open() for _ in range(4)]
    assert [b.open() for _ in range(4)] == ids
    a.close(3)
    b.close(3)
    x = [synth.tone_noise_audio(1600, seed=i) for i in range(3)]
    first = a.push({0: x[0], 1: x[1]})
    assert all(np.array_equal(first[s], v) for s, v in b.push({0: x[0], 1: x[1]}).items())
    L = m._L
    audio = np.concatenate(x)
    out = np.zeros(128 * 1000, np.float32)
    frames = np.zeros(3, np.int64)

    def raw(sessions, offsets, out_len=out.size):
        s = np.array(sessions, np.int32)
        o = np.array(offsets, np.int64)
        return L.fa_mel_stream_push(m._h, s.size, s.ctypes.data, audio.ctypes.data, o.ctypes.data, None,
                                    out.ctypes.data, out_len, frames.ctypes.data)

    assert raw([0, 1, 0], [0, 1600, 3200, 4800]) == INVALID            # duplicate id
    assert raw([0, 3], [0, 1600, 3200]) == INVALID                     # closed id
    assert raw([0, 1, 2], [0, 3200, 1600, 4800]) == INVALID            # offsets decrease
    assert raw([0, 1, 2], [0, 1600, 3200, 4800], out_len=128) == TOO_SMALL
    assert raw([0, 7], [0, 1600, 3200]) == INVALID                     # never opened
    nxt = a.push({0: x[2], 1: x[0], 2: x[1]}, finish=(1,))
    ref = b.push({0: x[2], 1: x[0], 2: x[1]}, finish=(1,))
    for s in ref:
        assert np.array_equal(nxt[s], ref[s])
    for bad in (dict(pad_to=2), dict(hop_length=401)):
        sid = C.c_int32()
        assert L.fa_mel_stream_open(AudioMelSpectrogram(**bad)._h, C.byref(sid)) == INVALID


@pytest.mark.gpu
@pytest.mark.parametrize("prec", PRECISIONS, ids=lambda p: p.name)
def test_nan_chunk_stays_in_its_frames(gpu_lib, prec):
    m = AudioMelSpectrogram(precision=prec)
    streams = MelStreams(m)
    s0, s1 = streams.open(), streams.open()
    ref = MelStreamSession(m, gpu_mel_fn(m))
    audio = synth.tone_noise_audio(16000 * 2, seed=4)
    other = synth.tone_noise_audio(16000 * 2, seed=5)
    nan_at = 5000 + 17
    audio[nan_at] = np.nan
    got, want, other_rows = [], [], []
    for i in range(0, audio.size, 1600):
        fin = i + 1600 >= audio.size
        out = streams.push({s0: audio[i:i + 1600], s1: other[i:i + 1600]}, finish=(s0, s1) if fin else ())
        got.append(out[s0].copy())
        other_rows.append(out[s1].copy())
        want.append(ref.push(audio[i:i + 1600], finish=fin))
    g, w = np.concatenate(got), np.concatenate(want)
    assert np.array_equal(g, w, equal_nan=True)
    start = np.arange(g.shape[0]) * m.hop_length + (m.n_fft - m.win_length) // 2 - m.n_fft // 2
    holds = (start - 1 <= nan_at) & (nan_at < start + m.win_length)   # the window, and the sample pre-emphasis reads first
    assert np.array_equal(np.isnan(g).any(axis=1), holds) and holds.any()
    assert np.isfinite(g[np.flatnonzero(holds)[-1] + 1:]).all()
    alone = replay_alone(AudioMelSpectrogram(precision=prec),
                         [(other[i:i + 1600], i + 1600 >= other.size) for i in range(0, other.size, 1600)])
    assert all(np.array_equal(a, b) for a, b in zip(other_rows, alone))
