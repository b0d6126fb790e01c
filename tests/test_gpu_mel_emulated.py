"""mel512_kernel against the host emulation of its own arithmetic (run with ``-m gpu`` on an H100).

tests/mel_lane_emulated.py states the comparison and its bars.  Float32 pairs (``Precision.f32``): the emulated log
argument x is the device's bit for bit, so the only tolerance is the device log's, |y - ln x| <= 4u ln 2 + 6u |ln x|; x = 0
must give -inf, x NaN NaN (the NaN pattern of the quad-rounded bands, not the oracle's dense rule), x inf inf.  FP64
transform: the bar derived there from mel_ex_restated.py's steps 2 to 6 for two evaluations that differ only in nvcc's
double contractions.  Only configurations the plan gives to mel512_kernel are compared (``plan_kernel``), and each test
asserts how many it covered per precision.  The worst deviation as a fraction of the bar is printed per precision and
layout.
"""
import random

import numpy as np
import pytest

import mel_lane_emulated as ME
from fluidaudio_b200 import _lib, synth
from fluidaudio_b200.mel import AudioMelSpectrogram, MelStreams, Precision
from test_gpu_mel_sweep import _View, plan_kernel
from test_mel_stream import MelStreamSession, chunking, stream_frames

pytestmark = pytest.mark.gpu

CENTER, PRE_PADDED, LEGACY = ME.CENTER, ME.PRE_PADDED, ME.LEGACY
TIME_MAJOR, MEL_MAJOR = ME.TIME_MAJOR, ME.MEL_MAJOR
WORST = {}     # (precision, layout) -> worst fraction of the bar


def _note(prec, layout, frac):
    key = f"{prec.name} {'time-major' if layout == TIME_MAJOR else 'mel-major'}"
    WORST[key] = max(WORST.get(key, 0.0), frac)


@pytest.fixture(scope="module", autouse=True)
def report():
    yield
    print("\nworst |y - ln x| / bar per precision and layout:", {k: round(v, 3) for k, v in sorted(WORST.items())})


class Emu:
    """A handle and its emulation: the handle's own window and filterbank, and the log floor and floor mode it was made
    with (AudioMelSpectrogram does not keep them)."""

    def __init__(self, sr=16000, n_mels=80, hop=160, win=400, preemph=0.97, floor=2.0 ** -24, clamped=0,
                 precision=Precision.f32):
        self.m = AudioMelSpectrogram(sample_rate=sr, n_mels=n_mels, hop_length=hop, win_length=win, preemph=preemph,
                                     log_floor=floor, log_floor_mode=clamped, precision=precision)
        self.floor, self.clamped = float(np.float32(floor)), clamped
        self.window = self.m.get_hann_window()
        self.fb = self.m.get_filterbank()

    def args(self, mode):
        """(window offset, centre pad, pre-emphasis) of a call in ``mode``."""
        return ME.placement(dict(win=self.m.win_length, preemph=self.m.preemph), mode)

    def run(self, x, last, mode, T, power=False):
        off, pad, pre = self.args(mode)
        m = self.m
        return ME.lane_frames(m.precision == Precision.f32, x, last, m.hop_length, self.window, off, pad, pre, self.fb,
                              self.floor, self.clamped, T, power=power)

    def check(self, y, x, last, mode, layout, what):
        """y: [T x M] device rows of ``x`` in ``mode``; compares within the precision's bar."""
        m = self.m
        T = y.shape[0]
        f32 = m.precision == Precision.f32
        P, E, xa, _ = self.run(x, last, mode, T, power=not f32)
        if f32:
            frac = ME.check_f32(y, xa, what)
        else:
            off, pad, pre = self.args(mode)
            S = ME.frame_abs_sums(x, last, m.hop_length, self.window, off, pad, pre, T)
            frac = ME.check_f64(y, E, xa, P, S, self.fb, self.floor, self.clamped, what)
        _note(m.precision, layout, frac)


def rows(m, x, last, mode, layout):
    out, ml, nf = m._run(x, last, mode, None, layout)
    y = out[: ml * m.n_mels]
    return (y.reshape(ml, m.n_mels) if layout == TIME_MAJOR else y.reshape(m.n_mels, -1)[:, :ml].T), ml


# ================================================================================================ axes
def test_every_even_hop(gpu_lib):
    """Every even hop from 2 to past the plan's switch to the any-nFFT kernel, both precisions, two clips each: a short
    .center clip (every tile takes the edge pre-emphasis) and a 33-frame .prePadded clip, whose second tile lies inside the
    clip and so takes the interior pre-emphasis: the float4 steps at hops 0 mod 4, the scalar loop at hops 2 mod 4.  Only
    mel512 hops are compared, all of 2..860."""
    covered = {Precision.f32: 0, Precision.f64: 0}
    for hop in range(2, 961, 2):
        e = Emu(hop=hop)
        m = e.m
        if plan_kernel(m) != "mel512":
            assert hop > 860, hop
            m.close()
            continue
        clips = [(CENTER, synth.tone_noise_audio(ME.length_for(ME.FRAMES[hop // 2 % 7], hop, 400, CENTER), seed=hop)),
                 (PRE_PADDED, synth.tone_noise_audio(ME.length_for(33, hop, 400, PRE_PADDED), seed=hop + 1))]
        for prec in (Precision.f32, Precision.f64):
            m.set_precision(prec)
            for mode, x in clips:
                y, ml = rows(m, x, 0.1, mode, TIME_MAJOR)
                assert ml == ME.frame_count(x.size, hop, 400, mode)
                e.check(y, x, 0.1, mode, TIME_MAJOR, dict(hop=hop, mode=mode, precision=prec.name))
            covered[prec] += 1
        m.close()
    print("\neven hops on mel512_kernel per precision:", {p.name: v for p, v in covered.items()})
    assert covered[Precision.f32] == covered[Precision.f64] >= 430, covered


def test_configuration_cross_product(gpu_lib):
    """Window (both sides of mid_full, centred and at offset 0) x rate x floor mode x log floor, with the mel count, hop,
    pre-emphasis (0 too: the plain copy path), frame count, signal and mode dealt round robin, a non-zero `last`, both
    layouts and both precisions; then subnormal power at every mel count under a log floor of 0."""
    cases = ME.cross_cases()
    covered = {Precision.f32: 0, Precision.f64: 0}
    for c in cases:
        e = Emu(sr=c["sr"], n_mels=c["n_mels"], hop=c["hop"], win=c["win"], preemph=c["preemph"], floor=c["floor"],
                clamped=c["clamped"])
        m = e.m
        if plan_kernel(m) != "mel512":
            m.close()
            continue
        n = ME.length_for(c["frames"], c["hop"], c["win"], c["mode"])
        x = ME.signal(c["signal"], n, c["seed"], c["sr"])
        for prec in (Precision.f32, Precision.f64):
            m.set_precision(prec)
            for layout in (TIME_MAJOR, MEL_MAJOR):
                y, ml = rows(m, x, c["last"], c["mode"], layout)
                assert ml == ME.frame_count(n, c["hop"], c["win"], c["mode"]), c
                e.check(y, x, c["last"], c["mode"], layout, dict(c, precision=prec.name, layout=layout))
            covered[prec] += 1
        m.close()
    print("\ncross-product configurations on mel512_kernel per precision:", {p.name: v for p, v in covered.items()})
    assert covered[Precision.f32] == covered[Precision.f64] == len(cases), covered


# ================================================================================================ entry points
def test_device_input_at_four_bytes(gpu_lib):
    """compute_device with the input at +4 bytes: no bulk copy, every tile takes the edge pre-emphasis."""
    for kw in (dict(), dict(n_mels=81, hop=158, win=383), dict(n_mels=128, hop=256, win=512, clamped=1, floor=0.0)):
        e = Emu(**kw)
        m = e.m
        a = synth.speech_like_audio(16000 * 2 + 37, seed=5)
        for prec in (Precision.f32, Precision.f64):
            m.set_precision(prec)
            T = m.frame_count(a.size)
            d_in = _lib.DeviceBuffer(a.nbytes + 64)
            d_in.upload(np.concatenate([np.zeros(1, np.float32), a]))
            d_out = _lib.DeviceBuffer(T * m.n_mels * 4)
            assert m.compute_device(_View(d_in, 4), a.size, d_out, last_audio_sample=0.25)[0] == T
            _lib.synchronize()
            y = d_out.download((T, m.n_mels), np.float32)
            e.check(y, a, 0.25, CENTER, TIME_MAJOR, dict(kw, precision=prec.name))
            d_in.free()
            d_out.free()
        m.close()


def _tiny_clips(hop, win, count, seed):
    rng = np.random.default_rng(seed)
    frames = rng.integers(1, 34, count)
    lens = np.array([ME.length_for(int(f), hop, win, CENTER) for f in frames], np.int64) + rng.integers(0, 5, count)
    base = synth.tone_noise_audio(1 << 20, seed=seed)
    starts = rng.integers(0, base.size - int(lens.max()), count)
    offsets = np.zeros(count + 1, np.int64)
    offsets[1:] = np.cumsum(lens)
    packed = np.concatenate([base[s:s + n] for s, n in zip(starts, lens)])
    last = rng.uniform(-0.5, 0.5, count).astype(np.float32)
    return packed, offsets, last


def test_batches_of_tiny_clips(gpu_lib):
    """compute_batch with 3 000 clips of 1..33 frames, each with its own `last` (CTAs hand over between units), and
    compute_batch_device with no clip starting at a multiple of four floats (no bulk copy); float32 pairs, every clip."""
    e = Emu(n_mels=80)
    m = e.m
    packed, offsets, last = _tiny_clips(160, 400, 3000, 31)
    out, offs, ml, nf = m.compute_batch(None, last_samples=last, packed_audio=packed, offsets=offsets)
    for i in range(offsets.size - 1):
        x = packed[offsets[i]:offsets[i + 1]]
        e.check(out[offs[i]:offs[i] + ml[i] * 80].reshape(ml[i], 80), x, float(last[i]), CENTER, TIME_MAJOR, ("batch", i))
    # The device batch reads clip k as d_audio[bounds[k]:bounds[k + 1]], so every clip ends where the next one starts.
    # Between the first 700 clips of the host batch sit one-sample clips of silence: clip 2i is host clip i, clip 2i + 1
    # is one zero, and host clip i starts at its host offset + i, so the clip starts take every residue mod 4 and the
    # launch moves every sample through the read-only path.  No `last` (zero).  The outputs follow each other with one
    # float between consecutive ones, so their offsets take every residue mod 4 too (no float4 copy-out).
    count = 700
    real = offsets[:count] + np.arange(count)
    bounds = np.empty(2 * count + 1, np.int64)
    bounds[0:2 * count:2] = real
    bounds[1:2 * count:2] = real + np.diff(offsets[:count + 1])
    bounds[2 * count] = bounds[2 * count - 1] + 1
    buf = np.zeros(int(bounds[-1]) + 8, np.float32)
    for i in range(count):
        buf[bounds[2 * i]:bounds[2 * i + 1]] = packed[offsets[i]:offsets[i + 1]]
    d_a = _lib.DeviceBuffer(buf.nbytes)
    d_a.upload(buf)
    Ts = np.array([m.frame_count(int(n)) for n in np.diff(bounds)])
    out_off = np.zeros(2 * count + 1, np.int64)
    out_off[1:] = np.cumsum(np.maximum(Ts, 1) * 80 + 1)
    d_o = _lib.DeviceBuffer(int(out_off[-1]) * 4 + 64)
    ml2, nf2 = m.compute_batch_device(d_a, bounds, d_o, out_off)
    _lib.synchronize()
    got = d_o.download((int(out_off[-1]),), np.float32)
    assert np.array_equal(ml2[0::2], ml[:count]) and (ml2[1::2] == 1).all()
    for k in range(2 * count):
        x = buf[bounds[k]:bounds[k + 1]]
        e.check(got[out_off[k]:out_off[k] + ml2[k] * 80].reshape(ml2[k], 80), x, 0.0, CENTER, TIME_MAJOR, ("device", k))
    d_a.free()
    d_o.free()
    m.close()


def test_stream_sessions(gpu_lib):
    """MelStreams: three dozen sessions advanced together across random chunkings; every push's rows against
    MelStreamSession (tests/test_mel_stream.py) driven by the emulation instead of fa_mel_compute, so each row is held to
    the emulated log argument of the very buffer and `last` the reference's session would compute it from."""
    e = Emu(n_mels=80)
    m = e.m
    streams = MelStreams(m)
    sessions = 36
    emulated = {}

    def emu_fn(buf, last, count):
        _, _, x, _ = e.run(buf, last, PRE_PADDED, count)
        emulated.setdefault("rows", 0)
        emulated["rows"] += count
        return x

    ids = [streams.open() for _ in range(sessions)]
    refs = {s: MelStreamSession(m, emu_fn) for s in ids}
    audio = {s: synth.tone_noise_audio(16000 * 2 + 37 * k, seed=40 + k) for k, s in enumerate(ids)}
    plans = {s: chunking(audio[s].size, 100 + k) for k, s in enumerate(ids)}
    at = {s: 0 for s in ids}
    step = 0
    while any(plans.values()):
        chunks, fin = {}, []
        for s in ids:
            if plans[s] and random.Random(step * 97 + s).random() < 0.8:
                k = plans[s].pop(0)
                chunks[s] = audio[s][at[s]:at[s] + k]
                at[s] += k
                if not plans[s]:
                    fin.append(s)
        if not chunks:
            step += 1
            continue
        for s in chunks:
            assert streams.pending_frames(s, chunks[s].size, s in fin) == stream_frames(
                m, refs[s].received, refs[s].emitted, refs[s].finished, chunks[s].size, s in fin)
        got = streams.push(chunks, finish=fin)
        for s in chunks:
            x = refs[s].push(chunks[s], finish=s in fin)
            assert got[s].shape == x.shape, (s, step)
            _note(Precision.f32, TIME_MAJOR, ME.check_f32(got[s], x, ("stream", s, step)))
        step += 1
    assert all(r.finished for r in refs.values()) and emulated["rows"] >= sessions * 190
    m.close()


def test_ten_minute_clip(gpu_lib):
    """One 10-minute clip: the persistent grid, many tiles per CTA, the bulk copies' double-buffer parity; every row."""
    e = Emu(n_mels=80)
    m = e.m
    x = synth.speech_like_audio(16000 * 600 + 91, seed=17)
    for layout in (TIME_MAJOR, MEL_MAJOR):
        y, ml = rows(m, x, -0.2, CENTER, layout)
        assert ml == m.frame_count(x.size) > 60_000
        if layout == TIME_MAJOR:
            ref = y
            e.check(y, x, -0.2, CENTER, layout, "10 min")
        else:
            assert np.array_equal(y, ref)   # the mel-major copy-out of the same rows
    m.close()


def test_bench_hour(gpu_lib):
    """The hour bench.py times (BASELINE configs[1]: 16 kHz tone + noise, seed 7, 80 mels, float32 pairs) from HBM,
    every one of its 360 001 rows against one emulation of the whole hour."""
    n = 16000 * 3600
    e = Emu(n_mels=80)
    m = e.m
    x = synth.tone_noise_audio(n, seed=7)
    T = m.frame_count(n)
    assert T == 360_001
    d_in = _lib.DeviceBuffer(x.nbytes + 64)
    d_in.upload(x)
    d_out = _lib.DeviceBuffer(T * 80 * 4)
    assert m.compute_device(d_in, n, d_out)[0] == T
    _lib.synchronize()
    y = d_out.download((T, 80), np.float32)
    d_in.free()
    d_out.free()
    e.check(y, x, 0.0, CENTER, TIME_MAJOR, "hour")
    m.close()
