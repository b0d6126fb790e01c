"""The torch-style log-mel frontends on the H100 (``-m gpu``): Cohere, StyleTTS2 and LuxTTS handles.

Bit for bit, on one handle, so that no transform error enters:
* the preset tables (``fa_mel_get_window`` / ``fa_mel_get_filterbank``) equal the oracle's;
* a handle from ``fa_mel_ex_default_config`` equals ``fa_mel_create`` on every precision, layout and padding mode;
* reflect ``.center`` equals ``.prePadded`` on the host-reflect-padded clip; the affine output equals numpy float32
  ``(L - mean) / std`` of the same configuration's log-mel ``L``; ``fa_mel_cohere_features`` equals ``oracle_torch.cohere_cmvn``
  (CMVN + padOrTruncate) of the handle's own log-mel, for fixed_frames below, at and above valid and valid 0, 1, 2;
* batches equal per-clip calls and device buffers equal host buffers, including chunked host-pipeline calls.

Against the oracle (oracle_mel_torch.cpp through oracle/oracle_torch.py): the generic-kernel bar 1e-5 + 4e-7 |r| in the log domain, divided by
``log_std`` for StyleTTS2; for Cohere the first-order CMVN bar of test_gpu_mel_adapter_sweep.py, with the library's
log-mel standing in for the oracle's in the bar's magnitudes.  Pre-emphasis: the library runs one fused multiply-add per
sample, the reference rounds the product and the difference separately.  The test measures what that changes in the
Cohere log-mel and keeps it inside the bar.  The worst |d| / bar is printed per bar (``-s``).
"""
import ctypes as C

import numpy as np
import pytest

from fluidaudio_b200 import _lib, synth
from oracle import oracle_torch as OT
from fluidaudio_b200.mel import (AudioMelSpectrogram, CohereMelSpectrogram, LuxTtsMelExtractor, Precision,
                                 StyleTTS2MelExtractor, ex_config)

pytestmark = pytest.mark.gpu
F32 = np.float32
CENTER, PRE_PADDED, LEGACY = 0, 1, 2
TIME_MAJOR, MEL_MAJOR = 0, 1
WORST = {}


def _note(key, frac):
    WORST[key] = max(WORST.get(key, 0.0), float(frac))
    print(f"  worst |d| / bar so far: " + ", ".join(f"{k} {v:.3g}" for k, v in sorted(WORST.items())))


def same_bits(a, b):
    a, b = np.asarray(a, F32), np.asarray(b, F32)
    if a.shape != b.shape:
        return False
    na, nb = np.isnan(a), np.isnan(b)
    return bool(np.array_equal(na, nb) and np.array_equal(a[~na].view(np.uint32), b[~nb].view(np.uint32)))


def _signal(kind, n, rate, seed=0):
    rng = np.random.default_rng(seed + n)
    if kind == "noise":
        return (rng.standard_normal(n) * 0.3).astype(F32)
    if kind == "speech":
        return synth.speech_like_audio(n, sample_rate=rate) if n else np.zeros(0, F32)
    if kind == "silence":
        return np.zeros(n, F32)
    x = (rng.standard_normal(n) * 0.3).astype(F32)
    if kind == "nan" and n:
        x[n // 2] = np.nan
    if kind == "overflow" and n:
        x[n // 3] = F32(3e38)
    return x


def _lengths(n_fft, hop, rate):
    return sorted({0, 1, 2, n_fft // 2 - 1, n_fft // 2, n_fft // 2 + 1, 5 * hop - 1, 5 * hop, 5 * hop + 1, 10 * rate})


def _log_mel(mel, audio, T, layout=TIME_MAJOR, mode=CENTER):
    """The handle's plain log-mel of exactly T frames (fa_mel_compute with an expected count)."""
    out, ml, nf = mel._run(audio, 0.0, mode, T, layout)
    assert ml == nf == T
    return out[:T * mel.n_mels].reshape((T, mel.n_mels) if layout == TIME_MAJOR else (mel.n_mels, T))


def _launches(fn):
    before = _lib.kernel_launch_count()
    r = fn()
    return r, _lib.kernel_launch_count() - before


def _bar(r_log):
    return 1e-5 + 4e-7 * np.abs(r_log)


def _check_bar(got, ref, bar, key, what):
    """Non-finite only where the oracle is, finite entries within the bar.  The oracle can be non-finite where the library
    is not, in two stated ways (DESIGN §2): the Swift multiplies the whole nFFT span by the zero-padded window, so a NaN
    outside the window but inside the span poisons its frame (0 * NaN); and its dense table product turns an overflowing
    bin into NaN in every mel (0 * inf), where the kernels read each filter's band only."""
    assert not (~np.isfinite(got) & np.isfinite(ref)).any(), (what, "non-finite where the oracle is finite")
    fin = np.isfinite(got) & np.isfinite(ref)
    if fin.any():
        frac = (np.abs(got[fin].astype(np.float64) - ref[fin]) / bar[fin]).max()
        _note(key, frac)
        assert frac <= 1.0, (what, float(frac))


# ================================================================================================ tables, neutrality
def test_preset_tables_equal_the_oracle(gpu_lib, oracle):
    coh = CohereMelSpectrogram()
    assert same_bits(coh.mel.get_hann_window(), OT.cohere_window(400))
    assert same_bits(coh.mel.get_filterbank(), OT.cohere_filterbank(16000, 512, 128, 0.0, 8000.0))
    one = AudioMelSpectrogram.from_ex_config(ex_config("cohere", win_length=1, n_fft=32, hop_length=1))
    assert one.get_hann_window().tolist() == [0.0]
    sty = StyleTTS2MelExtractor()
    assert same_bits(sty.mel.get_hann_window(), OT.styletts2_window(1200, 2048)[424:424 + 1200])
    assert same_bits(sty.mel.get_filterbank(), OT.styletts2_filterbank(80, 2048, 16000))
    lux = LuxTtsMelExtractor()
    assert same_bits(lux.mel.get_hann_window(), OT.luxtts_window(1024))
    assert same_bits(lux.mel.get_filterbank(), OT.luxtts_filterbank(1024, 100, 24000))


@pytest.mark.parametrize("shape", [dict(), dict(n_fft=1024, win_length=1024, hop_length=256, n_mels=80),
                                   dict(hop_length=161, pad_to=3)])
def test_neutral_ex_handle_equals_fa_mel_create(gpu_lib, shape):
    plain = AudioMelSpectrogram(**shape)
    ex = AudioMelSpectrogram.from_ex_config(ex_config(None, **shape))
    assert same_bits(plain.get_hann_window(), ex.get_hann_window())
    assert same_bits(plain.get_filterbank(), ex.get_filterbank())
    a = synth.tone_noise_audio(16000 * 2 + 37)
    for prec in (Precision.f64, Precision.f32):
        plain.set_precision(prec)
        ex.set_precision(prec)
        for mode in (CENTER, PRE_PADDED, LEGACY):
            for layout in (TIME_MAJOR, MEL_MAJOR):
                g, gm, gn = plain._run(a, 0.25, mode, None, layout)
                h, hm, hn = ex._run(a, 0.25, mode, None, layout)
                assert (gm, gn) == (hm, hn) and same_bits(g, h), (shape, prec, mode, layout)


def test_ex_handles_are_refused_where_they_do_not_apply(gpu_lib):
    L = gpu_lib
    sty = StyleTTS2MelExtractor()
    sid = C.c_int32()
    assert L.fa_mel_stream_open(sty.mel._h, C.byref(sid)) == 1
    out = np.zeros(4096, F32)
    T, v = C.c_int64(), C.c_int32()
    a = np.zeros(1600, F32)
    assert L.fa_mel_unified_features(sty.mel._h, a.ctypes.data, a.size, a.size, out.ctypes.data, out.size,
                                     C.byref(T), C.byref(v)) == 1
    for bad in (dict(filterbank=7), dict(center_edge=2), dict(spectrum_power=0.0), dict(log_std=0.0),
                dict(f_min=10.0), dict(center_edge=1)):   # the last: reflect with the default preemph 0.97
        cfg = ex_config(None, **bad)
        h = C.c_void_p()
        before = _lib.kernel_launch_count()
        assert L.fa_mel_create_ex(C.byref(cfg), C.byref(h)) == 1 and not h.value, bad
        assert L.fa_last_error().decode() and _lib.kernel_launch_count() == before


# ================================================================================================ by composition
def test_reflect_center_equals_prepadded_on_the_padded_clip(gpu_lib, oracle):
    for make, n_fft, hop in ((lambda: StyleTTS2MelExtractor().mel, 2048, 300),
                             (lambda: LuxTtsMelExtractor().mel, 1024, 256)):
        mel = make()
        for n in (1, 2, n_fft // 2 - 1, n_fft // 2, n_fft // 2 + 1, 7 * hop - 1, 7 * hop + 1, 48000):
            a = _signal("noise", n, 24000)
            T = 1 + n // hop
            c = _log_mel(mel, a, T)
            p = _log_mel(mel, OT.reflect_pad(a, n_fft // 2), T, mode=PRE_PADDED)
            assert same_bits(c, p), (n_fft, n)


def test_affine_epilogue_equals_numpy_on_the_same_log_mel(gpu_lib):
    sty = StyleTTS2MelExtractor()
    plain = AudioMelSpectrogram.from_ex_config(ex_config("styletts2", log_mean=0.0, log_std=1.0))
    for n in (0, 1, 300, 24000 * 3 + 11):
        a = _signal("speech", n, 24000)
        got, T = sty.compute(a)
        L = _log_mel(plain, a, T, MEL_MAJOR) if n else None
        if n:
            assert same_bits(got, (L - F32(-4.0)) / F32(4.0)), n
        else:   # an empty clip is nFFT zeros: one frame of (log(1e-5) + 4) / 4
            want = (np.log(1e-5) + 4.0) / 4.0
            assert T == 1 and np.abs(got[:, 0] - want).max() <= _bar(np.log(1e-5)) / 4


@pytest.mark.parametrize("n, fixed", [(0, 3), (1, 3), (160, 5), (320, 5), (160 * 40 + 7, 10), (160 * 40 + 7, 40),
                                      (160 * 40 + 7, 41), (160 * 40 + 7, 100), (160 * 40 + 7, -1), (160 * 40, 0)])
def test_cohere_features_equal_cmvn_of_the_handles_log_mel(gpu_lib, oracle, n, fixed):
    coh = CohereMelSpectrogram()
    for kind in ("speech", "nan", "silence"):
        a = _signal(kind, n, 16000)
        T, valid = 1 + n // 160, n // 160
        got, fl = coh.features(a, fixed)
        if n == 0:   # no valid frame: everything is zero (the plain call has no frame to compare with)
            assert got.shape == (128, fixed) and not got.any() and fl == 0
            continue
        lm = _log_mel(coh.mel, a, T)
        ref = OT.cohere_cmvn(lm, valid, fixed)
        assert same_bits(got, ref), (kind, n, fixed)
        assert fl == (valid if fixed < 0 else min(valid, fixed))


# ================================================================================================ against the oracle
def _cmvn64(mel_tm, valid):
    x = mel_tm[:valid].astype(np.float64)
    with np.errstate(all="ignore"):
        sd = np.sqrt(((x - x.mean(0)) ** 2).sum(0) / (valid - 1)) + 1e-5
        return (x - x.mean(0)) / sd, sd


@pytest.mark.parametrize("kind", ["noise", "speech", "silence", "nan", "overflow"])
def test_against_the_oracle(gpu_lib, oracle, kind):
    sty, lux, coh = StyleTTS2MelExtractor(), LuxTtsMelExtractor(), CohereMelSpectrogram()
    for n in _lengths(2048, 300, 24000) + [60 * 24000]:
        if n == 60 * 24000 and kind != "speech":
            continue
        a = _signal(kind, n, 24000)
        got, T = sty.compute(a)
        ref, rT = OT.styletts2_compute(a)
        assert T == rT
        _check_bar(got, ref, _bar(ref.astype(np.float64) * 4 - 4) / 4 + 2 * np.finfo(F32).eps * np.abs(ref),
                   "styletts2", (kind, n))
    for n in _lengths(1024, 256, 24000) + [60 * 24000]:
        if n == 60 * 24000 and kind != "speech":
            continue
        a = _signal(kind, n, 24000)
        got, ref = lux.extract(a), OT.luxtts_extract(a)
        assert got.shape == ref.shape, n
        _check_bar(got, ref, _bar(ref), "luxtts", (kind, n))
    tiny = 0
    for n in _lengths(512, 160, 16000):
        a = _signal(kind, n, 16000)
        got, valid = coh.features(a, -1)
        ref, rvalid = OT.cohere_compute(a)
        assert valid == rvalid and got.shape == ref.shape
        assert not got[:, valid:].any() and not ref[:, valid:].any()
        lib_fin, ref_fin = np.isfinite(got[:, :valid]).all(1), np.isfinite(ref[:, :valid]).all(1)
        assert not (~lib_fin & ref_fin).any(), (kind, n)   # a non-finite mel poisons its whole CMVN column
        if valid == 1:
            _check_bar(got[:, :1], ref[:, :1], _bar(ref[:, :1].astype(np.float64)), "cohere log-mel", (kind, n))
        elif valid > 1:
            frac, t = cmvn_frac(coh, a, got, ref, valid)
            tiny += t
            if frac is not None:
                _note("cohere cmvn", frac)
                assert frac <= 1.0, (kind, n, float(frac))
    print(f"  Cohere columns left to the bit-exact checks for a tiny spread ({kind}): {tiny}")


def cmvn_frac(coh, a, got, ref, valid, e=None):
    """Worst |d| / bar of two Cohere feature arrays [M x T] over the columns where the first-order CMVN bar applies
    (test_gpu_mel_adapter_sweep.py), with the handle's own log-mel for the bar's magnitudes; and the count of columns
    left out for a tiny spread (E > 0.05 sd).  ``e`` [valid x M]: the log-mel difference budget (default: the
    generic-kernel bar of the handle's log-mel)."""
    lm = _log_mel(coh.mel, a, 1 + a.size // coh.config.hop_length)
    cols = np.isfinite(got[:, :valid]).all(1) & np.isfinite(ref[:, :valid]).all(1)
    e = _bar(lm[:valid].astype(np.float64)) if e is None else np.asarray(e, np.float64)
    E = e.max(0)
    z, sd = _cmvn64(lm, valid)
    use = cols & np.isfinite(sd) & (E <= 0.05 * sd)
    tiny = int((cols & np.isfinite(sd) & ~use).sum())
    if not use.any():
        return None, tiny
    g, r = got[use, :valid].T.astype(np.float64), ref[use, :valid].T.astype(np.float64)
    first = (e[:, use] + E[use]) / sd[use] + np.abs(z[:, use]) * np.sqrt(2.0) * E[use] / sd[use]
    limit = 1.25 * first + 2 * np.abs(g - z[:, use]) + 1e-6
    return float((np.abs(g - r) / limit).max()), tiny


def test_cohere_preemphasis_deviation_is_inside_the_bar(gpu_lib):
    """The library pre-emphasises with one fused multiply-add, the reference with x[i] - (a * x[i-1]) in two roundings.
    Feeding the handle without pre-emphasis the two-rounded signal isolates the fusion's whole effect.  In the log-mel it
    exceeds the generic mel bar in weak bands (pre-emphasis is a high-pass filter, so the low bands are small and the
    half-ulp perturbation is white); it is reported, not bounded.  In Cohere's features, the output of the class, it
    must be inside the first-order CMVN bar."""
    coh = CohereMelSpectrogram()
    nopre = CohereMelSpectrogram(CohereMelSpectrogram.Config(preemph=0.0))
    worst_mel, worst_feat = 0.0, 0.0
    for kind in ("noise", "speech"):
        a = _signal(kind, 16000 * 10, 16000)
        two = a.copy()
        two[1:] = a[1:] - F32(0.97) * a[:-1]
        T = 1 + a.size // 160
        fused, ref = _log_mel(coh.mel, a, T), _log_mel(nopre.mel, two, T)
        worst_mel = max(worst_mel, float((np.abs(fused.astype(np.float64) - ref) / _bar(ref.astype(np.float64))).max()))
        g, valid = coh.features(a, -1)
        r, _ = nopre.features(two, -1)
        frac, _ = cmvn_frac(coh, a, g, r, valid)
        worst_feat = max(worst_feat, frac)
    print(f"\nCohere pre-emphasis, fused vs two roundings: log-mel worst |d| / mel bar {worst_mel:.3g}, "
          f"features worst |d| / CMVN bar {worst_feat:.3g}")
    assert worst_feat <= 1.0


def test_nan_poisons_exactly_the_frames_that_read_it(gpu_lib):
    """A NaN at sample k makes exactly the frames whose window reads k, directly or through a reflection, NaN (in every
    mel with a non-empty band: all of them here)."""
    for ext, n_fft, win, hop, ks in ((LuxTtsMelExtractor(), 1024, 1024, 256, (0, 1, 5, 700, 3000, 4999)),
                                     (StyleTTS2MelExtractor(), 2048, 1200, 300, (0, 3, 100, 2500, 4999))):
        for k in ks:
            n = 5000
            a = _signal("noise", n, 24000)
            a[k] = np.nan
            T = 1 + n // hop
            mel = _log_mel(ext.mel, a, T)
            lo = (n_fft - win) // 2
            hit = np.zeros(T, bool)
            for f in range(T):
                for j in range(lo, lo + win):
                    i = f * hop - n_fft // 2 + j
                    r = min(-i, n - 1) if i < 0 else (max(2 * n - 2 - i, 0) if i >= n else i)
                    if r == k:
                        hit[f] = True
                        break
            assert np.array_equal(np.isnan(mel).any(1), hit) and np.isnan(mel[hit]).all(), (n_fft, k)


# ================================================================================================ batches, device buffers
def test_batches_and_device_buffers_equal_single_host_calls(gpu_lib):
    rng = np.random.default_rng(4)
    for ext in (StyleTTS2MelExtractor(), LuxTtsMelExtractor(), CohereMelSpectrogram()):
        mel = ext.mel
        clips = [_signal("speech", int(m), mel.sample_rate, seed=i)
                 for i, m in enumerate([1, 2, 511, 1025, 24000, 2 * mel.sample_rate + 17, 300, 4096])]
        clips += [rng.standard_normal(int(rng.integers(3, 30000))).astype(F32) for _ in range(20)]
        for layout_tm in (True, False):
            out, oo, ml, nf = mel.compute_batch(clips, time_major=layout_tm)
            for i, c in enumerate(clips):
                single, sml, snf = mel._run(c, 0.0, CENTER, None, TIME_MAJOR if layout_tm else MEL_MAJOR)
                assert (ml[i], nf[i]) == (sml, snf) and same_bits(out[oo[i]:oo[i + 1]], single[:snf * mel.n_mels])
        # device buffers: fa_mel_compute_device equals fa_mel_compute
        a = clips[5]
        d_in, d_out = _lib.DeviceBuffer(4 * a.size), _lib.DeviceBuffer(4 * mel.n_mels * (a.size // mel.hop_length + 16))
        d_in.upload(a)
        ml, nf = mel.compute_device(d_in, a.size, d_out)
        host, hml, hnf = mel._run(a, 0.0, CENTER, None, TIME_MAJOR)
        assert (ml, nf) == (hml, hnf) and same_bits(d_out.download(nf * mel.n_mels, F32), host[:nf * mel.n_mels])
        # chunked host pipeline (24 units) against one unit: reflected frames cross unit boundaries
        long = _signal("noise", 12500 * mel.hop_length + 7, mel.sample_rate)   # >= 3 units of >= 4096 frames
        T = 1 + long.size // mel.hop_length
        mel._L.fa_mel_set_pipeline_chunks(mel._h, 24)
        chunked = _log_mel(mel, long, T)
        mel._L.fa_mel_set_pipeline_chunks(mel._h, 1)
        assert same_bits(chunked, _log_mel(mel, long, T))


# ================================================================================================ launches, arguments
def test_launch_counts_and_argument_checks(gpu_lib):
    L = gpu_lib
    sty, lux, coh = StyleTTS2MelExtractor(), LuxTtsMelExtractor(), CohereMelSpectrogram()
    a = _signal("noise", 24000, 24000)
    assert _launches(lambda: sty.compute(a))[1] == 1
    assert _launches(lambda: sty.compute(a[:0]))[1] == 1
    assert _launches(lambda: lux.extract(a))[1] == 1
    assert _launches(lambda: lux.extract(a[:100]))[1] == 0      # (100 + 128) / 256 = 0 frames: nothing to run
    assert _launches(lambda: coh.features(a[:16000]))[1] == 2
    assert _launches(lambda: coh.features(a[:0]))[1] == 2
    # a handle of another class, or a short buffer: no launch, no write
    out = np.full(80 * 100 * 200, 7.0, F32)
    fr, va = C.c_int64(-5), C.c_int64(-5)
    calls = [lambda o, n: L.fa_mel_styletts2_features(lux.mel._h, a.ctypes.data, a.size, o.ctypes.data, n, C.byref(fr)),
             lambda o, n: L.fa_mel_luxtts_features(sty.mel._h, a.ctypes.data, a.size, o.ctypes.data, n, C.byref(fr)),
             lambda o, n: L.fa_mel_cohere_features(sty.mel._h, a.ctypes.data, a.size, 50, o.ctypes.data, n,
                                                   C.byref(fr), C.byref(va))]
    for call in calls:
        st, k = _launches(lambda: call(out, out.size))
        assert st == 1 and k == 0 and (out == 7.0).all()
    for call, need in ((lambda o, n: L.fa_mel_styletts2_features(sty.mel._h, a.ctypes.data, a.size, o.ctypes.data, n,
                                                                 C.byref(fr)), 80 * 81),
                       (lambda o, n: L.fa_mel_luxtts_features(lux.mel._h, a.ctypes.data, a.size, o.ctypes.data, n,
                                                              C.byref(fr)), 100 * 94),
                       (lambda o, n: L.fa_mel_cohere_features(coh.mel._h, a.ctypes.data, a.size, 50, o.ctypes.data, n,
                                                              C.byref(fr), C.byref(va)), 128 * 50)):
        st, k = _launches(lambda: call(out, need - 1))
        assert st == 3 and k == 0 and (out == 7.0).all()
        st, k = _launches(lambda: call(out, need))
        assert st == 0 and k >= 1
        out[:] = 7.0
