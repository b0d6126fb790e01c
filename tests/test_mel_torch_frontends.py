"""The torch-style log-mel frontends on the CPU: the oracle, the reflect map and the frame-count rules.

``oracle_mel_torch.cpp`` (through ``oracle/oracle_torch.py``) restates CohereMelSpectrogram (ASR/Cohere/CoherePipeline.swift:41-324), StyleTTS2MelExtractor
and LuxTtsMelExtractor line by line in float32.  Here it is held to an independent numpy float64 restatement of each
class, its reflect padding to the reference's doc example and to the kernel's own ``reflect_index`` (compiled for the host
from ``mel_core.cuh``), and the frame counts the library's entry points use to the reference's rules.  The GPU side is
tests/test_gpu_mel_torch_sweep.py.
"""
import ctypes as C
import os
import subprocess

import numpy as np

from fluidaudio_b200 import synth
from oracle import oracle_torch as OT

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F32 = np.float32


# ================================================================================================ float64 restatements
def _hann(win, periodic):
    if win == 1 and not periodic:
        return np.zeros(1)
    d = win if periodic else win - 1
    return 0.5 * (1.0 - np.cos(2.0 * np.pi * np.arange(win) / d))


def _slaney_mel(hz):
    hz = np.asarray(hz, np.float64)
    return np.where(hz >= 1000.0, 15.0 + np.log(np.maximum(hz, 1e-30) / 1000.0) / (np.log(6.4) / 27.0), hz * 3.0 / 200.0)


def _slaney_hz(mel):
    mel = np.asarray(mel, np.float64)
    return np.where(mel >= 15.0, 1000.0 * np.exp(np.log(6.4) / 27.0 * (mel - 15.0)), 200.0 / 3.0 * mel)


def np_cohere_filterbank(sr, n_fft, n_mels, f_min, f_max):
    freqs = np.arange(n_fft // 2 + 1) * sr / n_fft
    hz = _slaney_hz(np.linspace(_slaney_mel(f_min), _slaney_mel(f_max), n_mels + 2))
    lo, c, hi = hz[:-2, None], hz[1:-1, None], hz[2:, None]
    up = (freqs - lo) / np.maximum(c - lo, 1e-10)
    down = (hi - freqs) / np.maximum(hi - c, 1e-10)
    fb = np.where((freqs < lo) | (freqs > hi), 0.0, np.where(freqs <= c, up, down))
    return fb * (2.0 / np.maximum(hi - lo, 1e-10))


def np_htk_filterbank(n_fft, n_mels, sr):
    to_mel = lambda f: 2595.0 * np.log10(1.0 + f / 700.0)
    hz = 700.0 * (10.0 ** (np.linspace(to_mel(0.0), to_mel(sr / 2.0), n_mels + 2) / 2595.0) - 1.0)
    freqs = np.linspace(0.0, sr / 2.0, n_fft // 2 + 1)
    up = (freqs - hz[:-2, None]) / (hz[1:-1, None] - hz[:-2, None])
    down = (hz[2:, None] - freqs) / (hz[2:, None] - hz[1:-1, None])
    return np.maximum(0.0, np.minimum(up, down))


def np_reflect(x, pad):
    """The Swift's reflectPad clamps in float64 (not numpy's np.pad, which fails for short clips)."""
    n = len(x)
    if n == 0:
        return np.zeros(2 * pad)
    idx = np.arange(-pad, n + pad)
    idx = np.where(idx < 0, np.minimum(-idx, n - 1), np.where(idx >= n, np.maximum(2 * n - 2 - idx, 0), idx))
    return np.asarray(x, np.float64)[idx]


def _stft(padded, n_fft, hop, window, frames):
    idx = np.arange(frames)[:, None] * hop + np.arange(n_fft)
    return np.abs(np.fft.rfft(padded[idx] * window, axis=1))   # [frames x bins]


def np_cohere(audio, sr=16000, win=400, hop=160, n_mels=128, f_min=0.0, f_max=8000.0, preemph=0.97, power=2.0,
              guard=2.0 ** -24, eps=1e-5):
    x = np.asarray(audio, np.float64)
    n = x.size
    n_fft = 1 << max(0, (win - 1).bit_length())
    if preemph and n > 1:
        x = np.concatenate([x[:1], x[1:] - preemph * x[:-1]])
    padded = np.concatenate([np.zeros(n_fft // 2), x, np.zeros(n_fft // 2)])
    T, valid = 1 + n // hop, n // hop
    w = np.zeros(n_fft)
    w[(n_fft - win) // 2:(n_fft - win) // 2 + win] = _hann(win, False)
    mag = _stft(padded, n_fft, hop, w, T)
    mel = np.log(np_cohere_filterbank(sr, n_fft, n_mels, f_min, f_max) @ (mag ** power).T + guard)   # [M x T]
    if valid > 1:
        v = mel[:, :valid]
        sd = np.sqrt(((v - v.mean(1, keepdims=True)) ** 2).sum(1, keepdims=True) / (valid - 1))
        mel[:, :valid] = (v - v.mean(1, keepdims=True)) / (sd + eps)
    mel[:, valid:] = 0.0
    return mel, valid


def np_styletts2(audio, n_fft=2048, win=1200, hop=300, n_mels=80, filter_sr=16000, mean=-4.0, std=4.0, eps=1e-5):
    padded = np_reflect(audio, n_fft // 2)
    T = 1 + len(audio) // hop
    w = np.zeros(n_fft)
    w[(n_fft - win) // 2:(n_fft - win) // 2 + win] = _hann(win, True)
    mag = _stft(padded, n_fft, hop, w, T)
    fb = np_htk_filterbank(n_fft, n_mels, filter_sr)
    return (np.log(fb @ (mag ** 2).T + eps) - mean) / std


def np_luxtts(audio, n_fft=1024, hop=256, n_mels=100, sr=24000, floor=1e-7):
    n = len(audio)
    T = (n + hop // 2) // hop if n else 0
    if T == 0:
        return np.zeros((0, n_mels))
    mag = _stft(np_reflect(audio, n_fft // 2), n_fft, hop, _hann(n_fft, True), T)
    return np.log(np.maximum(mag @ np_htk_filterbank(n_fft, n_mels, sr).T, floor))


# ================================================================================================ the oracle vs float64
def _close_in_mel_domain(got_log, ref_log, frame_axis):
    """float32 against float64: the window and table roundings move a mel value by ~1e-7 of the frame's strongest
    spectral line, which is large in the log of a weak band.  So compare mel values: within 1e-4 of the value plus 1e-6
    of the frame's largest mel value."""
    g, r = np.exp(np.asarray(got_log, np.float64)), np.exp(np.asarray(ref_log, np.float64))
    top = r.max(axis=1 - frame_axis, keepdims=True) if r.size else r
    return bool((np.abs(g - r) <= 1e-4 * r + 1e-6 * top + 1e-30).all())


def _fixtures():
    rng = np.random.default_rng(5)
    return {"noise": (rng.standard_normal(24000) * 0.3).astype(F32),
            "speech": synth.speech_like_audio(24000),
            "tone": synth.tone_noise_audio(17000)}


def test_oracle_cohere_matches_float64(oracle):
    """Log-mel before CMVN agrees to ~1e-5; the CMVN output inherits it, amplified by 1/sd (bar 1e-3)."""
    for name, a in _fixtures().items():
        for n in (a.size, 1, 2, 159, 161, 320):
            x = a[:n]
            got, valid = OT.cohere_compute(x)
            ref, rvalid = np_cohere(x)
            assert valid == rvalid == n // 160 and got.shape == ref.shape == (128, 1 + n // 160)
            assert np.abs(got - ref).max() <= 1e-3, (name, n, float(np.abs(got - ref).max()))
    # un-normalised log-mel (valid <= 1 leaves frame 0 as it is)
    x = _fixtures()["speech"][:300]
    got, _ = OT.cohere_compute(x)
    ref, _ = np_cohere(x)
    assert np.abs(got[:, 0] - ref[:, 0]).max() <= 1e-4


def test_oracle_styletts2_matches_float64(oracle):
    for name, a in _fixtures().items():
        for n in (a.size, 0, 1, 2, 1023, 1024, 1025, 299, 301):
            x = a[:n]
            got, T = OT.styletts2_compute(x)
            ref = np_styletts2(x)
            assert T == 1 + n // 300 and got.shape == ref.shape
            assert _close_in_mel_domain(got.astype(np.float64) * 4 - 4, ref * 4 - 4, 1), (name, n)


def test_oracle_luxtts_matches_float64(oracle):
    for name, a in _fixtures().items():
        for n in (a.size, 0, 1, 127, 128, 129, 511, 512, 513, 255, 257):
            x = a[:n]
            got = OT.luxtts_extract(x)
            ref = np_luxtts(x)
            assert got.shape == ref.shape == ((n + 128) // 256, 100)
            assert _close_in_mel_domain(got, ref, 0), (name, n)


# ================================================================================================ reflect padding
def _emul(tmp_path):
    out = str(tmp_path / "libmel_reflect_emul.so")
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-fPIC", "-shared", "-o", out,
                           os.path.join(ROOT, "tests", "emul", "mel_reflect_emul.cpp")])
    L = C.CDLL(out)
    L.reflect_map.argtypes = [C.c_longlong, C.c_int, np.ctypeslib.ndpointer(np.int64, flags="C_CONTIGUOUS")]
    f32p = np.ctypeslib.ndpointer(F32, flags="C_CONTIGUOUS")
    L.reflect_frames.argtypes = [f32p, C.c_longlong, C.c_int, C.c_int, f32p,
                                 np.ctypeslib.ndpointer(np.uint8, flags="C_CONTIGUOUS"), C.c_longlong, f32p]
    return L


def test_reflect_pad_doc_example_and_short_clips(oracle, tmp_path):
    """The reference's doc example, and n in {0, 1, 2, pad-1, pad, pad+1} for the two presets' pads: the oracle, the
    kernel's reflect_index and a float64 restatement agree; past n > pad + 1 it is numpy's 'reflect'."""
    L = _emul(tmp_path)
    a, b, c, d = 1.0, 2.0, 3.0, 4.0
    x = np.array([a, b, c, d], F32)
    assert OT.reflect_pad(x, 2).tolist() == [c, b, a, b, c, d, c, b]
    idx = np.zeros(8, np.int64)
    L.reflect_map(4, 2, idx)
    assert x[idx].tolist() == [c, b, a, b, c, d, c, b]
    rng = np.random.default_rng(3)
    for pad in (2, 512, 1024):
        for n in (0, 1, 2, pad - 1, pad, pad + 1, 3 * pad + 5):
            x = rng.standard_normal(n).astype(F32)
            ref = OT.reflect_pad(x, pad)
            assert np.array_equal(ref, np_reflect(x, pad).astype(F32)), (pad, n)
            if n:
                idx = np.zeros(n + 2 * pad, np.int64)
                L.reflect_map(n, pad, idx)
                assert np.array_equal(x[idx], ref), (pad, n)
            if n > pad:
                assert np.array_equal(ref, np.pad(x, pad, mode="reflect")), (pad, n)


def test_kernel_reflect_loader_matches_padded_frames(oracle, tmp_path):
    """The kernel's reflected .center frames (emulated from the shared header) equal the reference's frames of the
    host-padded signal times the window, for short clips, hop multiples and chunk-sized clips."""
    L = _emul(tmp_path)
    rng = np.random.default_rng(9)
    for n_fft, win, hop in ((2048, 1200, 300), (1024, 1024, 256)):
        w = OT.styletts2_window(win, n_fft)
        in_tab = np.zeros(n_fft, np.uint8)
        in_tab[(n_fft - win) // 2:(n_fft - win) // 2 + win] = 1
        for n in (0, 1, 2, n_fft // 2 - 1, n_fft // 2, n_fft // 2 + 1, hop * 7 - 1, hop * 7 + 1, 24000):
            x = rng.standard_normal(n).astype(F32)
            T = 1 + n // hop
            got = np.zeros((T, n_fft), F32)
            L.reflect_frames(x if n else np.zeros(1, F32), n, n_fft, hop, w, in_tab, T, got)
            padded = OT.reflect_pad(x, n_fft // 2)
            ref = np.stack([padded[f * hop:f * hop + n_fft] * w for f in range(T)]).astype(F32)
            assert np.array_equal(got, ref), (n_fft, n)


# ================================================================================================ frame counts
def test_frame_count_rules(oracle):
    """Cohere: T = 1 + n / hop, valid = n / hop; StyleTTS2: 1 + n / hop (1 for an empty clip); LuxTTS: (n + hop/2) / hop,
    0 for n == 0.  Short clips across 0 .. 3 hop and long clips, from the oracle's own output shapes."""
    x = synth.tone_noise_audio(3 * 300 + 1)
    for n in range(0, 3 * 160 + 2, 7):
        mel, valid = OT.cohere_compute(x[:n])
        assert mel.shape == (128, 1 + n // 160) and valid == n // 160
    for n in range(0, 3 * 300 + 2, 11):
        assert OT.styletts2_compute(x[:n])[1] == 1 + n // 300
    for n in range(0, 3 * 256 + 2, 5):
        assert OT.luxtts_extract(x[:n]).shape[0] == ((n + 128) // 256 if n else 0)
    long = synth.tone_noise_audio(24000 * 11 + 77)
    assert OT.styletts2_compute(long)[1] == 1 + long.size // 300
    assert OT.luxtts_extract(long).shape[0] == (long.size + 128) // 256


def test_luxtts_never_replicates_the_last_frame():
    """lhotse's count never exceeds the STFT's: (n + hop/2) / hop <= 1 + n / hop for every n >= 0, so
    LuxTtsMelExtractor.extract's replicate-last-frame loop (:126-130) is never entered and the library has no kernel for it.
    Exhaustive up to 10^6 samples, and in general: (n + h/2) / h <= (n + h) / h = 1 + n / h."""
    n = np.arange(0, 10 ** 6 + 1, dtype=np.int64)
    hop = 256
    assert ((n + hop // 2) // hop <= 1 + n // hop).all()
    for h in (1, 2, 3, 160, 255, 300, 1024):
        m = np.arange(0, 20 * h + 1, dtype=np.int64)
        assert ((m + h // 2) // h <= 1 + m // h).all()


# ================================================================================================ tables
def test_cohere_table_is_close_to_audio_mel_spectrograms(oracle):
    """At default settings (16 kHz, nFFT 512, 128 mels, 0 .. 8 kHz) CohereMelSpectrogram's Slaney table and
    AudioMelSpectrogram's describe the same filters but are not the same floats: a different mel step, different edge
    rules and its own constants.  They must stay close; the largest difference is reported."""
    coh = OT.cohere_filterbank(16000, 512, 128, 0.0, 8000.0)
    aud = oracle.mel_filterbank(512, 128)
    d = np.abs(coh.astype(np.float64) - aud)
    print(f"\nCohere vs AudioMelSpectrogram table: max |d| {d.max():.3g} (max weight {aud.max():.3g}), "
          f"{int((coh != aud).sum())} of {coh.size} entries differ")
    assert d.max() <= 1e-3 * aud.max()
    assert np.abs(coh - np_cohere_filterbank(16000, 512, 128, 0.0, 8000.0)).max() <= 1e-6 * aud.max() * 1e3
    # the window: symmetric Hann, and a length-1 window is [0] (AudioMelSpectrogram's formula would divide by zero)
    assert np.array_equal(OT.cohere_window(400), oracle.hann_window(400, False))
    assert OT.cohere_window(1).tolist() == [0.0]


def test_styletts2_table_uses_16khz_bins(oracle):
    """StyleTTS2's table is built for 16 kHz (StyleTTS2Constants.melFilterSampleRate) although the audio is 24 kHz: its
    filters span bins up to 8 kHz = bin 1024 of 2048, each filter peaks at its HTK centre on a 16000 / 2048 Hz grid,
    and it is not the table a 24 kHz build would give."""
    fb = OT.styletts2_filterbank(80, 2048, 16000)
    assert fb.shape == (80, 1025)
    ref = np_htk_filterbank(2048, 80, 16000)
    assert np.abs(fb - ref).max() <= 1e-5
    to_mel = lambda f: 2595.0 * np.log10(1.0 + f / 700.0)
    centres = 700.0 * (10.0 ** (np.linspace(0.0, to_mel(8000.0), 82)[1:-1] / 2595.0) - 1.0)
    assert (np.abs(fb.argmax(axis=1) * 16000.0 / 2048 - centres) <= 16000.0 / 2048).all()
    assert not np.array_equal(fb, OT.styletts2_filterbank(80, 2048, 24000))
    # LuxTTS's float64 table against the float64 restatement: bit for bit after the one rounding
    assert np.array_equal(OT.luxtts_filterbank(1024, 100, 24000), np_htk_filterbank(1024, 100, 24000).astype(F32))
