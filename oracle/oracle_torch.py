"""ORACLE — TEST INFRASTRUCTURE ONLY.  Not part of the shipped product path.

ctypes front-end to ``liboracle_torch.so``, the CPU restatement of the reference's torch-style log-mel frontends
(``oracle_mel_torch.cpp``: CohereMelSpectrogram, StyleTTS2MelExtractor, LuxTtsMelExtractor).  It has its own library so
that the main oracle (``oracle.py``, ``liboracle.so``) is untouched; it is compiled with the main oracle's pinned flags
(``-O2 -ffp-contract=off`` on baseline x86-64: every float32 operation rounded as the C++ states it).
Importers allowed: ``tests/``, ``__graft_entry__.build()`` and ``scripts/gpu_mel_torch_timing.py``.  The product package
``fluidaudio_b200`` never imports it.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, "oracle_mel_torch.cpp")
_LIB = os.path.join(_HERE, "liboracle_torch.so")
_FLAGS = ["-std=c++17", "-O2", "-ffp-contract=off", "-fPIC", "-Wall", "-Wextra", "-shared"]

_f32p = np.ctypeslib.ndpointer(np.float32, flags="C_CONTIGUOUS")
_lib = None


def build(force: bool = False) -> None:
    """Compile liboracle_torch.so when it is missing or older than its source."""
    if force or not os.path.exists(_LIB) or os.path.getmtime(_SRC) > os.path.getmtime(_LIB):
        cxx = os.environ.get("CXX", "g++")
        subprocess.check_call([cxx, *_FLAGS, "-o", _LIB, _SRC])


def lib():
    global _lib
    if _lib is None:
        build()
        L = C.CDLL(_LIB)
        i32, i64, f32 = C.c_int32, C.c_int64, C.c_float
        L.oracle_cohere_window.argtypes = [i32, _f32p]
        L.oracle_cohere_filterbank.argtypes = [i32, i32, i32, f32, f32, _f32p]
        L.oracle_cohere_compute.argtypes = [i32, i32, i32, i32, f32, f32, f32, f32, f32, f32, _f32p, i64, _f32p,
                                            C.POINTER(i64)]
        L.oracle_cohere_compute.restype = i64
        L.oracle_cohere_cmvn.argtypes = [_f32p, i64, i32, i64, i64, f32, _f32p]
        L.oracle_cohere_cmvn.restype = i64
        L.oracle_reflect_pad.argtypes = [_f32p, i64, i32, _f32p]
        L.oracle_styletts2_window.argtypes = [i32, i32, _f32p]
        L.oracle_styletts2_filterbank.argtypes = [i32, i32, i32, _f32p]
        L.oracle_styletts2_compute.argtypes = [i32, i32, i32, i32, i32, f32, f32, f32, i32, _f32p, i64, _f32p]
        L.oracle_styletts2_compute.restype = i64
        L.oracle_luxtts_window.argtypes = [i32, _f32p]
        L.oracle_luxtts_filterbank.argtypes = [i32, i32, i32, _f32p]
        L.oracle_luxtts_extract.argtypes = [i32, i32, i32, i32, f32, _f32p, i64, _f32p]
        L.oracle_luxtts_extract.restype = i64
        _lib = L
    return _lib


# CohereMelSpectrogram (CoherePipeline.swift:41-324), StyleTTS2MelExtractor, LuxTtsMelExtractor.
COHERE_DEFAULTS = dict(sample_rate=16000, win_length=400, hop_length=160, n_mels=128, f_min=0.0, f_max=8000.0,
                       preemph=0.97, mag_power=2.0, log_zero_guard=2.0 ** -24, cmvn_epsilon=1e-5)
STYLETTS2_DEFAULTS = dict(n_fft=2048, win_length=1200, hop_length=300, n_mels=80, filter_sample_rate=16000, mean=-4.0,
                          std=4.0, log_epsilon=1e-5)
LUXTTS_DEFAULTS = dict(n_fft=1024, hop_length=256, n_mels=100, sample_rate=24000, log_floor=1e-7)


def _f32(a):
    return np.ascontiguousarray(a, np.float32).reshape(-1)


def cohere_window(win_length=400) -> np.ndarray:
    out = np.zeros(max(win_length, 1), np.float32)
    lib().oracle_cohere_window(win_length, out)
    return out[:win_length]


def cohere_filterbank(sample_rate=16000, n_fft=512, n_mels=128, f_min=0.0, f_max=8000.0) -> np.ndarray:
    out = np.zeros(n_mels * (n_fft // 2 + 1), np.float32)
    lib().oracle_cohere_filterbank(sample_rate, n_fft, n_mels, f_min, f_max, out)
    return out.reshape(n_mels, n_fft // 2 + 1)


def cohere_compute(audio, **cfg):
    """CohereMelSpectrogram.compute: ([nMels x T] float32, validFrames)."""
    c = {**COHERE_DEFAULTS, **cfg}
    a = _f32(audio)
    T = 1 + a.size // c["hop_length"]
    out = np.zeros(c["n_mels"] * T, np.float32)
    valid = C.c_int64()
    got = lib().oracle_cohere_compute(c["sample_rate"], c["win_length"], c["hop_length"], c["n_mels"], c["f_min"],
                                      c["f_max"], c["preemph"], c["mag_power"], c["log_zero_guard"], c["cmvn_epsilon"],
                                      a if a.size else np.zeros(1, np.float32), a.size, out, C.byref(valid))
    assert got == T
    return out.reshape(c["n_mels"], T), int(valid.value)


def cohere_cmvn(mel_tm, valid, fixed_frames=-1, cmvn_epsilon=1e-5) -> np.ndarray:
    """Cohere's CMVN, invalid-frame zeroing and padOrTruncate on a given time-major log-mel [T x nMels] -> [nMels x W]."""
    x = np.ascontiguousarray(mel_tm, np.float32)
    T, M = x.shape
    W = T if fixed_frames < 0 else fixed_frames
    out = np.zeros(max(M * W, 1), np.float32)
    lib().oracle_cohere_cmvn(x.reshape(-1) if x.size else np.zeros(1, np.float32), T, M, valid, fixed_frames,
                             cmvn_epsilon, out)
    return out[:M * W].reshape(M, W)


def cohere_pad_or_truncate(mel, valid_frames, fixed_frames=3500):
    """CohereMelSpectrogram.padOrTruncate (:250-263)."""
    mel = np.asarray(mel, np.float32)
    if mel.shape[0] == 0:
        return mel, 0
    cur = mel.shape[1]
    if cur >= fixed_frames:
        return mel[:, :fixed_frames].copy(), min(valid_frames, fixed_frames)
    return np.concatenate([mel, np.zeros((mel.shape[0], fixed_frames - cur), np.float32)], 1), min(valid_frames,
                                                                                                    fixed_frames)


def reflect_pad(x, pad) -> np.ndarray:
    """StyleTTS2MelExtractor.reflectPad (:226-250)."""
    a = _f32(x)
    out = np.zeros(a.size + 2 * pad, np.float32)
    lib().oracle_reflect_pad(a if a.size else np.zeros(1, np.float32), a.size, pad, out)
    return out


def styletts2_window(win_length=1200, n_fft=2048) -> np.ndarray:
    out = np.zeros(n_fft, np.float32)
    lib().oracle_styletts2_window(win_length, n_fft, out)
    return out


def styletts2_filterbank(n_mels=80, n_fft=2048, sample_rate=16000) -> np.ndarray:
    out = np.zeros(n_mels * (n_fft // 2 + 1), np.float32)
    lib().oracle_styletts2_filterbank(n_mels, n_fft, sample_rate, out)
    return out.reshape(n_mels, n_fft // 2 + 1)


def styletts2_compute(audio, affine=True, **cfg):
    """StyleTTS2MelExtractor.compute: ([nMels x frames], frames); affine=False stops at log(mel + eps)."""
    c = {**STYLETTS2_DEFAULTS, **cfg}
    a = _f32(audio)
    T = 1 + a.size // c["hop_length"]
    out = np.zeros(c["n_mels"] * T, np.float32)
    got = lib().oracle_styletts2_compute(c["n_fft"], c["win_length"], c["hop_length"], c["n_mels"],
                                         c["filter_sample_rate"], c["mean"], c["std"], c["log_epsilon"], int(affine),
                                         a if a.size else np.zeros(1, np.float32), a.size, out)
    assert got == T
    return out.reshape(c["n_mels"], T), T


def luxtts_window(n_fft=1024) -> np.ndarray:
    out = np.zeros(n_fft, np.float32)
    lib().oracle_luxtts_window(n_fft, out)
    return out


def luxtts_filterbank(n_fft=1024, n_mels=100, sample_rate=24000) -> np.ndarray:
    out = np.zeros(n_mels * (n_fft // 2 + 1), np.float32)
    lib().oracle_luxtts_filterbank(n_fft, n_mels, sample_rate, out)
    return out.reshape(n_mels, n_fft // 2 + 1)


def luxtts_extract(audio, **cfg) -> np.ndarray:
    """LuxTtsMelExtractor.extract: [T x nMels]."""
    c = {**LUXTTS_DEFAULTS, **cfg}
    a = _f32(audio)
    T = (a.size + c["hop_length"] // 2) // c["hop_length"] if a.size else 0
    out = np.zeros(max(T * c["n_mels"], 1), np.float32)
    got = lib().oracle_luxtts_extract(c["n_fft"], c["hop_length"], c["n_mels"], c["sample_rate"], c["log_floor"],
                                      a if a.size else np.zeros(1, np.float32), a.size, out)
    assert got == T
    return out[:T * c["n_mels"]].reshape(T, c["n_mels"])
