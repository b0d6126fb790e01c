"""ORACLE — TEST INFRASTRUCTURE ONLY.  Not part of the shipped product path.

ctypes front-end to ``liboracle_lseend.so``, the sequential CPU restatement of LSEENDFeatureProvider and
StreamingChunkQueue (``oracle_lseend.cpp``: LSEENDPreprocessor.swift, one provider per object) on top of the main
oracle's log-mel and LS-EEND scaling restatements (``oracle_mel.cpp``, ``oracle_adapters.cpp``), compiled into its own
library with the main oracle's pinned flags (``-O2 -ffp-contract=off`` on baseline x86-64).
Importers allowed: ``tests/``, ``__graft_entry__`` and ``scripts/``.  The product package never imports it.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess
from types import SimpleNamespace

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRCS = [os.path.join(_HERE, f) for f in ("oracle_lseend.cpp", "oracle_mel.cpp", "oracle_adapters.cpp")]
_LIB = os.path.join(_HERE, "liboracle_lseend.so")
_FLAGS = ["-std=c++17", "-O2", "-ffp-contract=off", "-fPIC", "-Wall", "-Wextra", "-shared"]
_INTS = ("sample_rate", "n_mels", "hop_length", "win_length", "context_size", "subsampling", "chunk_size", "conv_delay")

_lib = None


def build(force: bool = False) -> None:
    """Compile liboracle_lseend.so when it is missing or older than a source."""
    if force or not os.path.exists(_LIB) or any(os.path.getmtime(s) > os.path.getmtime(_LIB) for s in _SRCS):
        cxx = os.environ.get("CXX", "g++")
        subprocess.check_call([cxx, *_FLAGS, "-o", _LIB, *_SRCS])


def lib():
    global _lib
    if _lib is None:
        build()
        L = C.CDLL(_LIB)
        vp, i64 = C.c_void_p, C.c_int64
        L.oracle_lseend_create.argtypes = [vp]
        L.oracle_lseend_create.restype = vp
        for name in ("oracle_lseend_destroy", "oracle_lseend_drain", "oracle_lseend_snapshot", "oracle_lseend_rollback",
                     "oracle_lseend_reset"):
            getattr(L, name).argtypes = [vp]
            getattr(L, name).restype = None
        L.oracle_lseend_enqueue.argtypes = [vp, vp, i64]
        L.oracle_lseend_enqueue.restype = None
        L.oracle_lseend_ready.argtypes = [vp]
        L.oracle_lseend_ready.restype = i64
        L.oracle_lseend_emit.argtypes = [vp, vp, vp, vp]
        L.oracle_lseend_emit.restype = C.c_int32
        L.oracle_lseend_lengths.argtypes = [vp, vp]
        L.oracle_lseend_lengths.restype = None
        L.oracle_lseend_state.argtypes = [vp, vp, vp, vp]
        L.oracle_lseend_state.restype = None
        _lib = L
    return _lib


def _get(cfg, k):
    return cfg[k] if isinstance(cfg, dict) else getattr(cfg, k)


def sizes(cfg) -> SimpleNamespace:
    """The provider's derived sizes (LSEENDPreprocessor.swift:52-67, LSEENDTypes.swift:53-57)."""
    hop, win, ctx, sub, chunk, delay = (int(_get(cfg, k)) for k in ("hop_length", "win_length", "context_size",
                                                                     "subsampling", "chunk_size", "conv_delay"))
    n_fft = 1 << (win - 1).bit_length()
    mel_frames = (chunk - 1) * sub + 2 * ctx + 1
    return SimpleNamespace(n_fft=n_fft, mel_frames=mel_frames, chunk_mels=sub * chunk, mel_context=mel_frames - sub * chunk,
                           chunk_samples=hop * sub * chunk, audio_left_context=n_fft // 2, audio_context=n_fft - hop,
                           flush_samples=(ctx + delay * sub) * hop + n_fft // 2, mask_length=delay + chunk,
                           audio_capacity=hop * sub * chunk + n_fft - hop)


class Provider:
    """One LSEENDFeatureProvider.  ``cfg`` has the fa_lseend_stream_config field names (a dict or attributes)."""

    def __init__(self, cfg):
        self.n_mels = int(_get(cfg, "n_mels"))
        self.chunk_size = int(_get(cfg, "chunk_size"))
        self.mel_frames = sizes(cfg).mel_frames
        ints = np.array([int(_get(cfg, k)) for k in _INTS], np.int32)
        self._h = lib().oracle_lseend_create(ints.ctypes.data)

    def __del__(self):
        try:
            lib().oracle_lseend_destroy(self._h)
        except Exception:
            pass

    def enqueue_audio(self, x):
        x = np.ascontiguousarray(x, np.float32).reshape(-1)
        lib().oracle_lseend_enqueue(self._h, x.ctypes.data, x.size)

    def drain_right_context_with_silence(self):
        lib().oracle_lseend_drain(self._h)

    @property
    def ready_chunks(self) -> int:
        return int(lib().oracle_lseend_ready(self._h))

    def emit_next_chunk(self):
        """(features [mel_frames x n_mels], mask [chunk_size], warmup) or None"""
        f = np.zeros((self.mel_frames, self.n_mels), np.float32)
        m = np.zeros(self.chunk_size, np.float32)
        w = C.c_int32()
        if not lib().oracle_lseend_emit(self._h, f.ctypes.data, m.ctypes.data, C.byref(w)):
            return None
        return f, m, int(w.value)

    def push(self, x, drain=False):
        """The library's push: enqueue, drain when asked, then every ready chunk.  Returns (features, masks, warmup)
        stacked over the chunks."""
        self.enqueue_audio(x)
        if drain:
            self.drain_right_context_with_silence()
        out = []
        while (c := self.emit_next_chunk()) is not None:
            out.append(c)
        f = np.stack([c[0] for c in out]) if out else np.zeros((0, self.mel_frames, self.n_mels), np.float32)
        m = np.stack([c[1] for c in out]) if out else np.zeros((0, self.chunk_size), np.float32)
        return f, m, np.array([c[2] for c in out], np.int32)

    def take_snapshot(self):
        lib().oracle_lseend_snapshot(self._h)

    def rollback(self):
        lib().oracle_lseend_rollback(self._h)

    def reset(self):
        lib().oracle_lseend_reset(self._h)

    def state(self) -> SimpleNamespace:
        """audio [unread samples], mel [unread rows x n_mels], cmn_mean, cmn_count, decoder_mask_end"""
        v = np.zeros(4, np.int64)
        lib().oracle_lseend_lengths(self._h, v.ctypes.data)
        audio = np.zeros(int(v[0]), np.float32)
        mel = np.zeros((int(v[1]), self.n_mels), np.float32)
        mean = np.zeros(self.n_mels, np.float32)
        lib().oracle_lseend_state(self._h, audio.ctypes.data, mel.ctypes.data, mean.ctypes.data)
        return SimpleNamespace(audio=audio, mel=mel, cmn_mean=mean, cmn_count=int(v[2]), decoder_mask_end=int(v[3]))
