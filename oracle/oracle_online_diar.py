"""ORACLE — TEST INFRASTRUCTURE ONLY.  Not part of the shipped product path.

ctypes front-end to ``liboracle_online_diar.so``, the sequential CPU restatement of streaming speaker tracking
(``oracle_online_diar.cpp``: DiarizerManager's chunk logic and segments, EmbeddingExtractor's input buffers, and
SpeakerManager's database with Speaker's FIFO, EMA and mergeWith), compiled into its own library with the main oracle's
pinned flags (``-O2 -ffp-contract=off`` on baseline x86-64).
Importers allowed: ``tests/``, ``__graft_entry__`` and ``scripts/``.  The product package never imports it.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRCS = [os.path.join(_HERE, "oracle_online_diar.cpp")]
_LIB = os.path.join(_HERE, "liboracle_online_diar.so")
_FLAGS = ["-std=c++17", "-O2", "-ffp-contract=off", "-fPIC", "-Wall", "-Wextra", "-shared"]

DIM, FIFO = 256, 50
SPEAKER = np.dtype([("key", "<i8"), ("numeric", "<i8"), ("update_count", "<i8"), ("duration", "<f4"),
                    ("named", "<i4"), ("has_numeric", "<i4"), ("permanent", "<i4"), ("raw_count", "<i4")], align=True)

_lib = None


def build(force: bool = False) -> None:
    """Compile liboracle_online_diar.so when it is missing or older than a source."""
    if force or not os.path.exists(_LIB) or any(os.path.getmtime(s) > os.path.getmtime(_LIB) for s in _SRCS):
        cxx = os.environ.get("CXX", "g++")
        subprocess.check_call([cxx, *_FLAGS, "-o", _LIB, *_SRCS])


def lib():
    global _lib
    if _lib is None:
        build()
        L = C.CDLL(_LIB)
        vp, i32, i64 = C.c_void_p, C.c_int32, C.c_int64
        L.oracle_od_new.restype = vp
        L.oracle_od_free.argtypes = [vp]
        L.oracle_od_inputs.argtypes = [vp, i64, i64, i32, vp, vp, vp]
        L.oracle_od_chunk.argtypes = [vp, vp, i32, i64, vp, C.c_double, vp, vp, vp, vp, vp, vp]
        L.oracle_od_chunk.restype = i32
        L.oracle_od_count.argtypes = [vp, C.POINTER(i64), C.POINTER(i64)]
        L.oracle_od_read.argtypes = [vp, vp, vp, vp]
        L.oracle_od_initialize.argtypes = [vp, i32, vp, vp, vp, i32, i32]
        L.oracle_od_remove.argtypes = [vp, i32, i64, i32]
        L.oracle_od_remove.restype = i32
        L.oracle_od_merge.argtypes = [vp, i32, i64, i32, i64, i32]
        L.oracle_od_merge.restype = i32
        L.oracle_od_set_permanent.argtypes = [vp, i32, i64, i32]
        L.oracle_od_set_permanent.restype = i32
        L.oracle_od_reset.argtypes = [vp, i32]
        L.oracle_od_query.argtypes = [vp, i32, vp, vp]
        L.oracle_od_upsert.argtypes = [vp, vp, vp, vp]
        _lib = L
    return _lib


def resolved(clustering_threshold=0.7, min_speech_duration=1.0, min_active_frames_count=10.0) -> np.ndarray:
    """speakerThreshold, embeddingThreshold, minSpeechDuration, minActiveFramesCount in float32"""
    t = np.float32(clustering_threshold)
    return np.array([t * np.float32(1.2), t * np.float32(0.8), min_speech_duration, min_active_frames_count],
                    np.float32)


def chunk_inputs(audio: np.ndarray, chunk_size: int):
    """(segmentation input, embedding waveform row 0) of one chunk"""
    a = np.ascontiguousarray(audio, np.float32)
    seg, wave = np.empty(160000, np.float32), np.empty(160000, np.float32)
    lib().oracle_od_inputs(a.ctypes.data if a.size else None, a.size, chunk_size, 0, seg.ctypes.data,
                           wave.ctypes.data, None)
    return seg, wave


def enrollment_inputs(audio: np.ndarray, frames: int):
    """(waveform row 0, mask row 0) of extractSpeakerEmbedding(from:)"""
    a = np.ascontiguousarray(audio, np.float32)
    wave, mask = np.empty(160000, np.float32), np.empty(frames, np.float32)
    lib().oracle_od_inputs(a.ctypes.data if a.size else None, a.size, 0, frames, None, wave.ctypes.data,
                           mask.ctypes.data)
    return wave, mask


class Session:
    """One SpeakerManager with DiarizerManager's chunk step"""

    def __init__(self):
        self._p = lib().oracle_od_new()

    def __del__(self):
        if getattr(self, "_p", None):
            lib().oracle_od_free(self._p)
            self._p = None

    def chunk(self, logits, chunk_size, model_embedding, offset, r):
        """logits [F x 7] and the model's embeddings [3 x 256] (rows whose need is 0 are replaced by zeros); returns
        masks, need, assigned and the segments' ids and values"""
        lg = np.ascontiguousarray(logits, np.float32)
        F = lg.shape[0]
        masks, need = np.empty((3, F), np.float32), np.empty(3, np.int32)
        emb = np.ascontiguousarray(model_embedding, np.float32).reshape(3, DIM)
        assigned = np.empty((3, 2), np.int64)
        bound = 3 * ((F + 1) // 2)
        ids, vals = np.empty((bound, 2), np.int64), np.empty((bound, 3), np.float32)
        n = lib().oracle_od_chunk(self._p, lg.ctypes.data, F, chunk_size, emb.ctypes.data, float(offset),
                                  np.ascontiguousarray(r, np.float32).ctypes.data, masks.ctypes.data,
                                  need.ctypes.data, assigned.ctypes.data, ids.ctypes.data, vals.ctypes.data)
        return masks, need, assigned, ids[:n].copy(), vals[:n].copy()

    def count(self):
        c, n = C.c_int64(), C.c_int64()
        lib().oracle_od_count(self._p, C.byref(c), C.byref(n))
        return c.value, n.value

    def read(self):
        c, _ = self.count()
        sp = np.zeros(c, SPEAKER)
        cur, raws = np.zeros((c, DIM), np.float32), np.zeros((c, FIFO, DIM), np.float32)
        if c:
            lib().oracle_od_read(self._p, sp.ctypes.data, cur.ctypes.data, raws.ctypes.data)
        return sp, cur, raws

    def initialize(self, speakers, current, raws, mode, preserve=True):
        sp = np.ascontiguousarray(speakers, SPEAKER)
        cur = np.ascontiguousarray(current, np.float32)
        rw = np.ascontiguousarray(raws, np.float32)
        lib().oracle_od_initialize(self._p, len(sp), sp.ctypes.data, cur.ctypes.data,
                                   rw.ctypes.data if rw.size else None, mode, int(preserve))

    def upsert(self, speaker, current, raws):
        sp = np.ascontiguousarray(np.asarray(speaker, SPEAKER).reshape(1))
        cur = np.ascontiguousarray(current, np.float32)
        rw = np.ascontiguousarray(raws, np.float32)
        lib().oracle_od_upsert(self._p, sp.ctypes.data, cur.ctypes.data, rw.ctypes.data if rw.size else None)

    def remove(self, named, key, keep=True):
        return bool(lib().oracle_od_remove(self._p, named, key, int(keep)))

    def merge(self, src, dst, stop=True):
        return bool(lib().oracle_od_merge(self._p, src[0], src[1], dst[0], dst[1], int(stop)))

    def set_permanent(self, named, key, flag):
        return bool(lib().oracle_od_set_permanent(self._p, named, key, int(flag)))

    def reset(self, keep=False):
        lib().oracle_od_reset(self._p, int(keep))

    def query(self, emb):
        e = np.ascontiguousarray(emb, np.float32).reshape(-1, DIM)
        c, _ = self.count()
        out = np.zeros((len(e), c), np.float32)
        if c and len(e):
            lib().oracle_od_query(self._p, len(e), e.ctypes.data, out.ctypes.data)
        return out
