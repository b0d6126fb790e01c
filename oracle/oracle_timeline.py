"""ORACLE — TEST INFRASTRUCTURE ONLY.  Not part of the shipped product path.

ctypes front-end to ``liboracle_timeline.so``, the sequential CPU restatement of DiarizerTimeline's numeric core
(``oracle_timeline.cpp``: DiarizerTimeline.swift, one timeline per object).  It has its own library, compiled with the
main oracle's pinned flags (``-O2 -ffp-contract=off`` on baseline x86-64).
Importers allowed: ``tests/``, ``__graft_entry__`` and ``scripts/``.  The product package never imports it.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess
from types import SimpleNamespace

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, "oracle_timeline.cpp")
_LIB = os.path.join(_HERE, "liboracle_timeline.so")
_FLAGS = ["-std=c++17", "-O2", "-ffp-contract=off", "-fPIC", "-Wall", "-Wextra", "-shared"]

SEGMENT = np.dtype([("start_frame", np.int64), ("end_frame", np.int64), ("activity", np.float32),
                    ("speaker", np.int32)])
SCRATCH = np.dtype([("start_frame", np.int64), ("end_frame", np.int64), ("unmerged_start_frame", np.int64),
                    ("active_frame_count", np.int64), ("unmerged_active_frame_count", np.int64),
                    ("activity_sum", np.float32), ("unmerged_activity_sum", np.float32), ("speaking", np.int32),
                    ("has_segment", np.int32)])

_lib = None


def build(force: bool = False) -> None:
    """Compile liboracle_timeline.so when it is missing or older than its source."""
    if force or not os.path.exists(_LIB) or os.path.getmtime(_SRC) > os.path.getmtime(_LIB):
        cxx = os.environ.get("CXX", "g++")
        subprocess.check_call([cxx, *_FLAGS, "-o", _LIB, _SRC])


def lib():
    global _lib
    if _lib is None:
        build()
        L = C.CDLL(_LIB)
        vp, i32, i64 = C.c_void_p, C.c_int32, C.c_int64
        L.oracle_tl_create.argtypes = [vp, vp]
        L.oracle_tl_create.restype = vp
        for name in ("oracle_tl_destroy", "oracle_tl_finalize", "oracle_tl_reset"):
            getattr(L, name).argtypes = [vp]
            getattr(L, name).restype = None
        L.oracle_tl_push.argtypes = [vp, vp, i64, vp, i64, i32, vp, vp, vp]
        L.oracle_tl_push.restype = None
        L.oracle_tl_clear_speaker.argtypes = [vp, i64]
        L.oracle_tl_clear_speaker.restype = None
        L.oracle_tl_lengths.argtypes = [vp, vp]
        L.oracle_tl_lengths.restype = None
        L.oracle_tl_state.argtypes = [vp, vp, vp, vp]
        L.oracle_tl_state.restype = None
        _lib = L
    return _lib


def _get(cfg, k):
    return cfg[k] if isinstance(cfg, dict) else getattr(cfg, k)


def bound(n: int, m: int) -> tuple[int, int]:
    """(finalized, tentative) segments one speaker may emit in a push of n finalized and m tentative rows"""
    return (n // 2 + 1 if n > 0 else 0), (m + 1) // 2 + 1


class Timeline:
    """One DiarizerTimeline.  ``cfg`` has the fa_diarizer_timeline_config field names (a dict or attributes);
    ``max_stored_frames`` None (or < 0) is the reference's nil, unlimited."""

    def __init__(self, cfg):
        self.S = int(_get(cfg, "num_speakers"))
        ms = _get(cfg, "max_stored_frames")
        ints = np.array([self.S, _get(cfg, "onset_pad_frames"), _get(cfg, "offset_pad_frames"), _get(cfg, "min_frames_on"),
                         _get(cfg, "min_frames_off"), int(_get(cfg, "activity_type")), -1 if ms is None else ms], np.int64)
        floats = np.array([_get(cfg, "frame_duration_seconds"), _get(cfg, "onset_threshold"),
                           _get(cfg, "offset_threshold")], np.float32)
        self._h = lib().oracle_tl_create(ints.ctypes.data, floats.ctypes.data)

    def __del__(self):
        try:
            lib().oracle_tl_destroy(self._h)
        except Exception:
            pass

    def _rows(self, a):
        return np.ascontiguousarray(np.asarray(a, np.float32).reshape(-1, self.S))

    def _push(self, fin, ten, rebuild):
        f, t = self._rows(fin), self._rows(ten)
        bf, bt = bound(f.shape[0], t.shape[0])
        fo, to = np.zeros(self.S * bf + 1, SEGMENT), np.zeros(self.S * bt + 1, SEGMENT)
        counts = np.zeros(2, np.int64)
        lib().oracle_tl_push(self._h, f.ctypes.data, f.shape[0], t.ctypes.data, t.shape[0], rebuild, fo.ctypes.data,
                             to.ctypes.data, counts.ctypes.data)
        return fo[:counts[0]].copy(), to[:counts[1]].copy()

    def add_chunk(self, finalized, tentative=()):
        """addChunk: (finalized segments, tentative segments) as SEGMENT records in emission order"""
        return self._push(finalized, tentative, -1)

    def rebuild(self, finalized, tentative=(), is_complete=True):
        return self._push(finalized, tentative, int(bool(is_complete)))

    def finalize(self):
        lib().oracle_tl_finalize(self._h)

    def reset(self):
        lib().oracle_tl_reset(self._h)

    def clear_speaker(self, k: int):
        lib().oracle_tl_clear_speaker(self._h, int(k))

    def state(self):
        """namespace(finalized_frames, stored [rows x S], tentative [rows x S], scratch [S] of SCRATCH)"""
        v = np.zeros(3, np.int64)
        lib().oracle_tl_lengths(self._h, v.ctypes.data)
        stored = np.zeros((int(v[1]), self.S), np.float32)
        tent = np.zeros((int(v[2]), self.S), np.float32)
        scratch = np.zeros(self.S, SCRATCH)
        lib().oracle_tl_state(self._h, stored.ctypes.data, tent.ctypes.data, scratch.ctypes.data)
        return SimpleNamespace(finalized_frames=int(v[0]), stored=stored, tentative=tent, scratch=scratch)
