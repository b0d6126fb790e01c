"""ORACLE — TEST INFRASTRUCTURE ONLY.  Not part of the shipped product path.

ctypes front-end to ``liboracle_sortformer.so``, the sequential CPU restatement of Sortformer's streaming state update
(``oracle_sortformer.cpp``: SortformerStateUpdater.swift and SortformerStreamingState, one session per object).  It has
its own library, compiled with the main oracle's pinned flags (``-O2 -ffp-contract=off`` on baseline x86-64).
Importers allowed: ``tests/``, ``__graft_entry__`` and ``scripts/``.  The product package never imports it.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess
from types import SimpleNamespace

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, "oracle_sortformer.cpp")
_LIB = os.path.join(_HERE, "liboracle_sortformer.so")
_FLAGS = ["-std=c++17", "-O2", "-ffp-contract=off", "-fPIC", "-Wall", "-Wextra", "-shared"]

D, S = 512, 4
INT_FIELDS = ("chunk_len", "chunk_left_context", "chunk_right_context", "fifo_len", "spkcache_len",
              "spkcache_update_period", "spkcache_sil_frames_per_spk")
FLOAT_FIELDS = ("silence_threshold", "pred_score_threshold", "scores_boost_latest", "strong_boost_rate",
                "weak_boost_rate", "min_pos_scores_rate")
INSUFFICIENT_PREDS, INSUFFICIENT_CHUNK = 1, 2

_lib = None


def build(force: bool = False) -> None:
    """Compile liboracle_sortformer.so when it is missing or older than its source."""
    if force or not os.path.exists(_LIB) or os.path.getmtime(_SRC) > os.path.getmtime(_LIB):
        cxx = os.environ.get("CXX", "g++")
        subprocess.check_call([cxx, *_FLAGS, "-o", _LIB, _SRC])


def lib():
    global _lib
    if _lib is None:
        build()
        L = C.CDLL(_LIB)
        vp, i32, i64 = C.c_void_p, C.c_int32, C.c_longlong
        L.oracle_sf_create.argtypes = [vp, vp]
        L.oracle_sf_create.restype = vp
        L.oracle_sf_destroy.argtypes = [vp]
        L.oracle_sf_destroy.restype = None
        L.oracle_sf_config.argtypes = [vp, vp]
        L.oracle_sf_config.restype = None
        L.oracle_sf_update.argtypes = [vp, vp, i64, vp, i64, i32, i32, vp, vp, vp]
        L.oracle_sf_update.restype = i32
        L.oracle_sf_lengths.argtypes = [vp, vp]
        L.oracle_sf_lengths.restype = None
        L.oracle_sf_state.argtypes = [vp] * 6
        L.oracle_sf_state.restype = None
        L.oracle_sf_last_pop.argtypes = [vp] * 3
        L.oracle_sf_last_pop.restype = i32
        L.oracle_sf_last_compression.argtypes = [vp] * 8
        L.oracle_sf_last_compression.restype = i32
        _lib = L
    return _lib


def _p(a):
    return a.ctypes.data if a is not None and a.size else None


class Session:
    """One SortformerStreamingState driven by streamingUpdate.  ``cfg`` maps the fa_sortformer_config field names to
    values (any object with those attributes works too)."""

    def __init__(self, cfg):
        get = (lambda k: cfg[k]) if isinstance(cfg, dict) else (lambda k: getattr(cfg, k))
        ints = np.array([get(k) for k in INT_FIELDS], np.int32)
        floats = np.array([get(k) for k in FLOAT_FIELDS], np.float32)
        self._h = lib().oracle_sf_create(ints.ctypes.data, floats.ctypes.data)
        out = np.zeros(7, np.int32)
        lib().oracle_sf_config(self._h, out.ctypes.data)
        self.config = dict(zip(INT_FIELDS, out.tolist()))
        self.chunks = 0
        self._rows = 0   # the most rows one update carried: bounds the pre-compression cache

    def __del__(self):
        try:
            lib().oracle_sf_destroy(self._h)
        except Exception:
            pass

    def update(self, chunk, preds, lc: int, rc: int):
        """streamingUpdate(chunk [rows x 512], preds [rows x 4]) -> (status, confirmed [core x 4], tentative [rc x 4])"""
        ch = np.ascontiguousarray(chunk, np.float32).reshape(-1)
        pr = np.ascontiguousarray(preds, np.float32).reshape(-1)
        counts = np.zeros(2, np.int64)
        cap = max(pr.size, 1)
        conf, tent = np.zeros(cap, np.float32), np.zeros(cap, np.float32)
        st = lib().oracle_sf_update(self._h, _p(ch), ch.size, _p(pr), pr.size, int(lc), int(rc), conf.ctypes.data,
                                    tent.ctypes.data, counts.ctypes.data)
        if st:
            return st, None, None
        self.chunks += 1
        self._rows = max(self._rows, ch.size // D)
        return 0, conf[:counts[0]].reshape(-1, S), tent[:counts[1]].reshape(-1, S)

    def lengths(self):
        v = np.zeros(5, np.int64)
        lib().oracle_sf_lengths(self._h, v.ctypes.data)
        return SimpleNamespace(spkcache_length=int(v[0]), fifo_length=int(v[1]), has_spkcache_preds=bool(v[2]),
                               has_fifo_preds=bool(v[3]), silence_frames=int(v[4]), chunks=self.chunks)

    def state(self):
        n = self.lengths()
        sc, sp = np.zeros((n.spkcache_length, D), np.float32), np.zeros((n.spkcache_length, S), np.float32)
        ff, fp = np.zeros((n.fifo_length, D), np.float32), np.zeros((n.fifo_length, S), np.float32)
        mean = np.zeros(D, np.float32)
        lib().oracle_sf_state(self._h, _p(sc), _p(sp), _p(ff), _p(fp), mean.ctypes.data)
        return SimpleNamespace(**vars(n), spkcache=sc, spkcache_preds=sp if n.has_spkcache_preds else None, fifo=ff,
                               fifo_preds=fp if n.has_fifo_preds else None, mean_silence=mean)

    def model_inputs(self):
        """runMainModel's padded copies (SortformerModelInference.swift:283-303): ([spkcacheLen x 512], [fifoLen x 512],
        spkcacheLength, fifoLength)"""
        s = self.state()
        sc = np.zeros((self.config["spkcache_len"], D), np.float32)
        ff = np.zeros((self.config["fifo_len"], D), np.float32)
        sc[:s.spkcache_length] = s.spkcache
        ff[:s.fifo_length] = s.fifo
        return sc, ff, s.spkcache_length, s.fifo_length

    def last_pop(self):
        """(embeddings [pop x 512], predictions [pop x 4]) the last update popped"""
        cap = self.config["fifo_len"] + self._rows + 1
        e, p = np.zeros((cap, D), np.float32), np.zeros((cap, S), np.float32)
        n = lib().oracle_sf_last_pop(self._h, e.ctypes.data, p.ctypes.data)
        return e[:n], p[:n]

    def last_compression(self):
        """The last update's compression stage by stage, or None: its input spkcachePreds, the scores, after disabling
        and the latest boost, after the strong and the weak boost ([L x 4] each), the gathered frame indices and
        disabled flags [spkcacheLen]."""
        K = self.config["spkcache_len"]
        L = K + self.config["fifo_len"] + self._rows + 1
        bufs = [np.zeros((L, S), np.float32) for _ in range(5)]
        idx, dis = np.zeros(K, np.int32), np.zeros(K, np.int32)
        n = lib().oracle_sf_last_compression(self._h, *[b.ctypes.data for b in bufs], idx.ctypes.data, dis.ctypes.data)
        if n == 0:
            return None
        return SimpleNamespace(frames=n, preds=bufs[0][:n], scores=bufs[1][:n], disabled=bufs[2][:n],
                               strong=bufs[3][:n], weak=bufs[4][:n], indices=idx, is_disabled=dis)
