"""ORACLE — TEST INFRASTRUCTURE ONLY.  Not part of the shipped product path.

ctypes front-end to ``liboracle_prepare.so``, the CPU restatement of the offline diarizer's prepare stage
(``oracle_prepare.cpp``: OfflineSegmentationProcessor's windows and powerset decoding, WeightInterpolation, and the
bookkeeping of OfflineEmbeddingExtractor).  It has its own library so that the main oracle (``oracle.py``,
``liboracle.so``) is untouched; it is compiled with the main oracle's pinned flags (``-O2 -ffp-contract=off`` on baseline
x86-64: every float32 operation rounded as the C++ states it).
Importers allowed: ``tests/``, ``__graft_entry__`` and ``scripts/``.  The product package never imports it.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess
from types import SimpleNamespace

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, "oracle_prepare.cpp")
_LIB = os.path.join(_HERE, "liboracle_prepare.so")
_FLAGS = ["-std=c++17", "-O2", "-ffp-contract=off", "-fPIC", "-Wall", "-Wextra", "-shared"]

_lib = None

SEG_DEFAULTS = dict(sample_rate=16000, window_duration=10.0, step_ratio=0.2, speech_onset_threshold=0.5)
PLAN_DEFAULTS = dict(exclude_overlap=True, min_segment_duration=1.0, skip_threshold=-1.0, weight_frames=589,
                     audio_sample_count=160000, fbank_batch=32)


def build(force: bool = False) -> None:
    """Compile liboracle_prepare.so when it is missing or older than its source."""
    if force or not os.path.exists(_LIB) or os.path.getmtime(_SRC) > os.path.getmtime(_LIB):
        cxx = os.environ.get("CXX", "g++")
        subprocess.check_call([cxx, *_FLAGS, "-o", _LIB, _SRC])


def lib():
    global _lib
    if _lib is None:
        build()
        L = C.CDLL(_LIB)
        vp, i32, i64, f32, f64 = C.c_void_p, C.c_int32, C.c_longlong, C.c_float, C.c_double
        L.oracle_seg_window_count.argtypes = [i64, i32, f64, f64, C.POINTER(i64), C.POINTER(i64)]
        L.oracle_seg_window_count.restype = i64
        L.oracle_seg_windows.argtypes = [vp, i64, i32, f64, f64, vp, vp]
        L.oracle_seg_windows.restype = None
        L.oracle_seg_decode.argtypes = [vp, i32, i32, i32, f32, vp, vp, vp, C.POINTER(i64), vp]
        L.oracle_seg_decode.restype = None
        L.oracle_weight_resample.argtypes = [vp, i64, i32, i32, vp]
        L.oracle_weight_resample.restype = None
        L.oracle_interp_table.argtypes = [i32, i32, vp, vp, vp, vp]
        L.oracle_interp_table.restype = None
        L.oracle_embedding_plan.argtypes = [vp, i32, i32, i32, vp, i32, f64, i64, i32, f64, i32, f64, f32, i32, i32] + \
            [vp] * 14
        L.oracle_embedding_plan.restype = i32
        L.oracle_embed_windows.argtypes = [vp, i64, vp, i32, vp, i32, i32, f64, i32, vp]
        L.oracle_embed_windows.restype = None
        _lib = L
    return _lib


def _p(a):
    return a.ctypes.data if a is not None and a.size else None


def seg_window_count(total_samples: int, sample_rate=16000, window_duration=10.0, step_ratio=0.2, **_):
    """(chunks, samplesPerWindow, samplesPerStep)"""
    w, s = C.c_longlong(), C.c_longlong()
    n = lib().oracle_seg_window_count(int(total_samples), sample_rate, window_duration, step_ratio, C.byref(w), C.byref(s))
    return int(n), int(w.value), int(s.value)


def seg_windows(audio, sample_rate=16000, window_duration=10.0, step_ratio=0.2, **_):
    """(windows float32 [chunks x window], chunkOffsets float64 [chunks])"""
    a = np.ascontiguousarray(audio, np.float32)
    n, w, _s = seg_window_count(a.size, sample_rate, window_duration, step_ratio)
    out, offs = np.zeros((n, w), np.float32), np.zeros(n, np.float64)
    lib().oracle_seg_windows(_p(a), a.size, sample_rate, window_duration, step_ratio, _p(out), _p(offs))
    return out, offs


def seg_decode(logits, speech_onset_threshold=0.5, **_):
    """logits [chunks x frames x classes] -> namespace(log_probs, speaker_weights, class_histogram, speech_frames,
    speech_probability [chunks x frames])"""
    x = np.ascontiguousarray(logits, np.float32)
    c, f, k = x.shape
    lp, w = np.zeros((c, f, k), np.float32), np.zeros((c, f, 3), np.float32)
    hist, sp, n = np.zeros(8, np.int64), np.zeros((c, f), np.float32), C.c_longlong()
    lib().oracle_seg_decode(_p(x), c, f, k, speech_onset_threshold, _p(lp), _p(w), hist.ctypes.data, C.byref(n), _p(sp))
    return SimpleNamespace(log_probs=lp, speaker_weights=w, class_histogram=hist, speech_frames=int(n.value),
                           speech_probability=sp)


def weight_resample(rows, out_len: int) -> np.ndarray:
    r = np.ascontiguousarray(rows, np.float32)
    r2 = r.reshape(-1, r.shape[-1])
    out = np.zeros((r2.shape[0], out_len), np.float32)
    lib().oracle_weight_resample(_p(r2), r2.shape[0], r2.shape[1], out_len, _p(out))
    return out.reshape(r.shape[:-1] + (out_len,))


def interp_table(in_len: int, out_len: int):
    """(left, right int32 [out_len], weightLeft, weightRight float32 [out_len])"""
    l, r = np.zeros(out_len, np.int32), np.zeros(out_len, np.int32)
    wl, wr = np.zeros(out_len, np.float32), np.zeros(out_len, np.float32)
    lib().oracle_interp_table(in_len, out_len, _p(l), _p(r), _p(wl), _p(wr))
    return l, r, wl, wr


def embedding_plan(speaker_weights, chunk_offsets, frame_duration: float, total_samples: int, seg=None, plan=None):
    """The embedding stage's bookkeeping: namespace with the per-entry arrays (trimmed to the entry count), `counters`
    (evaluated, empty, fallback, skipped), `active` [chunks] and `sums` [chunks x speakers x 3]."""
    seg = {**SEG_DEFAULTS, **(seg or {})}
    plan = {**PLAN_DEFAULTS, **(plan or {})}
    w = np.ascontiguousarray(speaker_weights, np.float32)
    c, f, s = w.shape
    offs = np.ascontiguousarray(chunk_offsets if chunk_offsets is not None else [], np.float64)
    cap, wf = max(c * s, 1), plan["weight_frames"]
    i32 = lambda: np.zeros(cap, np.int32)
    ci, si, sf, ef, fb, ro = i32(), i32(), i32(), i32(), i32(), i32()
    st, et, ms = np.zeros(cap, np.float64), np.zeros(cap, np.float64), np.zeros(cap, np.float32)
    fw, mw = np.zeros((cap, max(f, 1)), np.float32), np.zeros((cap, wf), np.float32)
    counters, active, sums = np.zeros(4, np.int64), np.zeros(max(c, 1), np.int32), np.zeros((max(c, 1), max(s, 1), 3), np.float32)
    n = lib().oracle_embedding_plan(_p(w), c, f, s, _p(offs), offs.size, frame_duration, int(total_samples),
                                    seg["sample_rate"], seg["window_duration"], int(plan["exclude_overlap"]),
                                    plan["min_segment_duration"], plan["skip_threshold"], wf, plan["fbank_batch"],
                                    _p(ci), _p(si), _p(sf), _p(ef), _p(st), _p(et), _p(ms), _p(fb), _p(ro), _p(fw), _p(mw),
                                    _p(counters), _p(active), _p(sums))
    return SimpleNamespace(count=n, chunk_index=ci[:n], speaker_index=si[:n], start_frame=sf[:n], end_frame=ef[:n],
                           start_time=st[:n], end_time=et[:n], mask_sum=ms[:n], used_fallback=fb[:n], reuse_of=ro[:n],
                           frame_weights=fw[:n, :f], model_weights=mw[:n], counters=counters, active=active[:c],
                           sums=sums[:c, :s])


def embed_windows(audio, chunk_offsets, chunks, audio_sample_count=160000, sample_rate=16000, window_duration=10.0, **_):
    a = np.ascontiguousarray(audio, np.float32)
    offs = np.ascontiguousarray(chunk_offsets if chunk_offsets is not None else [], np.float64)
    ch = np.ascontiguousarray(chunks, np.int32)
    out = np.zeros((ch.size, audio_sample_count), np.float32)
    lib().oracle_embed_windows(_p(a), a.size, _p(offs), offs.size, _p(ch), ch.size, sample_rate, window_duration,
                               audio_sample_count, _p(out))
    return out
