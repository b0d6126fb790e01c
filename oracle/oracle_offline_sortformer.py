"""ORACLE — TEST INFRASTRUCTURE ONLY.  Not part of the shipped product path.

ctypes front-end to ``liboracle_offline_sortformer.so``, the sequential CPU restatement of OfflineSortformerDiarizer's
window work (``oracle_offline_sortformer.cpp``: runOffline's copy, SortformerSpeakerStitcher.alignment with its
recursive enumeration, and processComplete's window loop, which calls the model one window at a time), compiled into
its own library with the main oracle's pinned flags (``-O2 -ffp-contract=off`` on baseline x86-64).  ``process_complete``
adds the timeline rebuild through ``oracle_timeline``.  Importers allowed: ``tests/``, ``__graft_entry__`` and
``scripts/``.  The product package never imports it.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRCS = [os.path.join(_HERE, "oracle_offline_sortformer.cpp")]
_LIB = os.path.join(_HERE, "liboracle_offline_sortformer.so")
_FLAGS = ["-std=c++17", "-O2", "-ffp-contract=off", "-fPIC", "-Wall", "-Wextra", "-shared"]

WINDOW_OUT, SUBSAMPLING, SPEAKERS, MELS = 384, 8, 4, 128
WINDOW_MEL = WINDOW_OUT * SUBSAMPLING

MODEL = C.CFUNCTYPE(None, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p)

_lib = None


def build(force: bool = False) -> None:
    """Compile liboracle_offline_sortformer.so when it is missing or older than a source."""
    if force or not os.path.exists(_LIB) or any(os.path.getmtime(s) > os.path.getmtime(_LIB) for s in _SRCS):
        cxx = os.environ.get("CXX", "g++")
        subprocess.check_call([cxx, *_FLAGS, "-o", _LIB, *_SRCS])


def lib():
    global _lib
    if _lib is None:
        build()
        L = C.CDLL(_LIB)
        vp, i64 = C.c_void_p, C.c_int64
        L.oracle_osf_run_offline.argtypes = [vp, i64, vp, vp]
        L.oracle_osf_run_offline.restype = None
        L.oracle_osf_alignment.argtypes = [vp, vp, i64, i64, vp]
        L.oracle_osf_alignment.restype = None
        L.oracle_osf_process_complete.argtypes = [vp, i64, i64, MODEL, vp, vp, vp, vp]
        L.oracle_osf_process_complete.restype = i64
        _lib = L
    return _lib


def _f32(a):
    return np.ascontiguousarray(a, np.float32)


def run_offline(mel_time_major, valid_mel_frames):
    """(mel [128 x 3072], mel_length) of one window's time-major rows"""
    rows = _f32(mel_time_major).reshape(-1)
    out, ml = np.empty((MELS, WINDOW_MEL), np.float32), C.c_int32()
    lib().oracle_osf_run_offline(rows.ctypes.data, int(valid_mel_frames), out.ctypes.data, C.byref(ml))
    return out, int(ml.value)


def alignment(global_rows, window_rows, frames, num_speakers=SPEAKERS):
    """mapping [num_speakers] with mapping[window column] = global speaker"""
    g, w = _f32(global_rows).reshape(-1), _f32(window_rows).reshape(-1)
    assert g.size >= frames * num_speakers and w.size >= frames * num_speakers
    out = np.empty(max(int(num_speakers), 0), np.int32)
    lib().oracle_osf_alignment(g.ctypes.data, w.ctypes.data, int(frames), int(num_speakers), out.ctypes.data)
    return out.tolist()


def stitch(mel_time_major, num_mel_frames, overlap, model):
    """processComplete's window loop over one file's rows [num_mel_frames x 128], calling
    model(mel [128 x 3072], mel_length) -> speaker_preds [384 x 4] once per window in order:
    (global [totalOut x 4], mappings [windows x 4])"""
    n = int(num_mel_frames)
    rows = _f32(mel_time_major).reshape(-1)
    assert rows.size >= n * MELS
    total = (n + SUBSAMPLING - 1) // SUBSAMPLING
    most = n // ((WINDOW_OUT - max(0, min(int(overlap), WINDOW_OUT - 1))) * SUBSAMPLING) + 2
    glob, maps, windows = np.zeros((max(total, 1), SPEAKERS), np.float32), np.zeros((most, SPEAKERS), np.int32), C.c_int64()
    errors = []

    def call(mel_p, mel_length, preds_p, _ctx):
        try:
            mel = np.ctypeslib.as_array(C.cast(mel_p, C.POINTER(C.c_float)), (MELS, WINDOW_MEL)).copy()
            out = _f32(model(mel, int(mel_length))).reshape(WINDOW_OUT * SPEAKERS)
            C.memmove(preds_p, out.ctypes.data, out.nbytes)
        except Exception as e:   # noqa: BLE001 — carried out of the callback
            errors.append(e)

    cb = MODEL(call)
    got = lib().oracle_osf_process_complete(rows.ctypes.data if rows.size else None, n, int(overlap), cb, None,
                                            glob.ctypes.data, maps.ctypes.data, C.byref(windows))
    if errors:
        raise errors[0]
    return glob[:got].copy(), maps[:windows.value].copy()


def process_complete(mel_time_major, num_mel_frames, overlap, model, timeline_config):
    """processComplete after the mel: the stitched rows rebuilt into a fresh timeline (keepingSpeakers: false,
    isComplete: true).  Returns (timeline, finalized segments, tentative segments, global rows)."""
    from oracle import oracle_timeline as TL
    glob, _ = stitch(mel_time_major, num_mel_frames, overlap, model)
    tl = TL.Timeline(timeline_config)
    if glob.shape[0] == 0:
        return tl, np.zeros(0, TL.SEGMENT), np.zeros(0, TL.SEGMENT), glob
    fin, ten = tl.rebuild(glob, is_complete=True)
    return tl, fin, ten, glob
