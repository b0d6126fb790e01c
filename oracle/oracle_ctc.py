"""ORACLE — TEST INFRASTRUCTURE ONLY.  Not part of the shipped product path.

ctypes front-end to ``liboracle_ctc.so``, the sequential CPU restatement of CTC keyword spotting (``oracle_ctc.cpp``:
applyLogSoftmax, the chunk concatenation with mergeOverlapFrame, and CtcDPAlgorithm's fillDPTable,
ctcWordSpotConstrained and ctcWordSpotMultiple with full tables), compiled into its own library with the main oracle's
pinned flags (``-O2 -ffp-contract=off`` on baseline x86-64).
Importers allowed: ``tests/``, ``__graft_entry__`` and ``scripts/``.  The product package never imports it.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRCS = [os.path.join(_HERE, "oracle_ctc.cpp")]
_LIB = os.path.join(_HERE, "liboracle_ctc.so")
_FLAGS = ["-std=c++17", "-O2", "-ffp-contract=off", "-fPIC", "-Wall", "-Wextra", "-shared"]

WILDCARD = -1
DEFAULT_BLANK = 1024

_lib = None


def build(force: bool = False) -> None:
    """Compile liboracle_ctc.so when it is missing or older than a source."""
    deps = _SRCS + [os.path.join(_HERE, "oracle_float.h")]
    if force or not os.path.exists(_LIB) or any(os.path.getmtime(s) > os.path.getmtime(_LIB) for s in deps):
        cxx = os.environ.get("CXX", "g++")
        subprocess.check_call([cxx, *_FLAGS, "-o", _LIB, *_SRCS])


def lib():
    global _lib
    if _lib is None:
        build()
        L = C.CDLL(_LIB)
        vp, i32, i64, f32 = C.c_void_p, C.c_int32, C.c_int64, C.c_float
        L.oracle_ctc_log_softmax.argtypes = [vp, i32, i32, i32, f32, f32, i32, vp]
        L.oracle_ctc_log_softmax.restype = None
        L.oracle_ctc_merge_chunks.argtypes = [vp, vp, i32, i32, i32, vp]
        L.oracle_ctc_merge_chunks.restype = C.c_longlong
        L.oracle_ctc_constrained.argtypes = [vp, i32, i32, vp, i32, i64, i64, i32, vp, vp, vp]
        L.oracle_ctc_constrained.restype = None
        L.oracle_ctc_multiple.argtypes = [vp, i32, i32, vp, i32, f32, i32, vp, vp, vp, i32]
        L.oracle_ctc_multiple.restype = i32
        L.oracle_ctc_threshold.argtypes = [i32, f32, i32]
        L.oracle_ctc_threshold.restype = f32
        L.oracle_ctc_non_wildcard_count.argtypes = [vp, i32]
        L.oracle_ctc_non_wildcard_count.restype = i32
        _lib = L
    return _lib


def _f32(a):
    return np.ascontiguousarray(a, dtype=np.float32)


def _i32(a):
    return np.ascontiguousarray(np.asarray(a, dtype=np.int64).astype(np.int32))


def log_softmax(logits, temperature=1.0, blank_bias=0.0, blank_id=DEFAULT_BLANK, vocab_major=False):
    """applyLogSoftmax: [T x V] (or the vocab-major [V x T]) logits -> [T x V] log-probs"""
    x = _f32(logits)
    T, V = (x.shape[1], x.shape[0]) if vocab_major else x.shape
    out = np.empty((T, V), np.float32)
    if T and V:
        lib().oracle_ctc_log_softmax(x.ctypes.data, T, V, int(vocab_major), temperature, blank_bias, blank_id,
                                     out.ctypes.data)
    return out


def merge_chunks(chunks, overlap_frames):
    """computeLogProbsChunked's concatenation of per-chunk [rows x V] log-probs"""
    chunks = [_f32(c) for c in chunks]
    V = next((c.shape[1] for c in chunks if c.ndim == 2 and c.shape[0]), 0)
    flat = np.concatenate([c.reshape(-1, V) for c in chunks]) if chunks and V else np.zeros((0, max(V, 1)), np.float32)
    off = np.zeros(len(chunks) + 1, np.int64)
    off[1:] = np.cumsum([len(c) for c in chunks]) if chunks else []
    out = np.empty_like(flat)
    rows = lib().oracle_ctc_merge_chunks(flat.ctypes.data, off.ctypes.data, len(chunks), V, overlap_frames,
                                         out.ctypes.data) if V else 0
    return out[:rows].copy()


def word_spot_constrained(log_probs, tokens, search_start, search_end, blank_id=DEFAULT_BLANK):
    """ctcWordSpotConstrained -> (score, start_frame, end_frame)"""
    lp = _f32(log_probs).reshape(len(log_probs), -1) if len(log_probs) else np.zeros((0, 1), np.float32)
    tok = _i32(tokens)
    s, a, b = C.c_float(), C.c_int64(), C.c_int64()
    lib().oracle_ctc_constrained(lp.ctypes.data, lp.shape[0], lp.shape[1], tok.ctypes.data, len(tok), search_start,
                                 search_end, blank_id, C.byref(s), C.byref(a), C.byref(b))
    return np.float32(s.value), a.value, b.value


def word_spot_multiple(log_probs, tokens, min_score=-15.0, blank_id=DEFAULT_BLANK):
    """ctcWordSpotMultiple with mergeOverlap -> [(score, start_frame, end_frame)]"""
    lp = _f32(log_probs).reshape(len(log_probs), -1) if len(log_probs) else np.zeros((0, 1), np.float32)
    tok = _i32(tokens)
    T = lp.shape[0]
    cap = T // 2 + 2
    sc, st, en = np.empty(cap, np.float32), np.empty(cap, np.int32), np.empty(cap, np.int32)
    n = lib().oracle_ctc_multiple(lp.ctypes.data, T, lp.shape[1], tok.ctypes.data, len(tok), min_score, blank_id,
                                  sc.ctypes.data, st.ctypes.data, en.ctypes.data, cap)
    assert n <= cap
    return [(np.float32(sc[i]), int(st[i]), int(en[i])) for i in range(n)]


def threshold(min_score, n_tokens):
    """spotKeywordsFromLogProbs' threshold of a term of n tokens (min_score None: -15 for every term)"""
    return np.float32(lib().oracle_ctc_threshold(int(min_score is not None), 0.0 if min_score is None else min_score,
                                                 n_tokens))


def non_wildcard_count(tokens):
    tok = _i32(tokens)
    return int(lib().oracle_ctc_non_wildcard_count(tok.ctypes.data, len(tok)))


def spot(clips, terms, min_score=None, blank_id=DEFAULT_BLANK):
    """spotKeywordsFromLogProbs without the text filter over every clip: counts [B x K] and the detections
    [(clip, term, score, start, end)] in clip, term, merged order"""
    counts = np.zeros((len(clips), len(terms)), np.int64)
    det = []
    for b, lp in enumerate(clips):
        for k, tok in enumerate(terms):
            found = word_spot_multiple(lp, tok, threshold(min_score, len(tok)), blank_id) if len(tok) else []
            counts[b, k] = len(found)
            det += [(b, k, s, a, e) for s, a, e in found]
    return counts, det
