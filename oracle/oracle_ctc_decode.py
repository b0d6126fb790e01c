"""ORACLE — TEST INFRASTRUCTURE ONLY.  Not part of the shipped product path.

ctypes front-end to ``liboracle_ctc_decode.so``, the sequential CPU restatement of CTC decoding
(``oracle_ctc_decode.cpp``: ctcGreedyDecode, ctcBeamSearch with its ARPA bigram LM terms, ARPALanguageModel.score and
logAddExp, prefixes as consed trie ids in an insertion-ordered map), compiled into its own library with the main
oracle's pinned flags (``-O2 -ffp-contract=off`` on baseline x86-64).
Importers allowed: ``tests/``, ``__graft_entry__`` and ``scripts/``.  The product package never imports it.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRCS = [os.path.join(_HERE, "oracle_ctc_decode.cpp")]
_LIB = os.path.join(_HERE, "liboracle_ctc_decode.so")
_FLAGS = ["-std=c++17", "-O2", "-ffp-contract=off", "-fPIC", "-Wall", "-Wextra", "-shared"]

DEFAULT_BLANK = 1024

_lib = None


def build(force: bool = False) -> None:
    """Compile liboracle_ctc_decode.so when it is missing or older than a source."""
    if force or not os.path.exists(_LIB) or any(os.path.getmtime(s) > os.path.getmtime(_LIB) for s in _SRCS):
        cxx = os.environ.get("CXX", "g++")
        subprocess.check_call([cxx, *_FLAGS, "-o", _LIB, *_SRCS])


def lib():
    global _lib
    if _lib is None:
        build()
        L = C.CDLL(_LIB)
        vp, i32, i64, f32 = C.c_void_p, C.c_int32, C.c_int64, C.c_float
        L.oracle_ctc_log_add_exp.argtypes = [f32, f32]
        L.oracle_ctc_log_add_exp.restype = f32
        L.oracle_ctc_greedy.argtypes = [vp, i32, i32, i32, vp]
        L.oracle_ctc_greedy.restype = i32
        lm = [i32, vp, vp, vp, vp, vp, i64, vp, vp, vp]
        L.oracle_ctc_lm_score.argtypes = lm + [C.c_char_p, i64, i32, C.c_char_p, i64]
        L.oracle_ctc_lm_score.restype = f32
        L.oracle_ctc_beam.argtypes = [vp, i32, i32, i32, vp, vp, i32] + lm + [i32, i32, f32, f32, vp, i64, C.POINTER(f32),
                                                                              C.POINTER(i64)]
        L.oracle_ctc_beam.restype = i64
        _lib = L
    return _lib


def _rows(log_probs):
    lp = np.ascontiguousarray(log_probs, np.float32)
    return lp if lp.ndim == 2 else np.zeros((0, 1), np.float32)


def blob(strings):
    """byte strings -> (bytes buffer, int64 offsets)"""
    data = [s if isinstance(s, bytes) else s.encode("utf-8") for s in strings]
    off = np.zeros(len(data) + 1, np.int64)
    off[1:] = np.cumsum([len(d) for d in data]) if data else []
    buf = np.frombuffer(b"".join(data) + b"\0", np.uint8).copy()
    return buf, off


class LmArrays:
    """An LM as fa_ctc_lm_create takes it: distinct words, unigram flags and values, bigrams by word index"""

    def __init__(self, unigrams, bigrams):
        """unigrams: {word: (log_prob, backoff)}; bigrams: {context: {word: log_prob}} (natural log, float32)"""
        words = list(unigrams)
        index = {w: i for i, w in enumerate(words)}
        for ctx, row in bigrams.items():
            for w in [ctx, *row]:
                if w not in index:
                    index[w] = len(words)
                    words.append(w)
        self.words = words
        self.buf, self.off = blob(words)
        self.has_uni = np.array([w in unigrams for w in words], np.int32)
        self.log_prob = np.array([unigrams[w][0] if w in unigrams else 0.0 for w in words], np.float32)
        self.backoff = np.array([unigrams[w][1] if w in unigrams else 0.0 for w in words], np.float32)
        pairs = [(index[c], index[w], p) for c, row in bigrams.items() for w, p in row.items()]
        self.ctx = np.array([p[0] for p in pairs], np.int32)
        self.word = np.array([p[1] for p in pairs], np.int32)
        self.bigram_lp = np.array([p[2] for p in pairs], np.float32)

    def args(self):
        return [len(self.words), self.buf.ctypes.data, self.off.ctypes.data, self.has_uni.ctypes.data,
                self.log_prob.ctypes.data, self.backoff.ctypes.data, len(self.ctx), self.ctx.ctypes.data,
                self.word.ctypes.data, self.bigram_lp.ctypes.data]


_NO_LM = None


def _no_lm_args():
    global _NO_LM
    if _NO_LM is None:
        _NO_LM = LmArrays({}, {})
    return _NO_LM.args()


def log_add_exp(a, b):
    return np.float32(lib().oracle_ctc_log_add_exp(a, b))


def greedy(log_probs, blank_id=DEFAULT_BLANK):
    """ctcGreedyDecode's ids"""
    lp = _rows(log_probs)
    out = np.zeros(max(1, lp.shape[0]), np.int32)
    n = lib().oracle_ctc_greedy(lp.ctypes.data, lp.shape[0], lp.shape[1], blank_id, out.ctypes.data) if lp.shape[0] else 0
    return [int(x) for x in out[:n]]


def lm_score(lm: LmArrays, word: str, prev=None):
    w = word.encode("utf-8")
    p = b"" if prev is None else prev.encode("utf-8")
    return np.float32(lib().oracle_ctc_lm_score(*lm.args(), w, len(w), int(prev is not None), p, len(p)))


def beam_search(log_probs, pieces, lm: LmArrays = None, beam_width=100, lm_weight=0.3, word_bonus=0.0,
                blank_id=DEFAULT_BLANK, token_candidates=40, stats=False):
    """ctcBeamSearch: (ids, total) of the best prefix; `pieces` lists token v's piece (None: not in the vocabulary).
    With stats, also the count of pruned prefixes re-created while a child of theirs was a beam."""
    lp = _rows(log_probs)
    T, V = lp.shape
    buf, off = blob([p or "" for p in pieces[:V]] + [""] * max(0, V - len(pieces)))
    out = np.zeros(max(1, T), np.int32)
    score, rec = C.c_float(), C.c_int64()
    lm_args = lm.args() if lm is not None else _no_lm_args()
    n = lib().oracle_ctc_beam(lp.ctypes.data, T, V, blank_id, buf.ctypes.data, off.ctypes.data, int(lm is not None),
                              *lm_args, beam_width, token_candidates, lm_weight, word_bonus, out.ctypes.data, out.size,
                              C.byref(score), C.byref(rec))
    res = ([int(x) for x in out[:n]], np.float32(score.value))
    return res + (rec.value,) if stats else res
