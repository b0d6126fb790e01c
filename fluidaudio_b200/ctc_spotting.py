"""CTC keyword spotting on the GPU (``fa_ctc_*``): CtcKeywordSpotter and CtcDPAlgorithm
(ASR/Parakeet/SlidingWindow/CustomVocabulary/WordSpotting/), the CTC-WS dynamic program behind custom-vocabulary
boosting, for every vocabulary term and clip in one launch.

``CtcKeywordSpotter.spot_keywords_from_log_probs`` is spotKeywordsFromLogProbs: it skips terms shorter than
``min_term_length`` characters, uses ``ctc_token_ids`` or else ``token_ids``, and reports detections in the reference's
order with times ``frame * frame_duration``.  One difference: Python's ``len`` counts code points where Swift's
``text.count`` counts grapheme clusters, so a term whose text combines characters (an accent written as a combining
mark, an emoji sequence) can be longer here than in Swift and pass a filter the reference would apply.

``apply_log_softmax``, ``merge_chunks`` and ``word_spot_constrained`` are applyLogSoftmax / makeLogProbs, the
concatenation of computeLogProbsChunked and ctcWordSpotConstrained; ``CtcSpotter`` holds a vocabulary in HBM and spots
it in many clips per call (``spot`` / ``spot_device``).  The CTC model and the tokenizers stay with the caller.
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass
from typing import List, Optional, Sequence

import numpy as np

from . import _lib

WILDCARD = -1          # ContextBiasingConstants.wildcardTokenId
DEFAULT_BLANK_ID = 1024
MAX_TERM_TOKENS = 127  # FA_CTC_MAX_TERM_TOKENS
CHUNK_OVERLAP_SAMPLES = 32_000
SAMPLE_RATE = 16_000


def _offsets(lengths) -> np.ndarray:
    off = np.zeros(len(lengths) + 1, np.int64)
    if len(lengths):
        off[1:] = np.cumsum(lengths)
    return off


def _tokens(lists) -> tuple:
    flat = np.ascontiguousarray(np.concatenate([np.asarray(t, np.int64) for t in lists]) if lists else [], np.int64)
    if flat.size and (flat.min() < -2 ** 31 or flat.max() >= 2 ** 31):
        raise ValueError("token ids must fit int32")
    return np.ascontiguousarray(flat.astype(np.int32)), _offsets([len(t) for t in lists])


def apply_log_softmax(logits, blank_id: int = DEFAULT_BLANK_ID, temperature: float = 1.0, blank_bias: float = 0.0,
                      vocab_major: bool = False) -> np.ndarray:
    """applyLogSoftmax: raw CTC logits [T x V] (or the rank-4 CoreML output as [V x T] with vocab_major) -> [T x V]"""
    x = np.ascontiguousarray(logits, np.float32)
    if x.ndim != 2:
        raise ValueError("logits must be 2-D")
    T, V = (x.shape[1], x.shape[0]) if vocab_major else x.shape
    out = np.empty((T, V), np.float32)
    _lib.check(_lib.load().fa_ctc_log_softmax(_lib.ptr(x), T, V, int(vocab_major), temperature, blank_bias, blank_id,
                                              _lib.ptr(out)), "fa_ctc_log_softmax")
    return out


def overlap_frames(frame_duration: float) -> int:
    """computeLogProbsChunked's overlap in frames: Int(32000 / 16000 / frameDuration)"""
    return int(CHUNK_OVERLAP_SAMPLES / SAMPLE_RATE / frame_duration)


def merge_chunks(chunks: Sequence[np.ndarray], frame_duration: Optional[float] = None,
                 overlap: Optional[int] = None) -> np.ndarray:
    """The per-chunk log-probs [rows x V] of a long clip joined as computeLogProbsChunked joins them, the overlap given
    in frames or derived from the frame duration"""
    if overlap is None:
        overlap = overlap_frames(frame_duration)
    chunks = [np.ascontiguousarray(c, np.float32) for c in chunks]
    V = next((c.shape[1] for c in chunks if c.ndim == 2 and c.shape[0]), 0)
    flat = np.ascontiguousarray(np.concatenate([c.reshape(-1, V) for c in chunks]) if V else np.zeros(0, np.float32))
    off = _offsets([c.shape[0] if c.ndim == 2 else 0 for c in chunks])
    rows = C.c_int32()
    out = np.empty((int(off[-1]), V), np.float32)
    _lib.check(_lib.load().fa_ctc_merge_chunks(_lib.ptr(flat), _lib.ptr(off), len(chunks), V, overlap, _lib.ptr(out),
                                               out.size, C.byref(rows)), "fa_ctc_merge_chunks")
    return out[:rows.value].copy()


def word_spot_constrained(log_probs, queries: Sequence[Sequence[int]], search_start, search_end,
                          blank_id: int = DEFAULT_BLANK_ID):
    """ctcWordSpotConstrained for many queries over one clip: (score [Q], start_frame [Q], end_frame [Q])"""
    lp = np.ascontiguousarray(log_probs, np.float32)
    tok, off = _tokens(list(queries))
    Q = len(queries)
    ss = np.ascontiguousarray(np.broadcast_to(np.asarray(search_start, np.int64), (Q,)))
    se = np.ascontiguousarray(np.broadcast_to(np.asarray(search_end, np.int64), (Q,)))
    score, start, end = np.empty(Q, np.float32), np.empty(Q, np.int64), np.empty(Q, np.int64)
    _lib.check(_lib.load().fa_ctc_spot_constrained(_lib.ptr(lp), lp.shape[0], lp.shape[1], blank_id, Q, _lib.ptr(tok),
                                                   _lib.ptr(off), _lib.ptr(ss), _lib.ptr(se), _lib.ptr(score),
                                                   _lib.ptr(start), _lib.ptr(end)), "fa_ctc_spot_constrained")
    return score, start, end


class CtcSpotter:
    """A vocabulary of token-id terms in HBM (fa_ctc_spotter): ctcWordSpotMultiple for every term in many clips."""

    def __init__(self, vocab_size: int, terms: Sequence[Sequence[int]], blank_id: int = DEFAULT_BLANK_ID):
        self.vocab_size, self.blank_id, self.term_count = int(vocab_size), int(blank_id), len(terms)
        tok, off = _tokens(list(terms))
        h = C.c_void_p()
        _lib.check(_lib.load().fa_ctc_spotter_create(self.vocab_size, self.blank_id, self.term_count, _lib.ptr(tok),
                                                     _lib.ptr(off), C.byref(h)), "fa_ctc_spotter_create")
        self._h = h

    def _call(self, fn, lp_ptr, row_offsets, min_score, det_ptr, capacity):
        B = len(row_offsets) - 1
        counts = np.zeros((B, self.term_count), np.int64)
        total = C.c_int64()
        ms = None if min_score is None else C.byref(C.c_float(min_score))
        st = fn(self._h, lp_ptr, _lib.ptr(row_offsets), B, ms, _lib.ptr(counts), C.byref(total), det_ptr, capacity)
        return st, counts, total.value

    def spot(self, clips: Sequence[np.ndarray], min_score: Optional[float] = None):
        """counts [B x K] and the detections (an array of CTC_DETECTION records: clip, term, merged order)"""
        clips = [np.ascontiguousarray(c, np.float32).reshape(-1, self.vocab_size) for c in clips]
        off = _offsets([len(c) for c in clips])
        lp = np.ascontiguousarray(np.concatenate(clips) if clips else np.zeros((0, self.vocab_size), np.float32))
        det = np.empty(max(1, int(off[-1]) // 8), _lib.CTC_DETECTION)
        L = _lib.load()
        st, counts, total = self._call(L.fa_ctc_spot, _lib.ptr(lp), off, min_score, _lib.ptr(det), len(det))
        if st == 3:   # more detections than the first guess: the counts give the size
            det = np.empty(total, _lib.CTC_DETECTION)
            st, counts, total = self._call(L.fa_ctc_spot, _lib.ptr(lp), off, min_score, _lib.ptr(det), len(det))
        _lib.check(st, "fa_ctc_spot")
        return counts, det[:total].copy()

    def spot_device(self, d_log_probs: "_lib.DeviceBuffer", row_offsets, d_detections: "_lib.DeviceBuffer",
                    capacity: int, min_score: Optional[float] = None):
        """fa_ctc_spot_device: log-probs and detections in HBM; returns (status, counts, total) with the status of
        FA_STATUS_OUTPUT_TOO_SMALL passed through, every other failure raised"""
        off = np.ascontiguousarray(row_offsets, np.int64)
        st, counts, total = self._call(_lib.load().fa_ctc_spot_device, d_log_probs.ptr, off, min_score,
                                       d_detections.ptr, capacity)
        if st not in (0, 3):
            _lib.check(st, "fa_ctc_spot_device")
        return st, counts, total

    def close(self):
        if getattr(self, "_h", None):
            _lib.load().fa_ctc_spotter_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


@dataclass
class CustomVocabularyTerm:
    """The fields of CustomVocabularyTerm the spotter reads"""
    text: str
    token_ids: Optional[List[int]] = None
    ctc_token_ids: Optional[List[int]] = None


@dataclass
class KeywordDetection:
    term: CustomVocabularyTerm
    score: float
    total_frames: int
    start_frame: int
    end_frame: int
    start_time: float
    end_time: float


class CtcKeywordSpotter:
    """spotKeywordsFromLogProbs over log-probs the caller's CTC model produced."""

    def __init__(self, blank_id: int = DEFAULT_BLANK_ID):
        self.blank_id = blank_id

    @staticmethod
    def _terms(vocabulary, min_term_length):
        kept = []
        for term in vocabulary:
            if len(term.text) < min_term_length:   # code points; Swift counts graphemes (module docstring)
                continue
            ids = term.ctc_token_ids if term.ctc_token_ids is not None else term.token_ids
            if ids:
                kept.append((term, list(ids)))
        return kept

    def spot_keywords_from_log_probs(self, log_probs, frame_duration: float, vocabulary: Sequence[CustomVocabularyTerm],
                                     min_score: Optional[float] = None, min_term_length: int = 3):
        return self.spot_keywords_batch([log_probs], frame_duration, vocabulary, min_score, min_term_length)[0]

    def spot_keywords_batch(self, clips, frame_duration: float, vocabulary: Sequence[CustomVocabularyTerm],
                            min_score: Optional[float] = None, min_term_length: int = 3) -> List[List[KeywordDetection]]:
        """spot_keywords_from_log_probs for many clips of one vocabulary in one call: a list per clip"""
        clips = [np.ascontiguousarray(c, np.float32) for c in clips]
        kept = self._terms(vocabulary, min_term_length)
        out: List[List[KeywordDetection]] = [[] for _ in clips]
        live = [c for c in clips if c.ndim == 2 and c.shape[0] > 0]
        if not kept or not live:
            return out
        V = live[0].shape[1]
        spotter = CtcSpotter(V, [ids for _, ids in kept], self.blank_id)
        try:
            counts, det = spotter.spot([c.reshape(-1, V) if c.size else np.zeros((0, V), np.float32) for c in clips],
                                       min_score)
        finally:
            spotter.close()
        for d in det:
            T = clips[d["clip"]].shape[0]
            out[d["clip"]].append(KeywordDetection(kept[d["term"]][0], float(d["score"]), T, int(d["start_frame"]),
                                                   int(d["end_frame"]), float(d["start_frame"]) * frame_duration,
                                                   float(d["end_frame"]) * frame_duration))
        return out
