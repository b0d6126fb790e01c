"""CTC decoding on the GPU (``fa_ctc_greedy``, ``fa_ctc_beam_search``): ctcGreedyDecode, ctcBeamSearch and
ARPALanguageModel (ASR/Parakeet/SlidingWindow/CTC/), for many clips per call.

``ctc_greedy_decode`` and ``ctc_beam_search`` take one clip's ``[T x V]`` log-probs and a ``{id: piece}`` vocabulary and
return text, with the reference's signatures and defaults; ``CtcDecoder`` holds a vocabulary in HBM and decodes batches
(``greedy``, ``beam_search``, ``beam_search_device``), returning ids, scores and texts.  ``decode_ctc_token_ids`` turns
ids into text on the host.  ``ARPALanguageModel.load`` reads a plain-text ARPA file as the reference reads it.  A search
given an ``ARPALanguageModel`` uploads it for that call; ``to_device()`` makes a ``CtcLanguageModel`` snapshot in HBM
for many searches on the current device.

Ties the reference breaks by its dictionaries' hash order are broken by first insertion (see
``include/fluidaudio_b200_ctc_decode.h``).  Two documented differences: words compare by their UTF-8 bytes, where Swift
treats canonically equivalent strings as equal; and the word-boundary test and ``dropFirst`` act on code points, where
Swift acts on grapheme clusters (this matters only for a ``▁`` followed by a combining mark).
"""
from __future__ import annotations

import ctypes as C
import math
import unicodedata
from dataclasses import dataclass
from typing import Dict, List, Optional, Sequence, Union

import numpy as np

from . import _lib

DEFAULT_BLANK_ID = 1024
WORD_BOUNDARY = "▁"        # ASRConstants.sentencePieceWordBoundary
MAX_BEAM_WIDTH = 128            # FA_CTC_DECODE_MAX_BEAM_WIDTH
MAX_TOKEN_CANDIDATES = 64       # FA_CTC_DECODE_MAX_TOKEN_CANDIDATES
STATUS_OK = 0                   # FA_STATUS_OK
STATUS_OUTPUT_TOO_SMALL = 3     # FA_STATUS_OUTPUT_TOO_SMALL


def _offsets(lengths) -> np.ndarray:
    off = np.zeros(len(lengths) + 1, np.int64)
    if len(lengths):
        off[1:] = np.cumsum(lengths)
    return off


def _blob(strings):
    data = [s.encode("utf-8") for s in strings]
    return np.frombuffer(b"".join(data) + b"\0", np.uint8).copy(), _offsets([len(d) for d in data])


def _is_whitespace(c: str) -> bool:
    """CharacterSet.whitespaces: Unicode Zs and tab (newlines are not in it)"""
    return c == "\t" or unicodedata.category(c) == "Zs"


def decode_ctc_token_ids(ids: Sequence[int], vocabulary: Dict[int, str]) -> str:
    """decodeCtcTokenIds: the known ids' pieces joined, U+2581 as a space, whitespace (not newlines) trimmed"""
    text = "".join(vocabulary[int(i)] for i in ids if int(i) in vocabulary).replace(WORD_BOUNDARY, " ")
    a, b = 0, len(text)
    while a < b and _is_whitespace(text[a]):
        a += 1
    while b > a and _is_whitespace(text[b - 1]):
        b -= 1
    return text[a:b]


# ---- ARPA ----------------------------------------------------------------------------------------------------------
_libc = C.CDLL(None)
_libc.strtof.argtypes = [C.c_char_p, C.POINTER(C.c_char_p)]
_libc.strtof.restype = C.c_float


def swift_float(text: str) -> Optional[np.float32]:
    """Float(String): no leading whitespace, not empty, then strtof in the C locale consuming every byte up to the first
    NUL (Swift hands the string to strtof as a C string); None otherwise"""
    raw = text.encode("utf-8").split(b"\0", 1)[0]
    if not raw or raw[:1] in (b"\t", b"\n", b"\v", b"\f", b"\r", b" "):
        return None
    buf = C.create_string_buffer(raw)
    end = C.c_char_p()
    value = _libc.strtof(buf, C.byref(end))
    if C.cast(end, C.c_void_p).value != C.addressof(buf) + len(raw):
        return None
    return np.float32(value)


_NEWLINES = "\n\u000b\u000c\r\u0085\u2028\u2029"


def _trim(line: str) -> str:
    """trimmingCharacters(in: .whitespacesAndNewlines)"""
    a, b = 0, len(line)
    while a < b and (_is_whitespace(line[a]) or line[a] in _NEWLINES):
        a += 1
    while b > a and (_is_whitespace(line[b - 1]) or line[b - 1] in _NEWLINES):
        b -= 1
    return line[a:b]


def _backoff(field: str) -> np.float32:
    """(Float(field) ?? 0.0) * log10ToNat"""
    x = swift_float(field)
    return np.float32((np.float32(0.0) if x is None else x) * ARPALanguageModel.LOG10_TO_NAT)


class ARPALanguageModel:
    """ARPALanguageModel: unigrams and bigrams in natural log (float32), scored with backoff."""

    @dataclass(frozen=True)
    class Entry:
        log_prob: np.float32
        backoff: np.float32

    LOG10_TO_NAT = np.float32(math.log(10.0))
    UNK_LOG_PROB = np.float32(-23.026)

    def __init__(self):
        self.unigrams: Dict[str, ARPALanguageModel.Entry] = {}
        self.bigrams: Dict[str, Dict[str, ARPALanguageModel.Entry]] = {}

    @classmethod
    def load(cls, path) -> "ARPALanguageModel":
        """ARPALanguageModel.load(from:), line for line: lines split on \\n, a line that is not UTF-8 ends the read,
        fields split on tabs (so a KenLM-style "p<TAB>w1 w2<TAB>b" bigram has context "w1 w2" and word "b", as in the
        reference), later duplicates overwrite earlier ones.  OSError when the file cannot be opened."""
        with open(path, "rb") as f:
            data = f.read()
        lines = data.split(b"\n")
        if lines and lines[-1] == b"":
            lines.pop()
        lm, section = cls(), ""
        for raw in lines:
            try:
                line = _trim(raw.decode("utf-8"))
            except UnicodeDecodeError:
                break
            if not line or line.startswith("\\data\\"):
                continue
            if line == "\\end\\":
                break
            if line.startswith("\\"):
                section = line
                continue
            if line.startswith("ngram "):
                continue
            parts = line.split("\t")
            log10 = swift_float(parts[0])
            if log10 is None:
                continue
            prob = np.float32(log10 * cls.LOG10_TO_NAT)
            if section == "\\1-grams:" and len(parts) >= 2:
                bo = _backoff(parts[2]) if len(parts) >= 3 else np.float32(0.0)
                lm.unigrams[parts[1]] = cls.Entry(prob, bo)
            elif section == "\\2-grams:" and len(parts) >= 3:
                bo = _backoff(parts[3]) if len(parts) >= 4 else np.float32(0.0)
                lm.bigrams.setdefault(parts[1], {})[parts[2]] = cls.Entry(prob, bo)
        return lm

    def score(self, word: str, prev: Optional[str]) -> np.float32:
        """score(word:prev:): the bigram when present, else backoff(prev) + logProb(word) (unkLogProb when unknown)"""
        if prev is not None and word in self.bigrams.get(prev, {}):
            return self.bigrams[prev][word].log_prob
        backoff = self.unigrams[prev].backoff if prev is not None and prev in self.unigrams else np.float32(0.0)
        lp = self.unigrams[word].log_prob if word in self.unigrams else self.UNK_LOG_PROB
        return np.float32(backoff + lp)

    def to_device(self) -> "CtcLanguageModel":
        """a snapshot of the model in HBM on the current device, for many searches: later edits to the dictionaries do
        not reach it"""
        return CtcLanguageModel(self)


class CtcLanguageModel:
    """An ARPALanguageModel uploaded to the current device (fa_ctc_lm): read-only, shared by decoders on that device."""

    def __init__(self, model: ARPALanguageModel):
        words = list(model.unigrams)
        index = {w: i for i, w in enumerate(words)}
        for ctx, row in model.bigrams.items():
            for w in [ctx, *row]:
                if w not in index:
                    index[w] = len(words)
                    words.append(w)
        buf, off = _blob(words)
        uni = model.unigrams
        has = np.array([w in uni for w in words], np.int32)
        lp = np.array([uni[w].log_prob if w in uni else 0.0 for w in words], np.float32)
        bo = np.array([uni[w].backoff if w in uni else 0.0 for w in words], np.float32)
        pairs = [(index[c], index[w], e.log_prob) for c, row in model.bigrams.items() for w, e in row.items()]
        ctx = np.array([p[0] for p in pairs], np.int32)
        wid = np.array([p[1] for p in pairs], np.int32)
        blp = np.array([p[2] for p in pairs], np.float32)
        h = C.c_void_p()
        _lib.check(_lib.load().fa_ctc_lm_create(len(words), _lib.ptr(buf), _lib.ptr(off), _lib.ptr(has), _lib.ptr(lp),
                                                _lib.ptr(bo), len(pairs), _lib.ptr(ctx), _lib.ptr(wid), _lib.ptr(blp),
                                                C.byref(h)), "fa_ctc_lm_create")
        self._h = h

    def close(self):
        if getattr(self, "_h", None):
            _lib.load().fa_ctc_lm_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


LanguageModel = Union[ARPALanguageModel, CtcLanguageModel]


# ---- decoding ------------------------------------------------------------------------------------------------------
def _clips(clips, V):
    clips = [np.ascontiguousarray(c, np.float32).reshape(-1, V) for c in clips]
    off = _offsets([len(c) for c in clips])
    lp = np.ascontiguousarray(np.concatenate(clips) if clips else np.zeros((0, V), np.float32))
    return lp, off


def _split(tokens, lengths):
    out, at = [], 0
    for n in lengths:
        out.append([int(x) for x in tokens[at:at + int(n)]])
        at += int(n)
    return out


def greedy_ids(clips: Sequence[np.ndarray], vocab_size: int, blank_id: int = DEFAULT_BLANK_ID) -> List[List[int]]:
    """ctcGreedyDecode's ids for every clip ([T x vocab_size] each), in one call"""
    lp, off = _clips(clips, vocab_size)
    B = len(off) - 1
    lengths, total = np.zeros(max(B, 1), np.int64), C.c_int64()
    tokens = np.zeros(max(1, int(off[-1])), np.int32)
    _lib.check(_lib.load().fa_ctc_greedy(_lib.ptr(lp), _lib.ptr(off), B, vocab_size, blank_id, _lib.ptr(lengths),
                                         _lib.ptr(tokens), tokens.size, C.byref(total)), "fa_ctc_greedy")
    return _split(tokens, lengths[:B])


def ctc_greedy_decode(log_probs, vocabulary: Dict[int, str], blank_id: int = DEFAULT_BLANK_ID) -> str:
    """ctcGreedyDecode(logProbs: [[Float]]): argmax per frame, repeats collapsed, blanks removed, as text"""
    lp = np.asarray(log_probs, np.float32)
    if lp.ndim != 2 or lp.shape[0] == 0 or lp.shape[1] == 0:
        return ""
    return decode_ctc_token_ids(greedy_ids([lp], lp.shape[1], blank_id)[0], vocabulary)


class CtcDecoder:
    """A vocabulary's pieces in HBM (fa_ctc_decoder): greedy decoding and prefix beam search for many clips per call."""

    def __init__(self, vocabulary: Dict[int, str], vocab_size: int, blank_id: int = DEFAULT_BLANK_ID):
        self.vocabulary, self.vocab_size, self.blank_id = dict(vocabulary), int(vocab_size), int(blank_id)
        buf, off = _blob([self.vocabulary.get(v, "") for v in range(self.vocab_size)])
        h = C.c_void_p()
        _lib.check(_lib.load().fa_ctc_decoder_create(self.vocab_size, self.blank_id, _lib.ptr(buf), _lib.ptr(off),
                                                     C.byref(h)), "fa_ctc_decoder_create")
        self._h = h

    @staticmethod
    def config(beam_width=100, token_candidates=40, lm_weight=0.3, word_bonus=0.0) -> "_lib.CtcBeamConfig":
        return _lib.CtcBeamConfig(beam_width, token_candidates, lm_weight, word_bonus)

    def greedy(self, clips: Sequence[np.ndarray]):
        """(ids per clip, text per clip)"""
        ids = greedy_ids(clips, self.vocab_size, self.blank_id)
        return ids, [decode_ctc_token_ids(i, self.vocabulary) for i in ids]

    def _search(self, fn, lp_ptr, off, lm, cfg, tok_ptr, capacity):
        B = len(off) - 1
        lengths, scores, total = np.zeros(max(B, 1), np.int64), np.zeros(max(B, 1), np.float32), C.c_int64()
        # an ARPALanguageModel is uploaded for this call alone, so the search always sees its current dictionaries
        dev_lm = lm.to_device() if isinstance(lm, ARPALanguageModel) else lm
        try:
            st = fn(self._h, dev_lm._h if dev_lm is not None else None, lp_ptr, _lib.ptr(off), B, C.byref(cfg),
                    _lib.ptr(lengths), _lib.ptr(scores), tok_ptr, capacity, C.byref(total))
        finally:
            if dev_lm is not lm:
                dev_lm.close()
        return st, lengths[:B], scores[:B], total.value

    def beam_search(self, clips: Sequence[np.ndarray], lm: Optional[LanguageModel] = None, beam_width=100,
                    lm_weight=0.3, word_bonus=0.0, token_candidates=40):
        """(ids per clip, best total per clip, text per clip)"""
        lp, off = _clips(clips, self.vocab_size)
        cfg = self.config(beam_width, token_candidates, lm_weight, word_bonus)
        tokens = np.zeros(max(1, int(off[-1])), np.int32)
        st, lengths, scores, _ = self._search(_lib.load().fa_ctc_beam_search, _lib.ptr(lp), off, lm, cfg,
                                              _lib.ptr(tokens), tokens.size)
        _lib.check(st, "fa_ctc_beam_search")
        ids = _split(tokens, lengths)
        return ids, scores, [decode_ctc_token_ids(i, self.vocabulary) for i in ids]

    def beam_search_device(self, d_log_probs: "_lib.DeviceBuffer", row_offsets, d_tokens: "_lib.DeviceBuffer",
                           capacity: int, lm: Optional[LanguageModel] = None, beam_width=100, lm_weight=0.3,
                           word_bonus=0.0, token_candidates=40):
        """fa_ctc_beam_search_device: (status, lengths, scores, total) with FA_STATUS_OUTPUT_TOO_SMALL passed through,
        every other failure raised"""
        off = np.ascontiguousarray(row_offsets, np.int64)
        cfg = self.config(beam_width, token_candidates, lm_weight, word_bonus)
        st, lengths, scores, total = self._search(_lib.load().fa_ctc_beam_search_device, d_log_probs.ptr, off, lm, cfg,
                                                  d_tokens.ptr, capacity)
        if st not in (STATUS_OK, STATUS_OUTPUT_TOO_SMALL):
            _lib.check(st, "fa_ctc_beam_search_device")
        return st, lengths, scores, total

    def close(self):
        if getattr(self, "_h", None):
            _lib.load().fa_ctc_decoder_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def ctc_beam_search(log_probs, vocabulary: Dict[int, str], lm: Optional[LanguageModel] = None,
                    beam_width: int = 100, lm_weight: float = 0.3, word_bonus: float = 0.0,
                    blank_id: int = DEFAULT_BLANK_ID, token_candidates: int = 40) -> str:
    """ctcBeamSearch(logProbs: [[Float]]): prefix beam search with optional ARPA LM rescoring, as text"""
    lp = np.asarray(log_probs, np.float32)
    if lp.ndim != 2 or lp.shape[0] == 0 or lp.shape[1] == 0:
        return ""
    dec = CtcDecoder(vocabulary, lp.shape[1], blank_id)
    try:
        return dec.beam_search([lp], lm, beam_width, lm_weight, word_bonus, token_candidates)[2][0]
    finally:
        dec.close()
