"""StyleTTS2 synthesis glue on the GPU (``include/fluidaudio_b200_styletts2.h``): everything
StyleTTS2Synthesizer.synthesize (Sources/FluidAudio/TTS/StyleTTS2/) does on the host between its eight models, for
many requests per launch.  The models stay with the caller.

* ``plan``: the bert / sampler bucket of a token count (57, 64, 128, 256) or the reason it has none.
* ``StyleTTS2Glue``: ``sampler_inputs`` (bert's padded tokens and mask, the sampler's seeded noise), ``blend_style``
  and ``align`` (durations, then the duration-aligned ``en`` and ``asr``), each with host arrays or, in the
  ``*_device`` form, raw HBM pointers.
* ``StyleTTS2Synthesizer.synthesize_batch``: the whole pipeline over caller-supplied model callables, requests grouped
  by bucket, with the tail trim and, optionally, chunks concatenated per utterance.
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass
from typing import Callable, List, Optional, Sequence

import numpy as np

from . import _lib

STYLE_DIM = 256          # FA_STYLETTS2_STYLE_DIM
REF_SPLIT = 128          # FA_STYLETTS2_REF_SPLIT
NOISE_ROWS = 5           # FA_STYLETTS2_NOISE_ROWS
BUCKETS = (57, 64, 128, 256)
MAX_TOKENS = 256
TAIL_TRIM = 50           # FA_STYLETTS2_TAIL_TRIM
SAMPLE_RATE = 24000
DEFAULT_ALPHA, DEFAULT_BETA = 0.3, 0.7
STATUS_OUTPUT_TOO_SMALL = 3
REASONS = ("ok", "no tokens", "more tokens than the largest bucket (256)", "a NaN duration logit")


class StyleTTS2Error(ValueError):
    """A request refused with one of the reason codes (``REASONS``)."""

    def __init__(self, reason: int, request: int = 0):
        super().__init__(f"request {request}: {REASONS[reason]}")
        self.reason, self.request = reason, request


def plan(token_count: int):
    """fa_styletts2_plan: (bucket, reason); bucket is 0 when reason is not 0"""
    b, r = C.c_int32(), C.c_int32()
    _lib.check(_lib.load().fa_styletts2_plan(int(token_count), C.byref(b), C.byref(r)), "fa_styletts2_plan")
    return int(b.value), int(r.value)


def tail_trim(audio) -> np.ndarray:
    """synthesize's last step: all but the last 50 samples (none of 50 or fewer)"""
    a = np.asarray(audio, np.float32).reshape(-1)
    return a[:max(a.size - TAIL_TRIM, 0)]


def _offsets(sizes):
    return np.concatenate([[0], np.cumsum(sizes, dtype=np.int64)]).astype(np.int64)


def _raise_reasons(st, reasons, where):
    if st != 0 and st != STATUS_OUTPUT_TOO_SMALL and reasons.any():
        i = int(np.flatnonzero(reasons)[0])
        err = StyleTTS2Error(int(reasons[i]), i)
        err.reasons = reasons
        raise err
    _lib.check(st, where)


class StyleTTS2Glue:
    """The fa_styletts2_* calls on the current device"""

    def __init__(self):
        self._L = _lib.load()

    # ------------------------------------------------------------------ sampler inputs
    def sampler_inputs(self, token_ids: Sequence[Sequence[int]], seeds, bucket: int):
        """(tokens [n x bucket] int32, attention_mask [n x bucket] int32, noise [n x 5 x 256]); row 0 of a request's
        noise is noise_init, rows 1 .. 4 are noises_aux"""
        n = len(token_ids)
        ids = np.concatenate([np.asarray(t, np.int32).reshape(-1) for t in token_ids]) if n else np.zeros(0, np.int32)
        off = _offsets([len(t) for t in token_ids])
        sd = np.ascontiguousarray(np.broadcast_to(np.asarray(seeds, np.uint64), (n,)))
        tokens, mask = np.empty((n, int(bucket)), np.int32), np.empty((n, int(bucket)), np.int32)
        noise, reasons = np.empty((n, NOISE_ROWS, STYLE_DIM), np.float32), np.zeros(n, np.int32)
        st = self._L.fa_styletts2_sampler_inputs(n, _lib.ptr(ids), _lib.ptr(off), _lib.ptr(sd), int(bucket),
                                                 _lib.ptr(tokens), _lib.ptr(mask), _lib.ptr(noise), _lib.ptr(reasons))
        _raise_reasons(st, reasons, "fa_styletts2_sampler_inputs")
        return tokens, mask, noise

    def sampler_inputs_device(self, count, d_token_ids, offsets, seeds, bucket, d_tokens, d_mask, d_noise):
        """the device form: HBM pointers for the ids and the outputs, host offsets [count + 1] and seeds; returns
        the reasons"""
        off, sd = np.ascontiguousarray(offsets, np.int64), np.ascontiguousarray(seeds, np.uint64)
        reasons = np.zeros(int(count), np.int32)
        st = self._L.fa_styletts2_sampler_inputs_device(int(count), d_token_ids, _lib.ptr(off), _lib.ptr(sd),
                                                        int(bucket), d_tokens, d_mask, d_noise, _lib.ptr(reasons))
        _raise_reasons(st, reasons, "fa_styletts2_sampler_inputs_device")
        return reasons

    # ------------------------------------------------------------------ style
    def blend_style(self, s_pred, ref_s, alphas, betas):
        """(ref [n x 128], s [n x 128]) from s_pred and ref_s [n x 256] and per-request alpha and beta"""
        p = np.ascontiguousarray(s_pred, np.float32).reshape(-1, STYLE_DIM)
        r = np.ascontiguousarray(ref_s, np.float32).reshape(-1, STYLE_DIM)
        n = p.shape[0]
        a = np.ascontiguousarray(np.broadcast_to(np.asarray(alphas, np.float32), (n,)))
        b = np.ascontiguousarray(np.broadcast_to(np.asarray(betas, np.float32), (n,)))
        ref, s = np.empty((n, REF_SPLIT), np.float32), np.empty((n, REF_SPLIT), np.float32)
        _lib.check(self._L.fa_styletts2_style(n, _lib.ptr(p), _lib.ptr(r), _lib.ptr(a), _lib.ptr(b), _lib.ptr(ref),
                                              _lib.ptr(s)), "fa_styletts2_style")
        return ref, s

    def blend_style_device(self, count, d_s_pred, d_ref_s, alphas, betas, d_ref, d_s):
        a, b = np.ascontiguousarray(alphas, np.float32), np.ascontiguousarray(betas, np.float32)
        _lib.check(self._L.fa_styletts2_style_device(int(count), d_s_pred, d_ref_s, _lib.ptr(a), _lib.ptr(b), d_ref,
                                                     d_s), "fa_styletts2_style_device")

    # ------------------------------------------------------------------ align
    def align(self, logits: Sequence[np.ndarray], d: Sequence[np.ndarray], t_en: Sequence[np.ndarray],
              frame_stride: Optional[int] = None):
        """(en [n x dC x stride], asr [n x tC x stride], frames [n], durations: a list of int32 arrays) from each
        request's logits [n_i x C], d [n_i x dC] and t_en [tC x n_i]; en and asr are zero from frame F on.  Without a
        frame_stride the call is repeated with the largest F when a first guess is too small."""
        count = len(logits)
        counts = np.array([np.shape(x)[0] for x in logits], np.int32)
        width = int(counts.max()) if count else 1
        C_ = np.shape(logits[0])[1] if count else 1
        dC = np.shape(d[0])[1] if count else 1
        tC = np.shape(t_en[0])[0] if count else 1
        L_ = np.zeros((count, width, C_), np.float32)
        D_ = np.zeros((count, width, dC), np.float32)
        T_ = np.zeros((count, tC, width), np.float32)
        for i in range(count):
            k = counts[i]
            L_[i, :k], D_[i, :k], T_[i, :, :k] = logits[i], d[i], t_en[i]
        stride = int(frame_stride) if frame_stride else max(1, width * min(C_, 8))
        while True:
            en = np.empty((count, dC, stride), np.float32)
            asr = np.empty((count, tC, stride), np.float32)
            frames, durations = np.zeros(count, np.int64), np.zeros(max(int(counts.sum()), 1), np.int32)
            reasons = np.zeros(count, np.int32)
            st = self._L.fa_styletts2_align(count, _lib.ptr(counts), _lib.ptr(L_), C_, C_, width * C_, _lib.ptr(D_), dC,
                                            dC, width * dC, _lib.ptr(T_), tC, width, tC * width, stride,
                                            _lib.ptr(en), _lib.ptr(asr), _lib.ptr(frames), _lib.ptr(durations),
                                            _lib.ptr(reasons))
            if st == STATUS_OUTPUT_TOO_SMALL and frame_stride is None:
                stride = int(frames.max())
                continue
            _raise_reasons(st, reasons, "fa_styletts2_align")
            at = _offsets(counts)
            return en, asr, frames, [durations[at[i]:at[i + 1]].copy() for i in range(count)]

    def align_device(self, token_counts, d_logits, logit_channels, logit_row_stride, logit_request_stride, d_d,
                     d_channels, d_row_stride, d_request_stride, d_t_en, t_en_channels, t_en_row_stride,
                     t_en_request_stride, frame_stride, d_en, d_asr):
        """the device form over HBM pointers with explicit strides; returns (status, frames, durations, reasons)
        with the status of fa_styletts2_align_device (0 or FA_STATUS_OUTPUT_TOO_SMALL; other refusals raise)"""
        counts = np.ascontiguousarray(token_counts, np.int32)
        n = counts.size
        frames, reasons = np.zeros(n, np.int64), np.zeros(n, np.int32)
        durations = np.zeros(max(int(counts.sum()), 1), np.int32)
        st = self._L.fa_styletts2_align_device(n, _lib.ptr(counts), d_logits, int(logit_channels),
                                               int(logit_row_stride), int(logit_request_stride), d_d, int(d_channels),
                                               int(d_row_stride), int(d_request_stride), d_t_en, int(t_en_channels),
                                               int(t_en_row_stride), int(t_en_request_stride), int(frame_stride),
                                               d_en, d_asr, _lib.ptr(frames), _lib.ptr(durations), _lib.ptr(reasons))
        if st != STATUS_OUTPUT_TOO_SMALL:
            _raise_reasons(st, reasons, "fa_styletts2_align_device")
        return st, frames, durations[:int(counts.sum())], reasons


@dataclass
class StyleTTS2SynthesisResult:
    samples: np.ndarray
    sample_rate: int
    frames: int            # F, the sum of the request's durations (for an utterance: the sum over its chunks)
    durations: np.ndarray  # per token (for an utterance: its chunks' in order)


class StyleTTS2Synthesizer:
    """StyleTTS2Synthesizer.synthesize for many requests per call, over model callables in the shapes synthesize
    feeds (numpy in, numpy out).  bert and the fused sampler take a batch of one bucket's requests; the models whose
    token or frame axis varies per request take one request:
      text_encoder(tokens [1 x n] int32, input_lengths [1] int32, text_mask [1 x n]) -> t_en [1 x tC x n]
      bert(tokens [k x T] int32, attention_mask [k x T] int32) -> (bert_dur [k x T x 768], d_en [k x dC' x T])
      ref_encoder(mel [1 x 1 x 80 x frames]) -> ref_s [1 x 256]
      sampler(noise_init [k x 1 x 256], noises_aux [k x 4 x 1 x 1 x 256], embedding [k x T x 768], features [k x 256])
        -> s_pred [k x 1 x 256]
      duration_predictor(d_en [1 x dC' x n], s [1 x 128], text_mask [1 x n]) -> (d [1 x n x dC], logits [1 x n x C])
      f0n_har(en [1 x dC x F], s [1 x 128]) -> (f0, n, har)
      decoder_pre(asr [1 x tC x F], f0, n, ref [1 x 128]) -> x_pre
      decoder_upsample(x_pre, ref [1 x 128], har) -> audio [1 x samples]"""

    def __init__(self, text_encoder: Callable, bert: Callable, ref_encoder: Callable, sampler: Callable,
                 duration_predictor: Callable, f0n_har: Callable, decoder_pre: Callable, decoder_upsample: Callable):
        self.text_encoder, self.bert, self.ref_encoder, self.sampler = text_encoder, bert, ref_encoder, sampler
        self.duration_predictor, self.f0n_har = duration_predictor, f0n_har
        self.decoder_pre, self.decoder_upsample = decoder_pre, decoder_upsample
        self.glue = StyleTTS2Glue()

    def synthesize_batch(self, token_ids: Sequence[Sequence[int]], reference_mels: Sequence[np.ndarray], seeds=0,
                         alphas=DEFAULT_ALPHA, betas=DEFAULT_BETA, references: Optional[Sequence[int]] = None,
                         utterances: Optional[Sequence[int]] = None) -> List[StyleTTS2SynthesisResult]:
        """Request i speaks token_ids[i] in the style of reference_mels[references[i]] (default: reference i), each
        mel [80 x frames] run through the ref encoder once.  With ``utterances``, request i is a chunk of utterance
        utterances[i] (0, 1, ...): chunks are concatenated in request order and one result per utterance returned, as
        the chunked text path does."""
        n = len(token_ids)
        refs = list(range(n)) if references is None else [int(r) for r in references]
        seeds = np.broadcast_to(np.asarray(seeds, np.uint64), (n,))
        alphas = np.broadcast_to(np.asarray(alphas, np.float32), (n,))
        betas = np.broadcast_to(np.asarray(betas, np.float32), (n,))
        buckets = []
        for i, t in enumerate(token_ids):
            b, r = plan(len(t))
            if r:
                raise StyleTTS2Error(r, i)
            buckets.append(b)
        t_en = [np.asarray(self.text_encoder(np.asarray(t, np.int32)[None], np.array([len(t)], np.int32),
                                             np.zeros((1, len(t)), np.float32)), np.float32)[0] for t in token_ids]
        ref_s = {r: np.asarray(self.ref_encoder(np.asarray(reference_mels[r], np.float32)[None, None]),
                               np.float32).reshape(STYLE_DIM) for r in sorted(set(refs))}
        ref_rows = np.stack([ref_s[r] for r in refs]) if n else np.zeros((0, STYLE_DIM), np.float32)
        s_pred, d_en = np.zeros((n, STYLE_DIM), np.float32), [None] * n
        for bucket in BUCKETS:
            sel = [i for i in range(n) if buckets[i] == bucket]
            if not sel:
                continue
            tokens, mask, noise = self.glue.sampler_inputs([token_ids[i] for i in sel], seeds[sel], bucket)
            bert_dur, d_en_padded = self.bert(tokens, mask)
            out = self.sampler(noise[:, :1, :], noise[:, 1:, None, None, :], np.asarray(bert_dur, np.float32),
                               ref_rows[sel])
            s_pred[sel] = np.asarray(out, np.float32).reshape(len(sel), STYLE_DIM)
            for j, i in enumerate(sel):
                d_en[i] = np.asarray(d_en_padded, np.float32)[j:j + 1, :, :len(token_ids[i])]
        ref128, s128 = self.glue.blend_style(s_pred, ref_rows, alphas, betas)
        outs = [self.duration_predictor(d_en[i], s128[i:i + 1], np.zeros((1, len(token_ids[i])), np.float32))
                for i in range(n)]
        en, asr, frames, durations = self.glue.align([np.asarray(lg, np.float32)[0] for _, lg in outs],
                                                     [np.asarray(d, np.float32)[0] for d, _ in outs], t_en)
        samples = []
        for i in range(n):
            F = int(frames[i])
            f0, nn, har = self.f0n_har(en[i:i + 1, :, :F], s128[i:i + 1])
            x_pre = self.decoder_pre(asr[i:i + 1, :, :F], f0, nn, ref128[i:i + 1])
            samples.append(tail_trim(self.decoder_upsample(x_pre, ref128[i:i + 1], har)))
        if utterances is None:
            return [StyleTTS2SynthesisResult(samples[i], SAMPLE_RATE, int(frames[i]), durations[i]) for i in range(n)]
        groups = {}
        for i, u in enumerate(utterances):
            groups.setdefault(int(u), []).append(i)
        return [StyleTTS2SynthesisResult(np.concatenate([samples[i] for i in groups[u]]), SAMPLE_RATE,
                                         int(sum(int(frames[i]) for i in groups[u])),
                                         np.concatenate([durations[i] for i in groups[u]]))
                for u in sorted(groups)]
