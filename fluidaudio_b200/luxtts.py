"""LuxTTS synthesis on the GPU (``include/fluidaudio_b200_luxtts.h``): everything LuxTtsSynthesizer.synthesize
(Sources/FluidAudio/TTS/LuxTts/) does on the host between its models, for many requests per launch.  The text
encoder, the FmDecoder and the vocoder stay with the caller.

* ``LuxTtsSolver``: the Swift enum's pure functions in float64 (features length, time steps, tokens index, the
  float64 anchor-Euler update).
* ``LuxTtsRequests``: the handle.  ``begin`` opens requests (prompt RMS, gain, mel, conditions, noise);
  ``text_condition``, ``model_inputs`` / ``advance`` (four times), ``vocoder_input`` and ``finish`` follow.
* ``LuxTtsSynthesizer.synthesize_batch``: the whole pipeline over caller-supplied model callables.
"""
from __future__ import annotations

import ctypes as C
import math
from dataclasses import dataclass
from typing import Callable, List, Optional, Sequence

import numpy as np

from . import _lib

FEAT_DIM = 100             # FA_LUXTTS_FEAT_DIM
MAX_FRAMES = 1024          # FA_LUXTTS_MAX_FRAMES
MAX_TOKENS = 256           # FA_LUXTTS_MAX_TOKENS
MAX_PROMPT_SAMPLES = 120000
NUM_STEPS = 4
T_SHIFT = 0.5
GUIDANCE_SCALE = 3.0
HOP_48K = 512
SAMPLE_RATE = 48000
VOCODER_BUCKETS = (282, 555)
STATUS_OUTPUT_TOO_SMALL = 3
REASONS = ("ok", "prompt produced no tokens", "text produced no tokens", "prompt audio has no samples",
           "speed must be > 0", "prompt audio is silent", "prompt too short for one mel frame",
           "prompt + text tokens + pad slot > 256", "features length > 1024 frames", "fewer than 2 generated frames",
           "generated frames exceed the largest vocoder bucket", "degenerate duration")


class LuxTtsError(ValueError):
    """A request refused with one of the reason codes (``REASONS``)."""

    def __init__(self, reason: int, request: int = 0):
        super().__init__(f"request {request}: {REASONS[reason]}")
        self.reason, self.request = reason, request


class LuxTtsSolver:
    """LuxTtsSolver.swift in float64"""

    @staticmethod
    def features_length(prompt_frames: int, prompt_token_count: int, text_token_count: int, speed: float) -> int:
        generated = float(prompt_frames) / float(prompt_token_count) * float(text_token_count) / float(speed)
        return prompt_frames + int(math.ceil(generated))

    @staticmethod
    def time_steps(num_steps: int = NUM_STEPS, t_shift: float = T_SHIFT) -> List[float]:
        out = []
        for i in range(num_steps + 1):
            u = float(i) / float(num_steps)
            out.append(t_shift * u / (1.0 + (t_shift - 1.0) * u))
        return out

    @staticmethod
    def tokens_index(tokens_count: int, features_length: int) -> List[int]:
        avg = features_length // tokens_count
        if avg < 1:
            raise LuxTtsError(11)
        index = [tokens_count] * features_length
        for f in range(tokens_count * avg):
            index[f] = f // avg
        return index

    @staticmethod
    def anchor_euler_update(x, v, t_cur: float, t_next: float, is_last: bool) -> np.ndarray:
        x, v = np.asarray(x, np.float64), np.asarray(v, np.float64)
        x1p = x + (1.0 - t_cur) * v
        if is_last:
            return x1p
        x0p = x - t_cur * v
        return (1.0 - t_next) * x0p + t_next * x1p


@dataclass
class LuxTtsPlan:
    reason: int
    prompt_samples: int
    prompt_frames: int
    token_count: int
    features_length: int
    gen_frames: int
    bucket: int
    boosted: bool
    prompt_rms: float
    step: int


def _plan_of(p: _lib.LuxTtsPlanInfo) -> LuxTtsPlan:
    return LuxTtsPlan(p.reason, p.prompt_samples, p.prompt_frames, p.token_count, p.features_length, p.gen_frames,
                      p.bucket, bool(p.boosted), float(np.float32(p.prompt_rms)), p.step)


def plan(prompt_samples: int, prompt_token_count: int, text_token_count: int, speed: float) -> LuxTtsPlan:
    """fa_luxtts_plan: the request geometry (reason 0) or the reason code it is refused with"""
    out = _lib.LuxTtsPlanInfo()
    _lib.check(_lib.load().fa_luxtts_plan(int(prompt_samples), int(prompt_token_count), int(text_token_count),
                                          float(np.float32(speed)), C.byref(out)), "fa_luxtts_plan")
    return _plan_of(out)


def _offsets(sizes):
    return np.concatenate([[0], np.cumsum(sizes, dtype=np.int64)]).astype(np.int64)


class LuxTtsRequests:
    """Live LuxTTS requests (fa_luxtts_*) on the current device"""

    def __init__(self):
        self._L = _lib.load()
        h = C.c_void_p()
        _lib.check(self._L.fa_luxtts_create(C.byref(h)), "fa_luxtts_create")
        self._h = h

    def close_handle(self):
        if getattr(self, "_h", None) is not None:
            self._L.fa_luxtts_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close_handle()
        except Exception:
            pass

    def begin(self, prompts, prompt_token_counts, text_token_counts, speeds, seeds):
        """(ids, plans, speech_condition [n x 1024 x 100], padding_mask [n x 1024]); LuxTtsError for the first
        refused request (its ``reasons`` attribute holds every request's code)"""
        xs = [np.ascontiguousarray(p, np.float32).reshape(-1) for p in prompts]
        n = len(xs)
        audio = np.concatenate(xs) if xs else np.zeros(0, np.float32)
        off = _offsets([x.size for x in xs])
        pt, tt = np.ascontiguousarray(prompt_token_counts, np.int32), np.ascontiguousarray(text_token_counts, np.int32)
        sp = np.ascontiguousarray(np.broadcast_to(np.asarray(speeds, np.float32), (n,)))
        sd = np.ascontiguousarray(np.broadcast_to(np.asarray(seeds, np.uint64), (n,)))
        reasons, ids = np.zeros(n, np.int32), np.zeros(n, np.int32)
        plans = (_lib.LuxTtsPlanInfo * max(n, 1))()
        sc, pm = np.empty((n, MAX_FRAMES, FEAT_DIM), np.float32), np.empty((n, MAX_FRAMES), np.float32)
        st = self._L.fa_luxtts_begin(self._h, n, _lib.ptr(audio), _lib.ptr(off), _lib.ptr(pt), _lib.ptr(tt),
                                     _lib.ptr(sp), _lib.ptr(sd), _lib.ptr(reasons), _lib.ptr(ids), plans, _lib.ptr(sc),
                                     _lib.ptr(pm))
        if st != 0 and reasons.any():
            i = int(np.flatnonzero(reasons)[0])
            err = LuxTtsError(int(reasons[i]), i)
            err.reasons = reasons
            raise err
        _lib.check(st, "fa_luxtts_begin")
        return ids, [_plan_of(plans[i]) for i in range(n)], sc, pm

    def text_condition(self, ids, token_embeds, row_stride: Optional[int] = None) -> np.ndarray:
        """text_condition [n x 1024 x 100] from token_embeds [n x rows x row_stride] (rows >= token_count + 1)"""
        ids = np.ascontiguousarray(ids, np.int32)
        e = np.ascontiguousarray(token_embeds, np.float32)
        rs = int(row_stride or e.shape[-1])
        out = np.empty((ids.size, MAX_FRAMES, FEAT_DIM), np.float32)
        _lib.check(self._L.fa_luxtts_text_condition(self._h, ids.size, _lib.ptr(ids), _lib.ptr(e), rs,
                                                    int(e[0].size) if ids.size else rs, _lib.ptr(out)),
                   "fa_luxtts_text_condition")
        return out

    def model_inputs(self, ids):
        """(x [n x 1024 x 100], t [n])"""
        ids = np.ascontiguousarray(ids, np.int32)
        x, t = np.empty((ids.size, MAX_FRAMES, FEAT_DIM), np.float32), np.empty(ids.size, np.float32)
        _lib.check(self._L.fa_luxtts_model_inputs(self._h, ids.size, _lib.ptr(ids), _lib.ptr(x), _lib.ptr(t)),
                   "fa_luxtts_model_inputs")
        return x, t

    def advance(self, ids, v, row_stride: Optional[int] = None):
        """one anchor-Euler update with v [n x rows x row_stride] (rows >= features_length)"""
        ids = np.ascontiguousarray(ids, np.int32)
        v = np.ascontiguousarray(v, np.float32)
        rs = int(row_stride or v.shape[-1])
        _lib.check(self._L.fa_luxtts_advance(self._h, ids.size, _lib.ptr(ids), _lib.ptr(v), rs,
                                             int(v[0].size) if ids.size else rs), "fa_luxtts_advance")

    def vocoder_input(self, ids, bucket: int) -> np.ndarray:
        ids = np.ascontiguousarray(ids, np.int32)
        out = np.empty((ids.size, FEAT_DIM, int(bucket)), np.float32)
        _lib.check(self._L.fa_luxtts_vocoder_input(self._h, ids.size, _lib.ptr(ids), int(bucket), _lib.ptr(out)),
                   "fa_luxtts_vocoder_input")
        return out

    def finish(self, ids, audio, row_length: Optional[int] = None) -> List[np.ndarray]:
        """each request's samples from audio [n x row_stride] (its first row_length samples); closes the requests"""
        ids = np.ascontiguousarray(ids, np.int32)
        a = np.ascontiguousarray(audio, np.float32).reshape(ids.size, -1) if ids.size else np.zeros((0, 1), np.float32)
        rl = int(a.shape[1] if row_length is None else row_length)
        lengths, total = np.zeros(ids.size, np.int64), C.c_int64()
        cap = int(ids.size * min(rl, (max(VOCODER_BUCKETS) - 1) * HOP_48K))
        out = np.empty(max(cap, 1), np.float32)
        _lib.check(self._L.fa_luxtts_finish(self._h, ids.size, _lib.ptr(ids), _lib.ptr(a), a.shape[1], rl,
                                            _lib.ptr(out), cap, _lib.ptr(lengths), C.byref(total)), "fa_luxtts_finish")
        at = _offsets(lengths)
        return [out[at[i]:at[i + 1]].copy() for i in range(ids.size)]

    def close(self, rid: int):
        _lib.check(self._L.fa_luxtts_close(self._h, int(rid)), "fa_luxtts_close")

    def state(self, rid: int, with_x: bool = True):
        """(plan, x [1024 x 100] or None)"""
        p = _lib.LuxTtsPlanInfo()
        x = np.empty((MAX_FRAMES, FEAT_DIM), np.float32) if with_x else None
        _lib.check(self._L.fa_luxtts_request_state(self._h, int(rid), C.byref(p), _lib.ptr(x)),
                   "fa_luxtts_request_state")
        return _plan_of(p), x


@dataclass
class LuxTtsSynthesisResult:
    samples: np.ndarray
    sample_rate: int
    prompt_frames: int
    generated_frames: int
    features_length: int


class LuxTtsSynthesizer:
    """LuxTtsSynthesizer.synthesize for many requests per call, over batched model callables:
      text_encoder(tokens [n x 256] int32, padding_mask [n x 256] float32) -> token_embeds [n x 256 x row_stride]
      fm_decoder(t [n], x, text_condition, speech_condition [n x 1024 x 100], guidance_scale [n], padding_mask
                 [n x 1024]) -> v [n x 1024 x row_stride]
      vocoder(mel [n x 100 x bucket]) -> audio [n x samples]
    Rows may be stride-padded past 100 floats, as CoreML's outputs are."""

    def __init__(self, text_encoder: Callable, fm_decoder: Callable, vocoder: Callable):
        self.text_encoder, self.fm_decoder, self.vocoder = text_encoder, fm_decoder, vocoder
        self.requests = LuxTtsRequests()

    @staticmethod
    def encoder_inputs(prompt_token_ids: Sequence[Sequence[int]], text_token_ids: Sequence[Sequence[int]]):
        """the text encoder's padded tokens and padding mask (1.0 from the token count on)"""
        n = len(prompt_token_ids)
        tokens, mask = np.zeros((n, MAX_TOKENS), np.int32), np.ones((n, MAX_TOKENS), np.float32)
        for i, (p, t) in enumerate(zip(prompt_token_ids, text_token_ids)):
            cat = list(p) + list(t)
            tokens[i, :len(cat)] = cat
            mask[i, :len(cat)] = 0.0
        return tokens, mask

    def synthesize_batch(self, prompt_token_ids, text_token_ids, prompt_audio_24k, speed=1.0,
                         seed=42) -> List[LuxTtsSynthesisResult]:
        n = len(prompt_audio_24k)
        R = self.requests
        ids, plans, sc, pm = R.begin(prompt_audio_24k, [len(p) for p in prompt_token_ids],
                                     [len(t) for t in text_token_ids], np.broadcast_to(np.float32(speed), (n,)),
                                     np.broadcast_to(np.uint64(seed), (n,)))
        try:
            tokens, tmask = self.encoder_inputs(prompt_token_ids, text_token_ids)
            embeds = np.ascontiguousarray(self.text_encoder(tokens, tmask), np.float32)
            tc = R.text_condition(ids, embeds)
            guidance = np.full(n, GUIDANCE_SCALE, np.float32)
            for _ in range(NUM_STEPS):
                x, t = R.model_inputs(ids)
                v = np.ascontiguousarray(self.fm_decoder(t, x, tc, sc, guidance, pm), np.float32)
                R.advance(ids, v)
            samples: List[Optional[np.ndarray]] = [None] * n
            for bucket in VOCODER_BUCKETS:
                sel = [i for i in range(n) if plans[i].bucket == bucket]
                if not sel:
                    continue
                mel = R.vocoder_input(ids[sel], bucket)
                audio = np.ascontiguousarray(self.vocoder(mel), np.float32)
                for i, s in zip(sel, R.finish(ids[sel], audio)):
                    samples[i] = s
        except BaseException:
            for rid in ids:
                try:
                    R.close(int(rid))
                except _lib.FluidAudioError:
                    pass
            raise
        return [LuxTtsSynthesisResult(samples[i], SAMPLE_RATE, plans[i].prompt_frames, plans[i].gen_frames,
                                      plans[i].features_length) for i in range(n)]
