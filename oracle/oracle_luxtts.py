"""ORACLE — TEST INFRASTRUCTURE ONLY.  Not part of the shipped product path.

ctypes front-end to ``liboracle_luxtts.so``, the sequential CPU restatement of LuxTtsSynthesizer.synthesize's host
arithmetic (``oracle_luxtts.cpp``: the plan and its guards, the RMS and gain, StyleTTS2NoiseSource, the conditions, the
float32 anchor-Euler steps, the vocoder input and the output's truncation, clip and rescale), compiled into its own
library with the main oracle's pinned flags (``-O2 -ffp-contract=off`` on baseline x86-64).  ``synthesize`` drives it
around caller-supplied models and the prompt mel.  Importers allowed: ``tests/``, ``__graft_entry__`` and
``scripts/``.  The product package never imports it.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRCS = [os.path.join(_HERE, "oracle_luxtts.cpp")]
_LIB = os.path.join(_HERE, "liboracle_luxtts.so")
_FLAGS = ["-std=c++17", "-O2", "-ffp-contract=off", "-fPIC", "-Wall", "-Wextra", "-shared"]

FEAT, MAX_FRAMES, MAX_TOKENS = 100, 1024, 256

_lib = None


def build(force: bool = False) -> None:
    """Compile liboracle_luxtts.so when it is missing or older than a source."""
    if force or not os.path.exists(_LIB) or any(os.path.getmtime(s) > os.path.getmtime(_LIB) for s in _SRCS):
        cxx = os.environ.get("CXX", "g++")
        subprocess.check_call([cxx, *_FLAGS, "-o", _LIB, *_SRCS])


def lib():
    global _lib
    if _lib is None:
        build()
        L = C.CDLL(_LIB)
        vp, i64, i32, f32, f64 = C.c_void_p, C.c_int64, C.c_int32, C.c_float, C.c_double
        L.oracle_luxtts_plan.argtypes = [i64, i32, i32, f32, vp]
        L.oracle_luxtts_plan.restype = C.c_int
        L.oracle_luxtts_rms.argtypes = [vp, i64]
        L.oracle_luxtts_rms.restype = f32
        L.oracle_luxtts_gain.argtypes = [vp, i64, f32, vp]
        L.oracle_luxtts_gain.restype = None
        L.oracle_luxtts_noise.argtypes = [C.c_uint64, i64, vp]
        L.oracle_luxtts_noise.restype = None
        L.oracle_luxtts_uniforms.argtypes = [C.c_uint64, i64, vp]
        L.oracle_luxtts_uniforms.restype = None
        L.oracle_luxtts_time_steps.argtypes = [vp]
        L.oracle_luxtts_time_steps.restype = None
        L.oracle_luxtts_tokens_index.argtypes = [i64, i64, vp]
        L.oracle_luxtts_tokens_index.restype = C.c_int
        L.oracle_luxtts_anchor_euler_f64.argtypes = [vp, vp, i64, f64, f64, C.c_int, vp]
        L.oracle_luxtts_anchor_euler_f64.restype = None
        L.oracle_luxtts_step.argtypes = [vp, vp, i64, C.c_int]
        L.oracle_luxtts_step.restype = None
        L.oracle_luxtts_conditions.argtypes = [vp, i64, i64, vp, i64, vp, vp, vp]
        L.oracle_luxtts_conditions.restype = C.c_int
        L.oracle_luxtts_vocoder_input.argtypes = [vp, i64, i64, i64, vp]
        L.oracle_luxtts_vocoder_input.restype = None
        L.oracle_luxtts_finish.argtypes = [vp, i64, i64, f32, vp]
        L.oracle_luxtts_finish.restype = i64
        _lib = L
    return _lib


def _f32(a):
    return np.ascontiguousarray(a, np.float32)


def plan(samples, prompt_tokens, text_tokens, speed):
    """(reason, prompt_samples, prompt_frames, token_count, features_length, gen_frames, bucket)"""
    out = np.zeros(6, np.int32)
    r = lib().oracle_luxtts_plan(int(samples), int(prompt_tokens), int(text_tokens), float(np.float32(speed)),
                                 out.ctypes.data)
    return (int(r), *(int(v) for v in out))


def rms(x) -> np.float32:
    x = _f32(x)
    return np.float32(lib().oracle_luxtts_rms(x.ctypes.data, x.size))


def gain(x, prompt_rms) -> np.ndarray:
    x = _f32(x)
    out = np.empty_like(x)
    lib().oracle_luxtts_gain(x.ctypes.data, x.size, float(prompt_rms), out.ctypes.data)
    return out


def noise(seed, count) -> np.ndarray:
    out = np.empty(int(count), np.float32)
    lib().oracle_luxtts_noise(int(seed) & (2**64 - 1), out.size, out.ctypes.data)
    return out


def uniforms(seed, count) -> np.ndarray:
    out = np.empty(int(count), np.float64)
    lib().oracle_luxtts_uniforms(int(seed) & (2**64 - 1), out.size, out.ctypes.data)
    return out


def time_steps() -> np.ndarray:
    out = np.empty(5, np.float64)
    lib().oracle_luxtts_time_steps(out.ctypes.data)
    return out


def tokens_index(tokens_count, features_length):
    """the index array, or None for the degenerate duration"""
    out = np.empty(max(int(features_length), 1), np.int64)
    r = lib().oracle_luxtts_tokens_index(int(tokens_count), int(features_length), out.ctypes.data)
    return None if r else out[:int(features_length)]


def anchor_euler_f64(x, v, t_cur, t_next, is_last) -> np.ndarray:
    x, v = np.ascontiguousarray(x, np.float64), np.ascontiguousarray(v, np.float64)
    out = np.empty_like(x)
    lib().oracle_luxtts_anchor_euler_f64(x.ctypes.data, v.ctypes.data, x.size, float(t_cur), float(t_next),
                                         int(bool(is_last)), out.ctypes.data)
    return out


def step(x, v, step_index) -> np.ndarray:
    """one float32 step over x.size active elements (a new array)"""
    x, v = _f32(x).copy(), _f32(v)
    lib().oracle_luxtts_step(x.ctypes.data, v.ctypes.data, x.size, int(step_index))
    return x


def conditions(embeds, token_count, features_length, prompt_mel):
    """(text_condition, speech_condition [1024 x 100], frame_mask [1024]) from compact embeds [(S + 1) x 100]"""
    embeds, prompt_mel = _f32(embeds), _f32(prompt_mel)
    tc, sc = np.empty((MAX_FRAMES, FEAT), np.float32), np.empty((MAX_FRAMES, FEAT), np.float32)
    mask = np.empty(MAX_FRAMES, np.float32)
    r = lib().oracle_luxtts_conditions(embeds.ctypes.data, int(token_count), int(features_length),
                                       prompt_mel.ctypes.data, prompt_mel.shape[0], tc.ctypes.data, sc.ctypes.data,
                                       mask.ctypes.data)
    assert r == 0
    return tc, sc, mask


def vocoder_input(x, prompt_frames, gen_frames, bucket) -> np.ndarray:
    x = _f32(x)
    out = np.empty((FEAT, int(bucket)), np.float32)
    lib().oracle_luxtts_vocoder_input(x.ctypes.data, int(prompt_frames), int(gen_frames), int(bucket), out.ctypes.data)
    return out


def finish(audio, gen_frames, prompt_rms) -> np.ndarray:
    audio = _f32(audio)
    out = np.empty(audio.size, np.float32)
    n = lib().oracle_luxtts_finish(audio.ctypes.data, audio.size, int(gen_frames), float(prompt_rms), out.ctypes.data)
    return out[:n]


def synthesize(prompt_tokens, text_tokens, prompt_audio, speed, seed, text_encoder, fm_decoder, vocoder, prompt_mel):
    """LuxTtsSynthesizer.synthesize for one request around the caller's models.  ``prompt_mel(gained_prompt)`` gives
    the unscaled [T x 100] mel.  text_encoder(tokens [1 x 256] int32, mask [1 x 256]) -> embeds [1 x 256 x 100];
    fm_decoder(t [1], x, text_condition, speech_condition, guidance [1], padding_mask [1 x 1024]) -> v [1 x 1024 x 100];
    vocoder(mel [1 x 100 x bucket]) -> audio [1 x samples].  Returns (samples, prompt_frames, gen_frames,
    features_length), or the reason code as an int."""
    prompt_audio = _f32(prompt_audio)
    r, n, P, S, L, G, bucket = plan(prompt_audio.size, len(prompt_tokens), len(text_tokens), speed)
    if r in (1, 2, 3, 4):
        return r
    prompt = prompt_audio[:n]
    prompt_rms = rms(prompt)
    if not prompt_rms > 0:
        return 5
    if r:
        return r
    mel = _f32(prompt_mel(gain(prompt, prompt_rms)))
    assert mel.shape[0] == P
    tokens = np.zeros((1, MAX_TOKENS), np.int32)
    tokens[0, :S] = list(prompt_tokens) + list(text_tokens)
    tmask = np.zeros((1, MAX_TOKENS), np.float32)
    tmask[0, S:] = 1.0
    embeds = _f32(text_encoder(tokens, tmask))[0, :S + 1, :FEAT]
    tc, sc, mask = conditions(embeds, S, L, mel)
    x = noise(seed, L * FEAT)
    for k in range(4):
        xa = np.zeros((MAX_FRAMES, FEAT), np.float32)
        xa.reshape(-1)[:L * FEAT] = x
        t = np.array([np.float32(time_steps()[k])], np.float32)
        v = _f32(fm_decoder(t, xa[None], tc[None], sc[None], np.array([3.0], np.float32), mask[None]))
        x = step(x, v.reshape(-1)[:L * FEAT], k)
    full = np.zeros(MAX_FRAMES * FEAT, np.float32)
    full[:L * FEAT] = x
    audio = _f32(vocoder(vocoder_input(full, P, G, bucket)[None])).reshape(-1)
    return finish(audio, G, prompt_rms), P, G, L
