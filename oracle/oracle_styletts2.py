"""ORACLE — TEST INFRASTRUCTURE ONLY.  Not part of the shipped product path.

ctypes front-end to ``liboracle_styletts2.so``, the sequential CPU restatement of StyleTTS2Synthesizer.synthesize's
glue between its models (``oracle_styletts2.cpp``: the bucket choice, bert's padding and mask, StyleTTS2NoiseSource,
roundDurations, buildAlignmentMatrix, matmulAligned as netlib's loop, transposeLast2D, hifiganShift, blendStyle and
the tail trim), compiled into its own library with the main oracle's pinned flags (``-O2 -ffp-contract=off`` on
baseline x86-64).  ``synthesize`` drives it around caller-supplied models.  Importers allowed: ``tests/``,
``__graft_entry__`` and ``scripts/``.  The product package never imports it.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRCS = [os.path.join(_HERE, "oracle_styletts2.cpp")]
_LIB = os.path.join(_HERE, "liboracle_styletts2.so")
_FLAGS = ["-std=c++17", "-O2", "-ffp-contract=off", "-fPIC", "-Wall", "-Wextra", "-shared"]

STYLE_DIM, REF_SPLIT, NOISE_ROWS = 256, 128, 5

_lib = None


def build(force: bool = False) -> None:
    """Compile liboracle_styletts2.so when it is missing or older than a source."""
    if force or not os.path.exists(_LIB) or any(os.path.getmtime(s) > os.path.getmtime(_LIB) for s in _SRCS):
        cxx = os.environ.get("CXX", "g++")
        subprocess.check_call([cxx, *_FLAGS, "-o", _LIB, *_SRCS])


def lib():
    global _lib
    if _lib is None:
        build()
        L = C.CDLL(_LIB)
        vp, i64, f32 = C.c_void_p, C.c_int64, C.c_float
        L.oracle_styletts2_bucket.argtypes = [i64, vp]
        L.oracle_styletts2_bucket.restype = C.c_int
        L.oracle_styletts2_sampler_inputs.argtypes = [vp, i64, i64, C.c_uint64, vp, vp, vp, vp]
        L.oracle_styletts2_sampler_inputs.restype = None
        L.oracle_styletts2_noise.argtypes = [C.c_uint64, i64, vp]
        L.oracle_styletts2_noise.restype = None
        L.oracle_styletts2_round_durations.argtypes = [vp, i64, i64, vp]
        L.oracle_styletts2_round_durations.restype = C.c_int
        L.oracle_styletts2_total_frames.argtypes = [vp, i64]
        L.oracle_styletts2_total_frames.restype = i64
        L.oracle_styletts2_alignment.argtypes = [vp, i64, i64, vp]
        L.oracle_styletts2_alignment.restype = None
        L.oracle_styletts2_matmul_aligned.argtypes = [vp, i64, i64, vp, i64, vp]
        L.oracle_styletts2_matmul_aligned.restype = None
        L.oracle_styletts2_transpose.argtypes = [vp, i64, i64, vp]
        L.oracle_styletts2_transpose.restype = None
        L.oracle_styletts2_hifigan_shift.argtypes = [vp, i64, i64, vp]
        L.oracle_styletts2_hifigan_shift.restype = None
        L.oracle_styletts2_blend.argtypes = [vp, vp, f32, f32, vp, vp]
        L.oracle_styletts2_blend.restype = None
        L.oracle_styletts2_trim.argtypes = [i64]
        L.oracle_styletts2_trim.restype = i64
        _lib = L
    return _lib


def _f32(a):
    return np.ascontiguousarray(a, np.float32)


def bucket(token_count):
    """(bucket, reason)"""
    r = C.c_int32()
    b = lib().oracle_styletts2_bucket(int(token_count), C.byref(r))
    return int(b), int(r.value)


def sampler_inputs(ids, padded_t, seed):
    """(tokens [T] int32, attention_mask [T] int32, noise_init [256], noises_aux [4 x 256])"""
    ids = np.ascontiguousarray(ids, np.int32)
    tokens, mask = np.empty(int(padded_t), np.int32), np.empty(int(padded_t), np.int32)
    ni, na = np.empty(STYLE_DIM, np.float32), np.empty((NOISE_ROWS - 1, STYLE_DIM), np.float32)
    lib().oracle_styletts2_sampler_inputs(ids.ctypes.data, ids.size, int(padded_t), int(seed) & (2**64 - 1),
                                          tokens.ctypes.data, mask.ctypes.data, ni.ctypes.data, na.ctypes.data)
    return tokens, mask, ni, na


def noise(seed, count) -> np.ndarray:
    out = np.empty(int(count), np.float32)
    lib().oracle_styletts2_noise(int(seed) & (2**64 - 1), out.size, out.ctypes.data)
    return out


def round_durations(logits):
    """durations [n] int64 from logits [n x C], or None where Int(NaN) traps"""
    logits = _f32(logits)
    out = np.empty(logits.shape[0], np.int64)
    r = lib().oracle_styletts2_round_durations(logits.ctypes.data, logits.shape[0], logits.shape[1], out.ctypes.data)
    return None if r else out


def alignment(durations):
    """(matrix [n x F], F)"""
    d = np.ascontiguousarray(durations, np.int64)
    total = int(lib().oracle_styletts2_total_frames(d.ctypes.data, d.size))
    out = np.empty((d.size, total), np.float32)
    lib().oracle_styletts2_alignment(d.ctypes.data, d.size, total, out.ctypes.data)
    return out, total


def matmul_aligned(features, alignment_matrix):
    features, a = _f32(features), _f32(alignment_matrix)
    out = np.empty((features.shape[0], a.shape[1]), np.float32)
    lib().oracle_styletts2_matmul_aligned(features.ctypes.data, features.shape[0], features.shape[1], a.ctypes.data,
                                          a.shape[1], out.ctypes.data)
    return out


def transpose(src):
    src = _f32(src)
    out = np.empty((src.shape[1], src.shape[0]), np.float32)
    lib().oracle_styletts2_transpose(src.ctypes.data, src.shape[0], src.shape[1], out.ctypes.data)
    return out


def hifigan_shift(x):
    x = _f32(x)
    out = np.empty_like(x)
    lib().oracle_styletts2_hifigan_shift(x.ctypes.data, x.shape[0], x.shape[1], out.ctypes.data)
    return out


def blend(s_pred, ref_s, alpha, beta):
    """(ref [128], s [128])"""
    p, r = _f32(s_pred).reshape(-1), _f32(ref_s).reshape(-1)
    ref, s = np.empty(REF_SPLIT, np.float32), np.empty(REF_SPLIT, np.float32)
    lib().oracle_styletts2_blend(p.ctypes.data, r.ctypes.data, float(np.float32(alpha)), float(np.float32(beta)),
                                 ref.ctypes.data, s.ctypes.data)
    return ref, s


def trim(audio):
    audio = _f32(audio).reshape(-1)
    return audio[:int(lib().oracle_styletts2_trim(audio.size))]


def align(logits, d, t_en):
    """synthesize's steps from roundDurations to the shifts: (durations, F, en [dC x F], asr [tC x F]) for one request
    with logits [n x C], d [n x dC] and t_en [tC x n]; None where roundDurations traps"""
    durations = round_durations(logits)
    if durations is None:
        return None
    aln, total = alignment(durations)
    d = _f32(d)
    en = matmul_aligned(transpose(d), aln)
    asr = matmul_aligned(_f32(t_en), aln)
    return durations, total, hifigan_shift(en), hifigan_shift(asr)


def synthesize(token_ids, ref_mel, alpha, beta, seed, text_encoder, bert, ref_encoder, sampler, duration_predictor,
               f0n_har, decoder_pre, decoder_upsample):
    """StyleTTS2Synthesizer.synthesize for one request around fake models (each takes and returns numpy arrays in the
    shapes synthesize feeds and reads):
      text_encoder(tokens [1 x n], lengths [1], text_mask [1 x n]) -> t_en [1 x tC x n]
      bert(tokens [1 x T], attention_mask [1 x T]) -> (bert_dur [1 x T x 768], d_en [1 x dC' x T])
      ref_encoder(mel [1 x 1 x 80 x frames]) -> ref_s [1 x 256]
      sampler(noise_init [1 x 1 x 256], noises_aux [4 x 1 x 1 x 256], embedding [1 x T x 768], features [1 x 256])
        -> s_pred [1 x 1 x 256]
      duration_predictor(d_en [1 x dC' x n], s [1 x 128], text_mask [1 x n]) -> (d [1 x n x dC], logits [1 x n x C])
      f0n_har(en [1 x dC x F], s [1 x 128]) -> (f0 [1 x k], n [1 x k], har [1 x 1 x h])
      decoder_pre(asr [1 x tC x F], f0, n, ref [1 x 128]) -> x_pre [1 x 512 x 2F]
      decoder_upsample(x_pre, ref [1 x 128], har) -> audio [1 x samples]
    Returns (samples, F, durations), or the reason code as an int."""
    ids = np.ascontiguousarray(token_ids, np.int32)
    real_n = ids.size
    chosen, reason = bucket(real_n)
    if reason:
        return reason
    t_en = _f32(text_encoder(ids[None], np.array([real_n], np.int32), np.zeros((1, real_n), np.float32)))
    tokens, mask, noise_init, noises_aux = sampler_inputs(ids, chosen, seed)
    bert_dur, d_en_padded = bert(tokens[None], mask[None])
    d_en = _f32(d_en_padded)[:, :, :real_n]
    ref_s = _f32(ref_encoder(_f32(ref_mel)[None, None])).reshape(-1)
    s_pred = _f32(sampler(noise_init.reshape(1, 1, STYLE_DIM), noises_aux.reshape(NOISE_ROWS - 1, 1, 1, STYLE_DIM),
                          _f32(bert_dur), ref_s[None])).reshape(-1)
    ref128, s128 = blend(s_pred, ref_s, alpha, beta)
    d, logits = duration_predictor(d_en, s128[None], np.zeros((1, real_n), np.float32))
    aligned = align(_f32(logits)[0], _f32(d)[0], t_en[0])
    if aligned is None:
        return 3
    durations, total, en, asr = aligned
    f0, n, har = f0n_har(en[None], s128[None])
    x_pre = decoder_pre(asr[None], f0, n, ref128[None])
    audio = decoder_upsample(x_pre, ref128[None], har)
    return trim(audio), total, durations
