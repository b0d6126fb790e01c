"""A literal Python restatement of StyleTTS2Synthesizer.synthesize's glue (test infrastructure), written from the Swift
source independently of oracle_styletts2.cpp: the bucket choice, bert's padding and mask, StyleTTS2NoiseSource
(luxtts_restated.Noise, the same Swift struct), roundDurations with numpy float32 scalars and expf the correctly
rounded float32 exp (float_exact.py), buildAlignmentMatrix, matmulAligned as netlib's loop, transposeLast2D, hifiganShift, blendStyle
and the tail trim."""
import math

import numpy as np

import float_exact
from luxtts_restated import Noise

F = np.float32


def bucket(n):
    if n == 0:
        return 0, 1
    if n <= 57:
        return 57, 0
    for size in (64, 128, 256):
        if n <= size:
            return size, 0
    return 0, 2


def sampler_inputs(ids, padded_t, seed):
    ids = list(ids)
    tokens = np.array(ids + [0] * (padded_t - len(ids)), np.int32)
    mask = np.array([1] * len(ids) + [0] * (padded_t - len(ids)), np.int32)
    rng = Noise(seed)
    noise_init = np.array([rng.gaussian() for _ in range(256)], np.float32)
    noises_aux = np.array([[rng.gaussian() for _ in range(256)] for _ in range(4)], np.float32)
    return tokens, mask, noise_init, noises_aux


_expf = float_exact.exp


def round_durations(logits):
    out = []
    with np.errstate(all="ignore"):
        for row in np.asarray(logits, np.float32):
            s = F(0)
            for x in row:
                s = F(s + F(F(1) / F(F(1) + _expf(-x))))
            if math.isnan(s):
                return None
            out.append(max(int(math.floor(float(s) + 0.5)), 1))   # s >= 0: half away from zero
    return out


def alignment(durations):
    total = sum(durations)
    m = np.zeros((len(durations), total), np.float32)
    col = 0
    for i, d in enumerate(durations):
        m[i, col:col + d] = 1
        col += d
    return m, total


def matmul_aligned(features, aln):
    features, aln = np.asarray(features, np.float32), np.asarray(aln, np.float32)
    out = np.zeros((features.shape[0], aln.shape[1]), np.float32)
    with np.errstate(all="ignore"):
        for j in range(aln.shape[1]):
            for l in range(aln.shape[0]):
                if aln[l, j] != 0:
                    out[:, j] = out[:, j] + F(1) * aln[l, j] * features[:, l]
    return out


def transpose(src):
    src = np.asarray(src, np.float32)
    return np.array([[src[r, c] for r in range(src.shape[0])] for c in range(src.shape[1])], np.float32).reshape(
        src.shape[1], src.shape[0])


def hifigan_shift(x):
    x = np.asarray(x, np.float32)
    out = np.zeros_like(x)
    out[:, 0] = x[:, 0]
    out[:, 1:] = x[:, :-1]
    return out


def blend(s_pred, ref_s, alpha, beta):
    p, r = np.asarray(s_pred, np.float32), np.asarray(ref_s, np.float32)
    a, b = F(alpha), F(beta)
    with np.errstate(all="ignore"):
        ref = np.array([F(F(a * p[i]) + F(F(F(1) - a) * r[i])) for i in range(128)], np.float32)
        s = np.array([F(F(b * p[128 + i]) + F(F(F(1) - b) * r[128 + i])) for i in range(128)], np.float32)
    return ref, s


def trim(audio):
    a = list(np.asarray(audio, np.float32).reshape(-1))
    k = min(50, len(a))
    return np.array(a[:len(a) - k] if k > 0 else a, np.float32)
