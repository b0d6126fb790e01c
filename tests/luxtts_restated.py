"""A literal Python restatement of LuxTtsSynthesizer.synthesize's host arithmetic (test infrastructure), written from
the Swift source independently of oracle_luxtts.cpp: the guards in order, vDSP_measqv as an index-order float64 sum,
StyleTTS2NoiseSource with Python's (libm) log and cos, the float32 vDSP anchor-Euler path with numpy float32 scalars,
the vocoder input and the output's truncation, vDSP_vclip and rescale."""
import math

import numpy as np

F = np.float32
MASK = (1 << 64) - 1


def plan(samples, prompt_tokens, text_tokens, speed):
    """(reason, prompt_samples, prompt_frames, token_count, features_length, gen_frames, bucket)"""
    z = [0] * 6
    if prompt_tokens == 0:
        return (1, *z)
    if text_tokens == 0:
        return (2, *z)
    if samples == 0:
        return (3, *z)
    speed = F(speed)
    if not speed > 0:
        return (4, *z)
    n = min(samples, int(5.0 * 24000.0))
    frames = (n + 128) // 256
    if not frames > 0:
        return (6, n, frames, 0, 0, 0, 0)
    count = prompt_tokens + text_tokens
    if not count + 1 <= 256:
        return (7, n, frames, 0, 0, 0, 0)
    gen = float(frames) / float(prompt_tokens) * float(text_tokens) / float(speed)
    if math.isinf(gen) or math.ceil(gen) >= 2**63 or frames + math.ceil(gen) >= 2**63:
        return (8, n, frames, count, 0, 0, 0)
    length = frames + math.ceil(gen)
    if not length <= 1024:
        return (8, n, frames, count, 0, 0, 0)
    g = length - frames
    if not g >= 2:
        return (9, n, frames, count, length, g, 0)
    bucket = next((b for b in (282, 555) if b >= g), 0)
    if not bucket:
        return (10, n, frames, count, length, g, 0)
    if length // count < 1:
        return (11, n, frames, count, length, g, bucket)
    return (0, n, frames, count, length, g, bucket)


def rms(x):
    s = 0.0
    for v in np.asarray(x, np.float32).tolist():
        s += v * v
    return F(math.sqrt(F(s / len(x))))


class Noise:
    def __init__(self, seed):
        self.state = 0xdeadbeefcafebabe if seed == 0 else seed

    def uniform(self):
        self.state = (self.state + 0x9E3779B97F4A7C15) & MASK
        z = self.state
        z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & MASK
        z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & MASK
        z = z ^ (z >> 31)
        u = float(z >> 11) / float(1 << 53)
        return u if u > 0 else 2.2250738585072014e-308

    def gaussian(self):
        u1 = self.uniform()
        u2 = self.uniform()
        mag = math.sqrt(-2.0 * math.log(u1))
        return F(mag * math.cos(2.0 * math.pi * u2))


def time_steps():
    return [0.5 * (i / 4) / (1.0 + (0.5 - 1.0) * (i / 4)) for i in range(5)]


def step(x, v, k):
    tc, tn = F(time_steps()[k]), F(time_steps()[k + 1])
    out = np.empty(len(x), np.float32)
    with np.errstate(all="ignore"):
        for i, (xi, vi) in enumerate(zip(np.asarray(x, np.float32), np.asarray(v, np.float32))):
            x1p = F(F(vi * F(F(1) - tc)) + xi)
            if k == 3:
                out[i] = x1p
                continue
            x0p = F(F(vi * F(-tc)) + xi)
            out[i] = F(F(x0p * F(F(1) - tn)) + F(x1p * tn))
    return out


def tokens_index(count, length):
    avg = length // count
    if avg < 1:
        return None
    index = [count] * length
    for f in range(count * avg):
        index[f] = f // avg
    return index


def vocoder_input(x, frames, gen, bucket):
    x = np.asarray(x, np.float32).reshape(-1)
    out = np.full((100, bucket), F(np.log(F(1e-7))), np.float32)
    for m in range(100):
        for f in range(gen):
            out[m, f] = F(x[(frames + f) * 100 + m] * F(F(1) / F(0.1)))
    return out


def finish(audio, gen, prompt_rms):
    a = np.asarray(audio, np.float32)[:min((gen - 1) * 512, len(audio))]
    out = np.array([F(-1) if v < -1 else F(1) if v > 1 else v for v in a.tolist()], np.float32)
    if prompt_rms < F(0.1):
        with np.errstate(all="ignore"):
            out = (out * F(F(prompt_rms) / F(0.1))).astype(np.float32)
    return out
