"""Deterministic synthetic workloads for tests, smoke() and bench.py (SURVEY.md §8d).

numpy only; no dependency on the CUDA library or on oracle/.  The shapes mirror BASELINE.json's configs:

* ``tone_noise_audio``   the reference's own mel fixture, Tests/FluidAudioTests/Diarizer/Sortformer/
  SortformerStreamingMelTests.swift:17-25: 0.3 sin(2 pi 220 t) + 0.15 sin(2 pi 517 t) + 0.05 (u - 0.5),
  computed in float32.  The noise term is mandatory: without broadband energy most mel bins sit at the float32
  FFT noise floor and no two float32 implementations agree to 1e-4 in the log domain.  The Swift test draws
  ``u`` from drand48 seeded with 7; here ``u`` comes from a counter-based hash (any length, any offset, no state)
  so that a 1-hour signal can be generated in chunks on any rank.
* ``speaker_embeddings``  K unit-norm speaker centres + isotropic noise, stored float32 (TimedEmbedding.embedding256).
* ``synthetic_plda``      a stand-in for the PLDA rho transform, whose real weights live in a CoreML model that is
  not part of the reference repository ("parity unpinned", SURVEY §0 D7): rho = (unit(e) - mean) W, psi decaying.
"""
from __future__ import annotations

import numpy as np


def _hash_uniform(idx: np.ndarray, seed: int) -> np.ndarray:
    """Counter-based U[0,1) in float64 from 64-bit indices (splitmix64 finaliser)."""
    z = idx.astype(np.uint64) + np.uint64(0x9E3779B97F4A7C15) * np.uint64(seed + 1)
    z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
    z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
    z = z ^ (z >> np.uint64(31))
    return (z >> np.uint64(11)).astype(np.float64) * (1.0 / 9007199254740992.0)


def tone_noise_audio(n: int, seed: int = 7, start: int = 0, sample_rate: int = 16000) -> np.ndarray:
    """float32 samples [start, start+n) of the tone+noise signal."""
    with np.errstate(over="ignore"):
        idx = np.arange(start, start + n, dtype=np.int64)
        t = (idx.astype(np.float32) / np.float32(sample_rate)).astype(np.float32)
        two_pi = np.float32(2.0) * np.float32(np.pi)
        tone = np.float32(0.3) * np.sin(two_pi * np.float32(220.0) * t, dtype=np.float32) + np.float32(0.15) * np.sin(
            two_pi * np.float32(517.0) * t, dtype=np.float32)
        u = _hash_uniform(idx, seed)
        noise = ((u - 0.5).astype(np.float32)) * np.float32(0.05)
        return (tone + noise).astype(np.float32)


def speech_like_audio(n: int, seed: int = 11, sample_rate: int = 16000) -> np.ndarray:
    """Harder mel fixture: amplitude-modulated harmonics with pauses + low-level noise (60 dB dynamic range)."""
    rng = np.random.default_rng(seed)
    t = np.arange(n, dtype=np.float64) / sample_rate
    f0 = 110.0 + 40.0 * np.sin(2 * np.pi * 0.7 * t)
    phase = 2 * np.pi * np.cumsum(f0) / sample_rate
    sig = sum((0.5 / k) * np.sin(k * phase + 0.3 * k) for k in range(1, 12))
    env = np.clip(np.sin(2 * np.pi * 1.3 * t), 0, None) ** 2
    sig = sig * env * 0.4 + 1e-3 * rng.standard_normal(n)
    return sig.astype(np.float32)


def speaker_embeddings(n: int, dim: int = 256, speakers: int = 8, weights=None, sigma: float = 0.02,
                       seed: int = 42) -> tuple[np.ndarray, np.ndarray]:
    """Returns (embeddings float32 [n x dim], true speaker id int32 [n])."""
    rng = np.random.default_rng(seed)
    centres = rng.standard_normal((speakers, dim))
    centres /= np.linalg.norm(centres, axis=1, keepdims=True)
    if weights is None:
        weights = np.arange(speakers, 0, -1, dtype=np.float64)
    w = np.asarray(weights, np.float64)
    w = w / w.sum()
    who = rng.choice(speakers, size=n, p=w).astype(np.int32)
    emb = centres[who] + sigma * rng.standard_normal((n, dim))
    return emb.astype(np.float32), who


def synthetic_plda(emb: np.ndarray, rho_dim: int = 128, seed: int = 1234) -> tuple[np.ndarray, np.ndarray]:
    """Returns (rho float64 [n x rho_dim], psi float64 [rho_dim]) from float32 embeddings."""
    e = emb.astype(np.float64)
    dim = e.shape[1]
    rng = np.random.default_rng(seed)
    q, _ = np.linalg.qr(rng.standard_normal((dim, dim)))
    W = q[:, :rho_dim] * np.sqrt(float(rho_dim))
    unit = e / np.maximum(np.linalg.norm(e, axis=1, keepdims=True), 1e-30)
    rho = (unit - unit.mean(axis=0, keepdims=True)) @ W
    psi = (0.1 + 10.0 * np.exp(-np.arange(rho_dim) / 32.0)).astype(np.float32).astype(np.float64)
    return np.ascontiguousarray(rho), psi


def segmentation_logits(duration_s: float, speakers: int = 3, seed: int = 5, frames: int = 589, classes: int = 7,
                        sample_rate: int = 16000, window_duration: float = 10.0, step_ratio: float = 0.2,
                        margin: float = 6.0, noise: float = 1.0) -> tuple[np.ndarray, dict]:
    """Powerset logits a segmentation network could emit for a synthetic conversation, and the conversation itself.

    A seeded turn-taking timeline (turns of 2.5-6 s, a third of them starting up to 1 s before the previous one ends, a
    fifth preceded by 0.5-1.5 s of silence) is cut into the analysis windows of OfflineSegmentationProcessor (a window
    every ``window_duration * step_ratio`` seconds, the last ones reaching past the end of the audio, where they are
    silent).  Inside a window the global speakers take local slots 0..2 in order of first appearance (a fourth is
    dropped, as a 3-speaker powerset model would); frame f is labelled by who speaks at offset + f * frame_duration, and
    its logits are ``noise`` * N(0, 1) with ``margin`` added to the class of that speaker set.

    Returns (logits float32 [chunks, frames, classes], truth) with truth = dict(turns float64 [n, 3] rows (speaker,
    start, end), chunk_offsets, frame_duration, total_samples, slot_speaker int32 [chunks, 3] (global speaker of each
    local slot, -1 = unused), labels int32 [chunks, frames] (the powerset class of every frame)).
    """
    rng = np.random.default_rng(seed)
    turns, t, prev = [], 0.0, -1
    while t < duration_s:
        if turns and rng.random() < 0.2:
            t += rng.uniform(0.5, 1.5)
        elif turns and rng.random() < 1.0 / 3.0:
            t -= rng.uniform(0.3, 1.0)
        who = int(rng.integers(speakers))
        if who == prev and speakers > 1:
            who = (who + 1) % speakers
        length = rng.uniform(2.5, 6.0)
        if t < duration_s:
            turns.append((who, max(t, 0.0), min(t + length, duration_s)))
        t, prev = t + length, who
    turns = np.asarray(turns, np.float64).reshape(-1, 3)
    total_samples = int(round(duration_s * sample_rate))
    window = int(sample_rate * window_duration)
    step = max(1, int(window * step_ratio))
    offsets = np.arange(0, total_samples, step, dtype=np.float64) / sample_rate
    frame_duration = window_duration / frames
    class_of_bits = np.array([0, 1, 2, 4, 3, 5, 6, 7])   # bit s = local speaker s -> {}, {0}, {1}, {0,1}, {2}, {0,2}, {1,2}, {0,1,2}
    chunks = offsets.size
    labels = np.zeros((chunks, frames), np.int32)
    slot_speaker = np.full((chunks, 3), -1, np.int32)
    for c, off in enumerate(offsets):
        times = off + np.arange(frames) * frame_duration
        active = np.zeros((frames, speakers), bool)
        for who, a, b in turns[(turns[:, 2] > off) & (turns[:, 1] < off + window_duration)]:
            active[:, int(who)] |= (times >= a) & (times < b) & (times < duration_s)
        order = [k for k in np.argsort([np.argmax(active[:, k]) if active[:, k].any() else frames + k
                                        for k in range(speakers)], kind="stable") if active[:, k].any()][:3]
        slot_speaker[c, :len(order)] = order
        who_bits = np.zeros(frames, np.int64)
        for s, k in enumerate(order):
            who_bits |= active[:, k].astype(np.int64) << s
        labels[c] = np.minimum(class_of_bits[who_bits], classes - 1)
    logits = (noise * rng.standard_normal((chunks, frames, classes))).astype(np.float32)
    np.put_along_axis(logits, labels[..., None].astype(np.int64),
                      np.take_along_axis(logits, labels[..., None].astype(np.int64), 2) + np.float32(margin), 2)
    truth = dict(turns=turns, chunk_offsets=offsets, frame_duration=frame_duration, total_samples=total_samples,
                 slot_speaker=slot_speaker, labels=labels)
    return logits, truth


SORTFORMER_MODES = ("turns", "quantized", "silence", "never_silent")


def sortformer_chunk(rng: np.random.Generator, mode: str, spkcache_length: int, fifo_length: int, core: int, lc: int,
                     rc: int) -> tuple[np.ndarray, np.ndarray]:
    """One Sortformer model output for a session holding ``spkcache_length`` + ``fifo_length`` state rows: (chunk
    embeddings [lc + core + rc x 512], probabilities [spkcache + fifo + lc + core + rc x 4]), every row drawn afresh
    (the model re-predicts the cache and FIFO rows each call).

    ``turns``: speakers take turns with silence, single-speaker and overlapped stretches; ``quantized``: the same on a
    1/8 grid (exact ties, exact 0.25 / 0.5 / 0.75); ``silence``: every frame's probabilities sum below 0.2;
    ``never_silent``: some speaker is above 0.5 in every frame."""
    rows = spkcache_length + fifo_length + lc + core + rc
    emb = rng.normal(0.0, 1.0, size=(lc + core + rc, 512)).astype(np.float32)
    if mode == "silence":
        return emb, rng.uniform(0.0, 0.045, size=(rows, 4)).astype(np.float32)
    state = rng.integers(0, 4, size=rows)   # 0 silence, 1 single speaker, 2 overlap, 3 single speaker (longer turns)
    state = np.repeat(state[::3], 3)[:rows] if rows else state
    who = np.repeat(rng.integers(0, 4, size=(rows + 4) // 4), 4)[:rows]
    other = (who + 1 + rng.integers(0, 3, size=rows)) % 4
    p = rng.uniform(0.0, 0.3, size=(rows, 4))
    speak = state > 0
    if mode == "never_silent":
        speak[:] = True
    idx = np.arange(rows)
    p[~speak] = rng.uniform(0.0, 0.05, size=(int((~speak).sum()), 4))
    p[idx[speak], who[speak]] = rng.uniform(0.55, 1.0, size=int(speak.sum()))
    both = state == 2
    p[idx[both], other[both]] = rng.uniform(0.5, 0.95, size=int(both.sum()))
    if mode == "quantized":
        p = np.round(p * 8.0) / 8.0
        emb = np.round(emb * 4.0) / 4.0
    return emb, p.astype(np.float32)
