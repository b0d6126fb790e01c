"""Shared inputs of the offline Sortformer tests (test infrastructure): a deterministic test model, the frame-count and
overlap edges, prediction sets that reach every branch of the stitcher's arithmetic, and a planted case whose windows
hold known permutations of one activity timeline."""
import numpy as np

WINDOW_OUT, SPEAKERS, MELS, WINDOW_MEL = 384, 4, 128, 3072
# mel-frame edges: 1, 30 s, a full window whose second window is all overlap, one past it, three windows
FRAME_EDGES = (1, 7, 8, 9, 3001, 3071, 3072, 3073, 5344, 5345, 6144)
HOUR = 360_001
OVERLAP_EDGES = (-5, 0, 1, 100, 383, 384, 10 ** 6)


def model(mel, mel_length):
    """A deterministic stand-in for the fused model: speaker_preds [384 x 4] from one window's (mel [128 x 3072],
    mel_length), or [B x 384 x 4] from a batch.  Uses both inputs, and columns outside the valid frames too."""
    mel = np.asarray(mel, np.float32)
    one = mel.ndim == 2
    m = mel[None] if one else mel
    ml = np.asarray(mel_length, np.int64).reshape(-1)
    x = m[:, [0, 37, 74, 127], ::8].transpose(0, 2, 1).astype(np.float64)   # [B x 384 x 4]
    out = np.abs(np.sin(x * 0.731 + ml[:, None, None] * 1e-3 + np.arange(4) * 0.5)).astype(np.float32)
    return out[0] if one else out


def mel_rows(rng, frames):
    """time-major log-mel-like rows [frames x 128]"""
    return (rng.normal(-4, 2, size=(int(frames), MELS))).astype(np.float32)


SPECIALS = np.array([np.nan, np.inf, -np.inf, 0.0, -0.0, 1e-45, -1e-45, 1e-39, 3e38, -3e38, 1.0, 0.5],
                    np.float32)


def adversarial_preds(rng, windows, kind):
    """speaker_preds [windows x 384 x 4] of one kind:
      random    uniform [0, 1)
      specials  NaN, ±inf, ±0, subnormals and huge values mixed into uniform values
      ties      columns that repeat exactly, so correlations and scores tie
      nan       every value NaN: every score NaN, identity must result
      binary    0 / 1 activity, many exact zeros (skipped frames) and tied scores
      subnormal sums of subnormals, so the average's multiply rounds"""
    shape = (int(windows), WINDOW_OUT, SPEAKERS)
    if kind == "random":
        return rng.random(shape, np.float32)
    if kind == "specials":
        p = rng.random(shape, np.float32)
        pick = rng.random(shape) < 0.3
        p[pick] = rng.choice(SPECIALS, size=int(pick.sum()))
        return p
    if kind == "ties":
        base = rng.choice(np.array([0.0, 0.25, 0.5, 1.0], np.float32), size=shape[:2] + (2,))
        return np.concatenate([base, base], axis=2)[:, :, rng.permutation(4)].astype(np.float32)
    if kind == "nan":
        return np.full(shape, np.nan, np.float32)
    if kind == "binary":
        return (rng.random(shape) < 0.4).astype(np.float32)
    if kind == "subnormal":
        return (rng.integers(0, 8, size=shape) * np.float32(1e-45)).astype(np.float32) * \
            np.where(rng.random(shape) < 0.5, np.float32(1), np.float32(-1))
    raise ValueError(kind)


KINDS = ("random", "specials", "ties", "nan", "binary", "subnormal")


def planted(rng, frames, overlap):
    """A ground-truth activity timeline [totalOut x 4] (one active speaker per frame, soft values; any 20 frames see
    every speaker) and, for each window of a file of `frames` mel frames, its rows with the columns permuted: window k's column perm_k[g]
    holds speaker g.  Returns (preds [windows x 384 x 4], perms [windows x 4], truth)."""
    from offline_sortformer_restated import plan, clamp_overlap
    windows, total = plan(frames, overlap)
    ov = clamp_overlap(overlap)
    hop = WINDOW_OUT - ov
    truth = np.zeros((total, SPEAKERS), np.float32)
    truth[np.arange(total), (np.arange(total) // 5) % SPEAKERS] = 0.9   # every speaker in any 20 frames
    truth[truth == 0] = 0.05
    preds = np.zeros((windows, WINDOW_OUT, SPEAKERS), np.float32)
    perms = np.zeros((windows, SPEAKERS), np.int32)
    for k in range(windows):
        perm = np.arange(SPEAKERS) if k == 0 else rng.permutation(SPEAKERS)
        perms[k] = perm
        rows = truth[k * hop:k * hop + WINDOW_OUT]
        preds[k, :rows.shape[0], perm] = rows.T
    return preds, perms, truth
