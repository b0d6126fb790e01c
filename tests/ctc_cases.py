"""Seeded CTC keyword-spotting cases that reach every rule of CtcDPAlgorithm (test infrastructure, shared by the CPU and
GPU tests): wildcards (adjacent, leading, all-wildcard), repeated tokens, out-of-range token and blank ids, T of N - 1,
N and N + 1, clamped and empty windows, constant matrices (ties everywhere), -inf log-probs, equal start frames in the
merge, the fallback, and thresholds down to -inf so that -FLT_MAX cells reach the output."""
from __future__ import annotations

import numpy as np

WILDCARD = -1
MIN_SCORES = (None, -15.0, -3.0, -3e38, float("-inf"), 0.5)


def log_probs(rng, T, V, kind="random"):
    """[T x V] float32 log-probs of one kind: random rows, a constant matrix, or peaky rows with -inf holes"""
    if kind == "constant":
        return np.full((T, V), -1.0, np.float32)
    x = rng.normal(0, 2, size=(T, V)).astype(np.float32)
    x -= np.log(np.exp(x.astype(np.float64)).sum(1, keepdims=True)).astype(np.float32)
    if kind == "coarse":   # few distinct values: equal scores and equal start frames
        x = np.round(x).astype(np.float32)
    if kind == "neginf":
        x[rng.uniform(size=x.shape) < 0.2] = -np.inf
    return x.astype(np.float32)


def windows(rng, T, n=6):
    out = [(0, T), (-5, T + 7), (T // 2, T // 2), (T, T + 3), (-10, -2), (3, 2)]
    out += [(int(a), int(a + rng.integers(0, T + 3))) for a in rng.integers(-3, T + 2, size=n)]
    return out


def cases(seed=0):
    """(name, log_probs, tokens, blank_id) tuples"""
    rng = np.random.default_rng(seed)
    out = []
    V = 7
    for T in (0, 1, 2, 3, 4, 5, 9, 24):
        for kind in ("random", "constant", "coarse", "neginf"):
            lp = log_probs(rng, T, V, kind)
            for toks in ([2, 3], [2, WILDCARD, WILDCARD, 3], [WILDCARD, 2, 3], [WILDCARD, WILDCARD], [2, 2, 3, 3],
                         [4, 9, 4], [-5, 1], [1], [3, 3, 3]):
                for blank in (V - 1, 1024):
                    out.append((f"T{T}-{kind}-{toks}-b{blank}", lp, toks, blank))
    # T of N - 1, N and N + 1 for longer terms
    for N in (4, 6):
        toks = [int(t) for t in rng.integers(0, V - 1, size=N)]
        for T in (N - 1, N, N + 1):
            out.append((f"edge-N{N}-T{T}", log_probs(rng, T, V), toks, V - 1))
    return out
