"""Pure-Python restatement of CTC keyword spotting (test infrastructure): applyLogSoftmax, mergeOverlapFrame and the
chunk concatenation (CtcKeywordSpotter.swift:268-306, +Inference.swift:96-126, :329-346) and CtcDPAlgorithm
(CtcDPAlgorithm.swift:121-392), every float operation a numpy float32 scalar operation and exp / log the double
functions rounded to float32.  It holds the C++ oracle (oracle/oracle_ctc.cpp) to the reference's description on small
cases; it is slow and written for clarity.
"""
from __future__ import annotations

import math

import numpy as np

F = np.float32
NEG = F(-np.finfo(np.float32).max)
WILDCARD = -1


def fexp(x):
    try:
        return F(math.exp(float(x)))
    except OverflowError:
        return F(np.inf)


def flog(x):
    x = float(x)
    if x == 0.0:
        return F(-np.inf)
    return F(math.log(x)) if x > 0 else F(np.nan)


def log_softmax(logits, temperature=1.0, blank_bias=0.0, blank_id=1024):
    temperature, blank_bias = F(temperature), F(blank_bias)
    out = []
    with np.errstate(all="ignore"):
        for row in np.asarray(logits, np.float32):
            x = [F(v) / temperature if temperature != F(1) else F(v) for v in row]
            m = x[0]
            for v in x[1:]:
                if m < v:
                    m = v
            s = F(0)
            for v in x:
                s = F(s + fexp(F(v - m)))
            lse = flog(s)
            r = [F(F(v - m) - lse) for v in x]
            if blank_bias != F(0) and blank_id < len(r):
                r[blank_id] = F(r[blank_id] - blank_bias)
            out.append(r)
    return np.array(out, np.float32).reshape(len(out), -1)


def merge_overlap_frame(a, b):
    out = []
    with np.errstate(all="ignore"):
        for x, y in zip(a, b):
            x, y = F(x), F(y)
            m = y if y >= x else x
            out.append(F(-np.inf) if m == F(-np.inf) else F(F(m + flog(F(fexp(F(x - m)) + fexp(F(y - m))))) -
                                                            F(0.69314718)))
    return out


def merge_chunks(chunks, overlap_frames):
    rows = []
    for idx, c in enumerate(chunks):
        c = [list(np.asarray(r, np.float32)) for r in c]
        if not c:
            continue
        if idx == 0:
            rows += c
            continue
        ov = min(overlap_frames, len(rows), len(c))
        start = len(rows) - ov
        for i in range(ov):
            rows[start + i] = merge_overlap_frame(rows[start + i], c[i])
        rows += c[ov:]
    return np.array(rows, np.float32).reshape(len(rows), -1) if rows else np.zeros((0, 0), np.float32)


def _emission(sym, frame, blank_id):
    kind, tok = sym
    V = len(frame)
    if kind == "blank":
        return F(frame[blank_id]) if 0 <= blank_id < V else F(0)
    if kind == "token":
        return F(frame[tok]) if 0 <= tok < V else NEG
    return F(0)


def _can_skip(s, i):
    if i < 2 or s[i][0] == "blank":
        return False
    if s[i][0] == "token":
        return not (s[i - 2][0] == "token" and s[i - 2][1] == s[i][1])
    return s[i - 2][0] != "wild"


def fill_dp_table(log_probs, tokens, blank_id):
    T, N = len(log_probs), len(tokens)
    dp = [[NEG] * (N + 1) for _ in range(T + 1)]
    back = [[0] * (N + 1) for _ in range(T + 1)]
    last = [[0] * (N + 1) for _ in range(T + 1)]
    for t in range(T + 1):
        dp[t][0] = F(0)
    if N == 0:
        return dp, back, last
    s = []
    for tok in tokens:
        s += [("blank", 0), ("wild", 0) if tok == WILDCARD else ("token", tok)]
    s.append(("blank", 0))
    L = len(s)
    d = [[NEG] * L for _ in range(T + 1)]
    st = [[0] * L for _ in range(T + 1)]
    lt = [[0] * L for _ in range(T + 1)]
    for t in range(T + 1):
        d[t][0], st[t][0] = F(0), t
    with np.errstate(all="ignore"):
        for t in range(1, T + 1):
            frame = log_probs[t - 1]
            for i in range(1, L):
                added = F(0) if s[i][0] == "wild" else _emission(s[i], frame, blank_id)
                stay, adv = d[t - 1][i], d[t - 1][i - 1]
                skip = d[t - 1][i - 2] if _can_skip(s, i) else NEG
                best, kind = stay, 0
                if adv > best:
                    best, kind = adv, 1
                if skip > best:
                    best, kind = skip, 2
                if best <= F(NEG / F(2)):
                    d[t][i] = NEG
                    continue
                d[t][i] = F(best + added)
                match = s[i][0] != "blank"
                src = i - kind
                st[t][i] = t - 1 if kind == 1 and i == 1 else st[t - 1][src]
                lt[t][i] = t if match else lt[t - 1][src]
    for t in range(T + 1):
        for n in range(1, N + 1):
            a, b = 2 * n - 1, 2 * n
            if d[t][a] >= d[t][b]:
                dp[t][n], back[t][n], last[t][n] = d[t][a], st[t][a], lt[t][a]
            else:
                dp[t][n], back[t][n], last[t][n] = d[t][b], st[t][b], lt[t][b]
    return dp, back, last


def non_wildcard_count(tokens):
    return sum(1 for t in tokens if t != WILDCARD)


def word_spot_constrained(log_probs, tokens, search_start, search_end, blank_id=1024):
    T, N = len(log_probs), len(tokens)
    cs, ce = max(0, search_start), min(T, search_end)
    if N == 0 or ce <= cs or ce - cs < N:
        return F(-np.inf), cs, cs
    dp, back, last = fill_dp_table(log_probs[cs:ce], tokens, blank_id)
    best_end, best = 0, NEG
    for t in range(N, ce - cs + 1):
        if dp[t][N] > best:
            best, best_end = dp[t][N], t
    k = non_wildcard_count(tokens)
    return (F(best / F(k)) if k > 0 else best), cs + back[best_end][N], cs + last[best_end][N]


def word_spot_multiple(log_probs, tokens, min_score=-15.0, blank_id=1024):
    T, N = len(log_probs), len(tokens)
    min_score = F(min_score)
    if N == 0 or T == 0:
        return []
    dp, back, last = fill_dp_table(log_probs, tokens, blank_id)
    k = non_wildcard_count(tokens)
    norm = F(k) if k > 0 else F(1)
    if T < N:
        return []
    with np.errstate(all="ignore"):
        cand = []
        for t in range(N, T + 1):
            s = F(dp[t][N] / norm)
            prev = F(dp[t - 1][N] / norm) if t > N else NEG
            nxt = F(dp[t + 1][N] / norm) if t < T else NEG
            if s >= prev and s > nxt and s >= min_score:
                cand.append((s, back[t][N], last[t][N]))
        if not cand:
            be, bs = 0, NEG
            for t in range(N, T + 1):
                s = F(dp[t][N] / norm)
                if s > bs:
                    bs, be = s, t
            if bs >= min_score:
                cand.append((bs, back[be][N], last[be][N]))
    merged = []
    for c in sorted(cand, key=lambda c: c[1]):   # Python's sort is stable
        if merged and c[1] <= merged[-1][2]:
            best = c if c[0] > merged[-1][0] else merged[-1]
            merged[-1] = (best[0], best[1], max(merged[-1][2], c[2]))
        else:
            merged.append(c)
    return merged


def threshold(min_score, n_tokens):
    if min_score is None:
        return F(-15)
    return F(F(min_score) - F(F(max(0, n_tokens - 3)) * F(1)))
