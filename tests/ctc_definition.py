"""CTC from its definition, in float64 with numpy (test infrastructure): the probability of a labelling as the sum over
its alignments, the most probable labelling by enumeration, the decoder's LM objective, and the CTC word-spotting score
as a maximum over explicitly enumerated alignments.  Written from the definitions, not from the decoders' recurrences,
so that a misreading the kernels and the oracles share shows up as a disagreement here.

Rounding bars.  The decoder's float32 arithmetic is `log_add_exp(a, b) = m + f_log(f_exp(a - m) + f_exp(b - m))` with
f_exp / f_log the correctly rounded (float)exp((double)x) / (float)log((double)x) of fa_float.cuh, plus one float32 add
per emission.  With u = 2^-24, one log_add_exp whose exact result is r is off by at most u * (|r| + 3) to first order:
the subtraction inside exp perturbs the smaller term by a relative u * |d| * e^d / (1 + e^d) <= 0.28 u, exp and the
add of 1 + e each round once (together <= 2 u relative on the sum, so <= 2 u absolute after the log), the log rounds
once on a value in [0, log 2] (<= 0.7 u), and the final add rounds once (u * |r|).  `LAE_ULPS` = 4 carries the
second-order terms.  A float32 add with exact result r is off by u * |r|.

An error made at one operation reaches a labelling's final log-probability scaled by the fraction of the final mass
that flows through that operation's value.  At each frame every alignment passes through one prefix's
`log_add_exp(pb, pnb)`, one emission add and at most one merge `log_add_exp`, and the values a frame's operations
produce carry disjoint sets of alignments.  An operation carrying the fraction f of the final mass F has
|r| <= |F| + G + log(1 / f), with G the sum over frames of max(0, log sum_v exp(lp[t, v])) (the most a suffix can add),
and sum f * log(1 / f) over a frame is at most log(S) for S trellis states.  Hence `decode_bar`."""
from __future__ import annotations

import itertools

import numpy as np

U = 2.0 ** -24
LAE_ULPS = 4.0
UNK = -23.026          # ARPALanguageModel.unkLogProb
BOUNDARY = "▁"    # SentencePiece word boundary
NEG_MAX = np.float32(-np.finfo(np.float32).max)
WILDCARD = -1


def _column(lp, v):
    T, V = lp.shape
    return lp[:, v].astype(np.float64) if 0 <= v < V else np.full(T, -np.inf)


def log_p(labels, lp, blank):
    """log P(labels | lp): the CTC forward algorithm over [blank, l1, blank, ..., lN, blank] in float64.  Returns
    (total, ends in blank, ends in non-blank) at the last frame; a blank outside [0, V) has log-prob -inf."""
    lp = np.asarray(lp)
    T = lp.shape[0]
    labels = [int(x) for x in labels]
    ext = [blank]
    for x in labels:
        ext += [x, blank]
    S = len(ext)
    em = np.stack([_column(lp, v) for v in ext], 1) if T else np.zeros((0, S))
    skip = np.zeros(S, bool)
    for s in range(2, S):
        skip[s] = ext[s] != blank and ext[s] != ext[s - 2]
    if T == 0:
        end_b = 0.0 if not labels else -np.inf
        return end_b, end_b, -np.inf
    a = np.full(S, -np.inf)
    a[0] = em[0, 0]
    if S > 1:
        a[1] = em[0, 1]
    with np.errstate(invalid="ignore"):
        for t in range(1, T):
            b = a.copy()
            b[1:] = np.logaddexp(b[1:], a[:-1])
            b[2:] = np.where(skip[2:], np.logaddexp(b[2:], a[:-2]), b[2:])
            a = b + em[t]
    end_b = a[-1]
    end_n = a[-2] if S > 1 else -np.inf
    return float(np.logaddexp(end_b, end_n)), float(end_b), float(end_n)


def all_labellings(V, blank, T):
    """every collapsed labelling T frames can emit: a repeat needs a blank frame between, and without a blank column
    every frame emits a token"""
    tokens = [v for v in range(V) if v != blank]
    has_blank = 0 <= blank < V
    out = []
    for n in range(0, T + 1):
        for seq in itertools.product(tokens, repeat=n):
            repeats = sum(seq[i] == seq[i - 1] for i in range(1, n))
            if has_blank:
                ok = n + repeats <= T
            else:
                ok = repeats == 0 and (n >= 1 or T == 0) and n <= T
            if ok:
                out.append(list(seq))
    return out


# ---- the LM objective ----------------------------------------------------------------------------------------------
def words_of(labels, pieces):
    """ctcBeamSearch's word split: a piece starting with U+2581 closes the partial word (when non-empty) and opens the
    next with its remainder; other pieces extend the partial word.  Returns the words in order, the trailing one last."""
    words, partial = [], ""
    for v in labels:
        pc = pieces[v] if 0 <= v < len(pieces) and pieces[v] is not None else ""
        if pc.startswith(BOUNDARY):
            if partial:
                words.append(partial)
            partial = pc[len(BOUNDARY):]
        else:
            partial += pc
    if partial:
        words.append(partial)
    return words


def lm_score(word, prev, unigrams, bigrams):
    """ARPALanguageModel.score in float64: the bigram when (prev, word) has one, else prev's backoff (0 without prev or
    when prev has no unigram) plus word's unigram log-prob (UNK when it has none)"""
    if prev is not None and prev in bigrams and word in bigrams[prev]:
        return float(bigrams[prev][word])
    backoff = float(unigrams[prev][1]) if prev is not None and prev in unigrams else 0.0
    return backoff + (float(unigrams[word][0]) if word in unigrams else UNK)


def lm_terms(labels, pieces, lm, weight, bonus):
    """(sum of weight * score + bonus over the labelling's words, first-order rounding bar of the decoder's float32
    accumulation of it); lm None: (0, 0)"""
    if lm is None:
        return 0.0, 0.0
    unigrams, bigrams = lm
    total, bar, prev = 0.0, 0.0, None
    for w in words_of(labels, pieces):
        s = lm_score(w, prev, unigrams, bigrams)
        d = weight * s + bonus
        total += d
        # backoff + log-prob, weight * score, + bonus, lm + delta: one rounding each
        bar += U * (abs(weight) * abs(s) + abs(weight * s) + abs(d) + abs(total))
        prev = w
    return total, bar


def objective(labels, lp, blank, pieces=None, lm=None, weight=0.3, bonus=0.0):
    """log_p(labels) + sum over its words of (weight * score + bonus)"""
    return log_p(labels, lp, blank)[0] + lm_terms(labels, pieces or [], lm, weight, bonus)[0]


def suffix_gain(lp):
    """G: the sum over frames of max(0, log sum_v exp(lp[t, v])), the most any stretch of frames can add"""
    lp = np.asarray(lp, np.float64)
    if lp.size == 0:
        return 0.0
    with np.errstate(divide="ignore"):
        m = np.logaddexp.reduce(lp, axis=1)
    return float(np.maximum(m, 0.0).sum())


def decode_bar(labels, lp, blank, F, pieces=None, lm=None, weight=0.3, bonus=0.0, G=None):
    """first-order bound on |float32 beam score - float64 objective| for the best prefix `labels` with acoustic
    log-probability of magnitude at most |F| (module docstring)"""
    T = np.asarray(lp).shape[0]
    G = suffix_gain(lp) if G is None else G
    F = abs(F) if np.isfinite(F) else 0.0
    states = 2 * len(labels) + 1
    per_frame = 3 * (F + G + np.log(states)) + 2 * LAE_ULPS
    lm_sum, lm_bar = lm_terms(labels, pieces or [], lm, weight, bonus)
    return U * (T * per_frame + F + LAE_ULPS + abs(F) + abs(lm_sum)) + lm_bar


def best_labelling(lp, blank, pieces=None, lm=None, weight=0.3, bonus=0.0):
    """(argmax labelling of the objective over all_labellings, its objective, runner-up's objective)"""
    lp = np.asarray(lp)
    T, V = lp.shape
    scored = [(objective(lab, lp, blank, pieces, lm, weight, bonus), lab) for lab in all_labellings(V, blank, T)]
    scored.sort(key=lambda x: -x[0])
    second = scored[1][0] if len(scored) > 1 else -np.inf
    return scored[0][1], scored[0][0], second


# ---- CTC word spotting ----------------------------------------------------------------------------------------------
def _graph(tokens, V, blank):
    """the expanded graph [B, t1, B, ..., tN, B]: per state its kind ('b', 't', 'w'), id, and whether a skip from two
    states back may enter it (CtcDPAlgorithm: never into a blank, not between equal token ids, not from a wildcard
    into a wildcard)"""
    kinds, ids = ["b"], [blank]
    for x in tokens:
        kinds += ["w" if x == WILDCARD else "t", "b"]
        ids += [x, blank]
    skip = [False] * len(kinds)
    for i in range(2, len(kinds)):
        if kinds[i] == "t":
            skip[i] = not (kinds[i - 2] == "t" and ids[i - 2] == ids[i])
        elif kinds[i] == "w":
            skip[i] = kinds[i - 2] != "w"
    return kinds, ids, skip


def _emission(kind, v, row, V, blank):
    """what a frame adds in a state: a blank's log-prob (0 for a blank id outside [0, V)), a token's (-FLT_MAX for an
    id outside [0, V)), 0 for a wildcard"""
    if kind == "b":
        return row[blank] if 0 <= blank < V else np.float32(0)
    if kind == "t":
        return row[v] if 0 <= v < V else NEG_MAX
    return np.float32(0)


_PATH_CACHE: dict = {}


def _paths(lp, tokens, blank):
    """every alignment of the term, as arrays over alignments: start frame, end (exclusive frame after the last),
    float32 value summed left to right, and the frame after the last token / wildcard frame (the reported end).
    An alignment starts in the leading blank at any frame (value 0) and advances one state, stays, or skips per frame.
    A partial sum at or below -FLT_MAX / 2 is clamped to -FLT_MAX instead of adding the next frame."""
    key = (lp.tobytes(), lp.shape, tuple(tokens), blank)
    if key in _PATH_CACHE:
        return _PATH_CACHE[key]
    T, V = lp.shape
    kinds, ids, skip = _graph(tokens, V, blank)
    L, N = len(kinds), len(tokens)
    rows = []
    half = NEG_MAX / np.float32(2)

    def walk(t, i, v, s0, last):
        # t frames consumed (absolute), in state i with value v
        if i >= 2 * N - 1:
            rows.append((s0, t, v, last))
        if t == T:
            return
        row = lp[t]
        for j in (i, i + 1, i + 2):
            if j >= L or j == 0 or (j == i + 2 and not skip[j]):
                continue
            if v <= half:
                nv = NEG_MAX
            else:
                with np.errstate(over="ignore"):
                    nv = np.float32(v + _emission(kinds[j], ids[j], row, V, blank))
            walk(t + 1, j, nv, s0, t + 1 if kinds[j] != "b" else last)

    for s0 in range(T):
        # from the leading blank (value 0 at every frame) the first move enters the first token's state
        if L > 1:
            row = lp[s0]
            nv = np.float32(np.float32(0) + _emission(kinds[1], ids[1], row, V, blank))
            walk(s0 + 1, 1, nv, s0, s0 + 1 if kinds[1] != "b" else s0)
    out = (np.array([r[0] for r in rows], np.int64), np.array([r[1] for r in rows], np.int64),
           np.array([r[2] for r in rows], np.float32), np.array([r[3] for r in rows], np.int64))
    _PATH_CACHE[key] = out
    if len(_PATH_CACHE) > 64:
        _PATH_CACHE.pop(next(iter(_PATH_CACHE)))
    return out


def ctcws_best(lp, tokens, blank, a, b):
    """ctcWordSpotConstrained's result by brute force: (score, start, end, unique) for the window [a, b) of frames.
    The score is max(-FLT_MAX, best alignment inside the window) over the non-wildcard count; start and end are the
    best alignment's and `unique` says whether exactly one alignment attains it (only then are the frames defined by
    the definition rather than by the recurrence's tie rules).  A window clamped to fewer frames than tokens scores
    -inf at its clamped start."""
    lp = np.asarray(lp, np.float32)
    T = lp.shape[0]
    tokens = [int(t) for t in tokens]
    N = len(tokens)
    cs, ce = max(0, a), min(T, b)
    if N == 0 or ce <= cs or ce - cs < N:
        return np.float32(-np.inf), cs, cs, True
    s0, te, val, last = _paths(lp, tokens, blank)
    inside = (s0 >= cs) & (te <= ce)
    nw = sum(t != WILDCARD for t in tokens)
    norm = np.float32(nw if nw > 0 else 1)
    if not inside.any():
        return NEG_MAX / norm if nw > 0 else NEG_MAX, cs, cs, False
    v = val[inside]
    best = v.max()
    if best <= NEG_MAX:
        return (NEG_MAX / norm if nw > 0 else NEG_MAX), cs, cs, False
    at = np.flatnonzero(v == best)
    k = at[0]
    score = np.float32(best / norm) if nw > 0 else best
    return score, int(s0[inside][k]), int(last[inside][k]), len(at) == 1


def ctcws_end_values(lp, tokens, blank):
    """per end frame t (1 .. T): the best alignment of the whole clip ending there over the non-wildcard count, with
    whether one alignment attains it and its start and reported end: dp[t][N] / norm by brute force"""
    lp = np.asarray(lp, np.float32)
    T = lp.shape[0]
    tokens = [int(t) for t in tokens]
    s0, te, val, last = _paths(lp, tokens, blank)
    nw = sum(t != WILDCARD for t in tokens)
    norm = np.float32(nw if nw > 0 else 1)
    out = {}
    for t in range(1, T + 1):
        m = te == t
        if not m.any():
            out[t] = (NEG_MAX / norm if nw > 0 else NEG_MAX, None, None, False)
            continue
        v = val[m]
        best = v.max()   # not clamped: an alignment through a -inf log-prob ends at -inf
        at = np.flatnonzero(v == best)
        out[t] = (np.float32(best / norm) if nw > 0 else best, int(s0[m][at[0]]), int(last[m][at[0]]), len(at) == 1)
    return out


# ---- log-softmax and the chunk merge --------------------------------------------------------------------------------
def log_softmax(logits, temperature=1.0, blank_bias=0.0, blank=None):
    """(float64 log-softmax of logits / temperature, minus blank_bias at the blank column; per-element bar of the
    float32 restatement: the division, the subtraction of the maximum, V float32 adds of correctly rounded exps, the
    log and the final subtraction)"""
    x = np.asarray(logits, np.float64)
    T, V = x.shape
    y = x / temperature if temperature != 1.0 else x
    m = y.max(1, keepdims=True)
    d = y - m
    lse = np.log(np.exp(d).sum(1, keepdims=True))
    out = d - lse
    p = np.exp(out)
    div = U * np.abs(y).max(1, keepdims=True) if temperature != 1.0 else 0.0
    # the division perturbs d_v and, through the softmax weights, lse; the sum of V exps rounds V times relative to it
    bar = (2 * div + U * np.abs(d) + U * (np.abs(d) * p).sum(1, keepdims=True) + U * (V + 2)
           + U * np.abs(lse) + U * np.abs(out))
    if blank_bias != 0.0 and blank is not None and 0 <= blank < V:
        out[:, blank] -= blank_bias
        bar[:, blank] += U * np.abs(out[:, blank])
    return out, bar


LN2_F32 = np.float32(0.69314718)


def merge_overlap(a, b):
    """(float64 log((e^a + e^b) / 2), bar of mergeOverlapFrame's float32 log_add_exp minus the float32 constant)"""
    a = np.asarray(a, np.float64)
    b = np.asarray(b, np.float64)
    with np.errstate(invalid="ignore"):
        r = np.logaddexp(a, b)
        out = r - np.log(2.0)
    fin = np.isfinite(r)
    bar = np.where(fin, U * (np.abs(r) + LAE_ULPS) + abs(float(LN2_F32) - np.log(2.0)) + U * np.abs(out), 0.0)
    return out, bar
