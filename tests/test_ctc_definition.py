"""The CTC oracles against CTC from its definition (tests/ctc_definition.py), on the CPU.

The kernels equal the oracles bit for bit elsewhere; these tests ask whether the oracles compute what CTC means: the
unpruned beam search's best prefix is the most probable labelling and its score that labelling's log-probability (plus
the LM terms) within a float32 bar derived from the operations; a pruned search never scores a prefix above its
log-probability by more than the bar; a CTC-WS score is the best alignment of the term, exactly; log-softmax and the
chunk merge are their float64 formulas within derived bars.  Inputs include peaky log-softmax rows like a model's."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import ctc_cases  # noqa: E402
import ctc_decode_cases as cases  # noqa: E402
import ctc_definition as D  # noqa: E402
from oracle import oracle_ctc as OC  # noqa: E402
from oracle import oracle_ctc_decode as O  # noqa: E402

W = D.WILDCARD
# (token columns, frame counts) where a beam of 128 keeps every prefix: 1 + n + ... + n^T <= 128
UNPRUNED = [(1, [1, 2, 5, 40, 127]), (2, [1, 3, 6]), (3, [2, 4]), (10, [1, 2])]
KINDS = ["peaky", "normal", "ties", "constant", "neginf"]


def clip(rng, T, V, kind, blank):
    return cases.peaky(rng, T, V, float(rng.uniform(3, 12)), blank) if kind == "peaky" else cases.rows(rng, T, V, kind)


def lm_arrays(lm):
    return O.LmArrays(*lm) if lm is not None else None


def unpruned_cases(seed=0):
    """(name, log-probs, blank, pieces, lm) over the grid, blank inside and past the columns"""
    rng = np.random.default_rng(seed)
    out = []
    for n_tok, Ts in UNPRUNED:
        for T in Ts:
            for kind in KINDS:
                for blank_in in (True, False):
                    V = n_tok + 1 if blank_in else n_tok
                    blank = V - 1 if blank_in else V + 3
                    if kind == "peaky" and not blank_in and n_tok == 1:
                        kind = "normal"
                    lp = clip(rng, T, V, kind, blank)
                    voc = cases.vocabulary(rng, V, letters="abcd", missing=0.0)
                    pieces = cases.pieces(voc, V)
                    for with_lm in (False, True):
                        lm = cases.synthetic_lm(rng, words=60, bigrams=200, letters="abcd", max_len=3) if with_lm else None
                        out.append((f"n{n_tok}-T{T}-{kind}-{'b' if blank_in else 'nob'}-{'lm' if with_lm else 'ac'}",
                                    lp, blank, pieces, lm))
    return out


def check_unpruned(name, lp, blank, pieces, lm, ids, score, weight=0.3, bonus=0.5):
    """asserts the definition's properties of one unpruned search result; returns (set aside, fraction of the bar)"""
    best, f_best, f_second = D.best_labelling(lp, blank, pieces, lm, weight, bonus)
    G = D.suffix_gain(lp)
    lp_ids = D.log_p(ids, lp, blank)[0]
    want = lp_ids + D.lm_terms(ids, pieces, lm, weight, bonus)[0]
    bar = D.decode_bar(ids, lp, blank, max(abs(lp_ids), abs(float(score))) if np.isfinite(score) else lp_ids, pieces,
                       lm, weight, bonus, G)
    if not np.isfinite(want):
        assert score == -np.inf and not np.isfinite(f_best), name
        return False, 0.0
    assert abs(float(score) - want) <= bar, (name, ids, float(score), want, bar)
    margin = f_best - f_second
    bar_best = D.decode_bar(best, lp, blank, f_best, pieces, lm, weight, bonus, G)
    if margin <= 2 * bar_best + 2 * bar:
        return True, abs(float(score) - want) / bar
    assert ids == best, (name, ids, best, float(score), f_best, f_second)
    return False, abs(float(score) - want) / bar


def test_unpruned_beam_search_is_the_most_probable_labelling():
    """B = 128 and K = every token column keep every prefix, so the best prefix is the argmax over all labellings"""
    aside, worst, n = 0, 0.0, 0
    for name, lp, blank, pieces, lm in unpruned_cases():
        V = lp.shape[1]
        K = V - (1 if 0 <= blank < V else 0)
        ids, score = O.beam_search(lp, pieces, lm_arrays(lm), 128, 0.3, 0.5, blank, K)
        a, frac = check_unpruned(name, lp, blank, pieces, lm, ids, score)
        aside += a
        worst = max(worst, frac)
        n += 1
    print(f"\nunpruned: {n} cases, {aside} near-ties set aside, worst |score - objective| = {worst:.3g} of the bar")
    assert aside < n // 4


@pytest.mark.parametrize("B,K", [(1, 1), (4, 2), (16, 5), (64, 40)])
def test_pruned_beam_search_never_beats_the_labellings_probability(B, K):
    """pruning only removes alignments, and a prefix re-made after a prune only carries later ones"""
    rng = np.random.default_rng(B * 7 + K)
    V = 33
    voc = cases.vocabulary(rng, V)
    pieces = cases.pieces(voc, V)
    lm = cases.synthetic_lm(rng, words=300, bigrams=1500)
    worst = 0.0
    for i, (T, kind) in enumerate([(300, "peaky"), (1000, "peaky"), (60, "normal"), (40, "ties"), (50, "neginf")]):
        for use_lm in (False, True):
            lp = clip(rng, T, V, kind, V - 1)
            the_lm = lm if use_lm else None
            ids, score = O.beam_search(lp, pieces, lm_arrays(the_lm), B, 0.3, 0.5, V - 1, K)
            lp_ids = D.log_p(ids, lp, V - 1)[0]
            ac = float(score) - D.lm_terms(ids, pieces, the_lm, 0.3, 0.5)[0]
            bar = D.decode_bar(ids, lp, V - 1, max(abs(lp_ids), abs(float(score))), pieces, the_lm, 0.3, 0.5)
            assert ac <= lp_ids + bar, (T, kind, use_lm, ac, lp_ids, bar)
            worst = max(worst, (ac - lp_ids) / bar)
    print(f"\npruned B={B} K={K}: worst (score - log_p(ids)) = {worst:.3g} of the bar")


# ---- CTC-WS ---------------------------------------------------------------------------------------------------------
TERMS = [[2], [2, 3], [3, 3], [2, 2, 3], [W, 2], [2, W], [W, W, 3], [2, W, W], [W, 2, W], [W], [9, 1], [1, -5],
         [4, 4, 4], [W, 3, 3]]


def ws_clips(seed=0):
    rng = np.random.default_rng(seed)
    V = 6
    out = []
    for T in (1, 2, 3, 6, 10):
        for kind in ("random", "constant", "coarse", "neginf", "peaky"):
            for blank in (V - 1, 1024):
                lp = (cases.peaky(rng, T, V, 6.0, blank) if kind == "peaky" else ctc_cases.log_probs(rng, T, V, kind))
                out.append((f"T{T}-{kind}-b{blank}", lp, blank))
    return out


def windows(T):
    return [(a, b) for a in range(-1, T + 1) for b in range(a, T + 2)]


def check_window(name, lp, tok, blank, a, b, got):
    score, start, end, unique = D.ctcws_best(lp, tok, blank, a, b)
    s, gs, ge = got
    assert np.float32(s).view(np.uint32) == np.float32(score).view(np.uint32), (name, tok, a, b, s, score)
    if unique:
        assert (gs, ge) == (start, end), (name, tok, a, b, (gs, ge), (start, end))
    return unique


def test_ctcws_constrained_is_the_best_alignment():
    n = fixed = 0
    for name, lp, blank in ws_clips():
        for tok in TERMS:
            for a, b in windows(lp.shape[0]):
                fixed += check_window(name, lp, tok, blank, a, b, OC.word_spot_constrained(lp, tok, a, b, blank))
                n += 1
    print(f"\nCTC-WS constrained: {n} windows, {fixed} with a unique best alignment (frames compared)")


def check_detections(name, lp, tok, blank, det):
    """each detection's score is dp[t][N] / norm at some end frame t, by brute force"""
    ends = D.ctcws_end_values(lp, tok, blank)
    values = {np.float32(v[0]).view(np.uint32) for t, v in ends.items() if t >= len(tok)}
    for s, a, e in det:
        assert np.float32(s).view(np.uint32) in values, (name, tok, s, a, e)


def test_ctcws_detections_are_best_alignments():
    for name, lp, blank in ws_clips(1):
        for tok in TERMS:
            check_detections(name, lp, tok, blank, OC.word_spot_multiple(lp, tok, -np.inf, blank))


# ---- log-softmax and the chunk merge --------------------------------------------------------------------------------
@pytest.mark.parametrize("temperature", [0.7, 1.0, 1.3])
@pytest.mark.parametrize("V", [2, 33, 1025])
def test_log_softmax_is_the_formula(temperature, V):
    rng = np.random.default_rng(V)
    for x in (rng.normal(0, 5, size=(64, V)), np.log(np.exp(rng.normal(0, 1, size=(64, V))) + 1e-3) * 4,
              cases.peaky(rng, 64, V, 12.0) * 3):
        x = x.astype(np.float32)
        for bias in (0.0, 0.5):
            want, bar = D.log_softmax(x, temperature, bias, V - 1)
            got = OC.log_softmax(x, temperature, bias, V - 1).astype(np.float64)
            assert (np.abs(got - want) <= bar).all(), np.max(np.abs(got - want) / bar)


def test_merge_overlap_is_the_formula():
    rng = np.random.default_rng(5)
    a = cases.peaky(rng, 40, 33, 9.0)
    b = cases.peaky(rng, 40, 33, 9.0)
    b[3, :5] = -np.inf
    a[3, :3] = -np.inf
    got = OC.merge_chunks([a, b], 40)
    want, bar = D.merge_overlap(a, b)
    fin = np.isfinite(want)
    assert (np.isneginf(got) == ~fin).all()
    assert (np.abs(got[fin] - want[fin]) <= bar[fin]).all()
