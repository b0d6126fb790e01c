"""A literal pure-Python restatement of ctcGreedyDecode, ctcBeamSearch, logAddExp and ARPALanguageModel.score
(CtcDecoder.swift, ARPALanguageModel.swift), independent of ``oracle/oracle_ctc_decode.cpp``: beams in a ``dict`` keyed
by the prefix tuple (insertion-ordered, as the contract fixes the reference's hash order), the prune a stable
``sorted(..., reverse=True)``, word pieces as lists of strings, float32 arithmetic through numpy, and exp / log the
correctly rounded float32 functions of ``tests/float_exact.py``, the library's definition."""
import numpy as np

import float_exact

F = np.float32
NEG_INF = F(-np.inf)
BOUNDARY = "▁"
UNK = F(-23.026)


f_exp = float_exact.exp
f_log = float_exact.log


def log_add_exp(a, b):
    a, b = F(a), F(b)
    if a == NEG_INF:
        return b
    if b == NEG_INF:
        return a
    m = b if b >= a else a   # Swift.max(a, b)
    return F(m + f_log(F(f_exp(F(a - m)) + f_exp(F(b - m)))))


def greedy(frames, blank_id):
    ids, prev = [], -1
    for frame in frames:
        if len(frame) == 0:
            continue
        best_idx, best_val = 0, frame[0]
        for v in range(1, len(frame)):
            if frame[v] > best_val:
                best_val, best_idx = frame[v], v
        if best_idx != blank_id and best_idx != prev:
            ids.append(best_idx)
        prev = best_idx
    return ids


class LM:
    """unigrams {word: (log_prob, backoff)}, bigrams {context: {word: log_prob}}"""

    def __init__(self, unigrams, bigrams):
        self.unigrams, self.bigrams = unigrams, bigrams

    def score(self, word, prev):
        if prev is not None and prev in self.bigrams and word in self.bigrams[prev]:
            return F(self.bigrams[prev][word])
        backoff = F(self.unigrams[prev][1]) if prev is not None and prev in self.unigrams else F(0.0)
        return F(backoff + (F(self.unigrams[word][0]) if word in self.unigrams else UNK))


class Beam:
    __slots__ = ("prefix", "p_blank", "p_non_blank", "lm_score", "word_pieces", "prev_word")

    def __init__(self, prefix, p_blank, p_non_blank, lm_score, word_pieces, prev_word):
        self.prefix, self.p_blank, self.p_non_blank = prefix, F(p_blank), F(p_non_blank)
        self.lm_score, self.word_pieces, self.prev_word = F(lm_score), word_pieces, prev_word

    def copy(self):
        return Beam(self.prefix, self.p_blank, self.p_non_blank, self.lm_score, list(self.word_pieces), self.prev_word)

    @property
    def total_acoustic(self):
        return log_add_exp(self.p_blank, self.p_non_blank)

    @property
    def total(self):
        return F(self.total_acoustic + self.lm_score)


def beam_search(frames, vocabulary, lm=None, beam_width=100, lm_weight=0.3, word_bonus=0.0, blank_id=1024,
                token_candidates=40, stats=None):
    """(ids, total) of the best prefix; `stats`, a dict, receives "recreated": the extensions that re-made a prefix
    that had been made before, was pruned, and has a child among the frame's beams"""
    lm_weight, word_bonus = F(lm_weight), F(word_bonus)
    if len(frames) == 0:
        return [], F(0.0)
    V = len(frames[0])
    if V == 0:
        return [], F(0.0)
    beams = {(): Beam((), 0.0, NEG_INF, 0.0, [], None)}
    made = {()}
    recreated = 0
    for frame in frames:
        frame = [F(x) for x in frame]
        blank_lp = frame[blank_id] if 0 <= blank_id < V else NEG_INF
        top = sorted((v for v in range(V) if v != blank_id), key=lambda v: frame[v], reverse=True)[:token_candidates]
        parents = {b.prefix[:-1] for b in beams.values() if b.prefix}
        new_beams = {}

        def merge(beam):
            k = beam.prefix
            if k in new_beams:
                e = new_beams[k]
                e.p_blank = log_add_exp(e.p_blank, beam.p_blank)
                e.p_non_blank = log_add_exp(e.p_non_blank, beam.p_non_blank)
            else:
                new_beams[k] = beam

        for beam in list(beams.values()):
            prev_total = beam.total_acoustic
            blank_beam = beam.copy()
            blank_beam.p_blank = F(prev_total + blank_lp)
            blank_beam.p_non_blank = NEG_INF
            merge(blank_beam)
            for v in top:
                token_lp = frame[v]
                is_repeat = bool(beam.prefix) and beam.prefix[-1] == v
                piece = vocabulary.get(v, "")
                new_pieces, new_prev, delta = list(beam.word_pieces), beam.prev_word, F(0.0)
                if lm is not None and piece.startswith(BOUNDARY):
                    completed = "".join(new_pieces)
                    has = completed != ""
                    delta = F(F(lm_weight * lm.score(completed, new_prev)) + word_bonus) if has else F(0.0)
                    new_prev = completed if has else new_prev
                    stripped = piece[1:]
                    new_pieces = [] if stripped == "" else [stripped]
                elif lm is not None:
                    new_pieces.append(piece)
                child = beam.prefix + (v,)
                if child in made and child not in beams and child in parents:
                    recreated += 1
                made.add(child)
                if is_repeat:
                    same = beam.copy()
                    same.p_blank = NEG_INF
                    same.p_non_blank = F(beam.p_non_blank + token_lp)
                    merge(same)
                    merge(Beam(child, NEG_INF, F(beam.p_blank + token_lp), F(beam.lm_score + delta), new_pieces,
                               new_prev))
                else:
                    merge(Beam(child, NEG_INF, F(prev_total + token_lp), F(beam.lm_score + delta), new_pieces,
                               new_prev))
        ranked = sorted(new_beams.values(), key=lambda b: b.total, reverse=True)
        beams = {b.prefix: b for b in ranked[:beam_width]}
    finals = []
    for beam in beams.values():
        b = beam.copy()
        last = "".join(b.word_pieces)
        if lm is not None and last != "":
            b.lm_score = F(b.lm_score + F(F(lm_weight * lm.score(last, b.prev_word)) + word_bonus))
        finals.append(b)
    if stats is not None:
        stats["recreated"] = recreated
    if not finals:
        return [], NEG_INF
    best = finals[0]
    for b in finals[1:]:
        if best.total < b.total:
            best = b
    return list(best.prefix), best.total
