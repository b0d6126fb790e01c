"""CTC decoding and keyword spotting on the H100 against CTC from its definition (tests/ctc_definition.py).

Every case is also compared bit for bit with the oracle, so a failure says which side moved.  The unpruned grid goes
through ``fa_ctc_beam_search`` and its device variant with and without an LM; pruned searches at the limits of beam
width and candidate count run on peaky rows, 257 clips per call and single clips of 20 000 and 45 000 frames, and print
the worst (score - log_p(ids)) as a fraction of the bar and how often greedy ids differ from the beam's; raw logits go
through ``fa_ctc_log_softmax_device`` into ``fa_ctc_beam_search_device``; ``fa_ctc_spot_constrained`` answers every
window of short clips and ``fa_ctc_spot``'s detections are best alignments."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import ctc_decode_cases as cases  # noqa: E402
import ctc_definition as D  # noqa: E402
import test_ctc_definition as T  # noqa: E402
from oracle import oracle_ctc as OC  # noqa: E402
from oracle import oracle_ctc_decode as O  # noqa: E402

pytestmark = pytest.mark.gpu


def bits(x):
    return np.float32(x).view(np.uint32)


@pytest.fixture(scope="module")
def dec_mod(gpu_lib):
    from fluidaudio_b200 import ctc_decoding
    return ctc_decoding


def gpu_lm(dec_mod, lm):
    if lm is None:
        return None
    uni, bi = lm
    m = dec_mod.ARPALanguageModel()
    m.unigrams = {w: dec_mod.ARPALanguageModel.Entry(*e) for w, e in uni.items()}
    m.bigrams = {c: {w: dec_mod.ARPALanguageModel.Entry(p, np.float32(0)) for w, p in r.items()} for c, r in bi.items()}
    return m


def run_beam(dec_mod, clips, V, blank, pieces, lm, B, K, w=0.3, bonus=0.5, device=False):
    """(ids, scores) per clip from the GPU"""
    from fluidaudio_b200 import _lib
    voc = {v: p for v, p in enumerate(pieces) if p is not None}
    dec = dec_mod.CtcDecoder(voc, V, blank)
    try:
        if not device:
            ids, scores, _ = dec.beam_search(clips, gpu_lm(dec_mod, lm), B, w, bonus, K)
            return ids, list(scores)
        lp, off = dec_mod._clips(clips, V)
        cap = max(1, int(off[-1]))
        d_lp, d_tok = _lib.DeviceBuffer(max(4, lp.nbytes)), _lib.DeviceBuffer(4 * cap)
        d_lp.upload(lp)
        st, lengths, scores, total = dec.beam_search_device(d_lp, off, d_tok, cap, gpu_lm(dec_mod, lm), B, w, bonus, K)
        assert st == 0
        return dec_mod._split(d_tok.download(cap, np.int32), lengths), list(scores)
    finally:
        dec.close()


def test_unpruned_grid_on_the_gpu(dec_mod):
    aside = n = 0
    worst = 0.0
    for name, lp, blank, pieces, lm in T.unpruned_cases(1):
        V = lp.shape[1]
        K = V - (1 if 0 <= blank < V else 0)
        want = O.beam_search(lp, pieces, T.lm_arrays(lm), 128, 0.3, 0.5, blank, K)
        for device in (False, True):
            ids, scores = run_beam(dec_mod, [lp], V, blank, pieces, lm, 128, K, device=device)
            assert ids[0] == want[0] and bits(scores[0]) == bits(want[1]), (name, device)
        a, frac = T.check_unpruned(name, lp, blank, pieces, lm, ids[0], scores[0])
        aside += a
        worst = max(worst, frac)
        n += 1
    print(f"\nGPU unpruned: {n} cases, {aside} near-ties set aside, worst |score - objective| = {worst:.3g} of the bar")
    assert aside < n // 4


def pruned_report(label, clips, V, blank, pieces, lm, ids, scores):
    worst, greedy_differs = -np.inf, 0
    for lp, got, s in zip(clips, ids, scores):
        lp_ids = D.log_p(got, lp, blank)[0]
        ac = float(s) - D.lm_terms(got, pieces, lm, 0.3, 0.5)[0]
        bar = D.decode_bar(got, lp, blank, max(abs(lp_ids), abs(float(s))), pieces, lm, 0.3, 0.5)
        assert ac <= lp_ids + bar, (label, len(lp), ac, lp_ids, bar)
        worst = max(worst, (ac - lp_ids) / bar)
        greedy_differs += O.greedy(lp, blank) != got
    print(f"\n{label}: {len(clips)} clips, worst (score - log_p(ids)) = {worst:.3g} of the bar, "
          f"greedy ids differ from the beam's in {greedy_differs}")


@pytest.mark.parametrize("B", [1, 64, 128])
@pytest.mark.parametrize("K", [1, 40, 64])
def test_pruned_limits_on_peaky_rows(dec_mod, B, K):
    rng = np.random.default_rng(B * 1000 + K)
    V = 129
    blank = V - 1
    voc = cases.vocabulary(rng, V)
    pieces = cases.pieces(voc, V)
    lm = cases.synthetic_lm(rng, words=400, bigrams=2000)
    clips = [cases.peaky(rng, int(n), V, float(rng.uniform(4, 12))) for n in rng.integers(0, 60, size=257)]
    ids, scores = run_beam(dec_mod, clips, V, blank, pieces, lm, B, K)
    for c, got, s in zip(clips, ids, scores):
        want = O.beam_search(c, pieces, T.lm_arrays(lm), B, 0.3, 0.5, blank, K)
        assert got == want[0] and bits(s) == bits(want[1])
    pruned_report(f"B={B} K={K} 257 clips, LM", clips, V, blank, pieces, lm, ids, scores)


@pytest.mark.parametrize("frames", [20000, 45000])
@pytest.mark.parametrize("B,K", [(1, 1), (128, 64)])
def test_pruned_long_clips(dec_mod, frames, B, K):
    """the host oracle needs minutes for one such clip at B = 128, K = 64, so there the device variant is held to the
    host variant's bits and both to the definition; at B = K = 1 also to the oracle's"""
    rng = np.random.default_rng(frames + B)
    V = 129
    blank = V - 1
    pieces = cases.pieces(cases.vocabulary(rng, V), V)
    lp = cases.peaky(rng, frames, V, 6.0)
    ids, scores = run_beam(dec_mod, [lp], V, blank, pieces, None, B, K)
    d_ids, d_scores = run_beam(dec_mod, [lp], V, blank, pieces, None, B, K, device=True)
    assert d_ids == ids and bits(d_scores[0]) == bits(scores[0])
    if B == 1:
        want = O.beam_search(lp, pieces, None, B, 0.3, 0.5, blank, K)
        assert ids[0] == want[0] and bits(scores[0]) == bits(want[1])
    pruned_report(f"{frames} frames B={B} K={K}", [lp], V, blank, pieces, None, ids, scores)


@pytest.mark.parametrize("temperature", [0.7, 1.0, 1.3])
def test_log_softmax_into_beam_search_on_the_device(dec_mod, temperature):
    from fluidaudio_b200 import _lib
    rng = np.random.default_rng(int(temperature * 10))
    V = 65
    blank = V - 1
    pieces = cases.pieces(cases.vocabulary(rng, V), V)
    lengths = [300, 0, 57, 1000]
    logits = [np.log(np.exp(cases.peaky(rng, n, V, 7.0).astype(np.float64)) + 1e-9).astype(np.float32) * 3
              for n in lengths]
    flat = np.ascontiguousarray(np.concatenate(logits), np.float32)
    rows = flat.shape[0]
    d_in, d_lp = _lib.DeviceBuffer(flat.nbytes), _lib.DeviceBuffer(flat.nbytes)
    d_in.upload(flat)
    _lib.check(_lib.load().fa_ctc_log_softmax_device(d_in.ptr, rows, V, 0, temperature, 0.0, blank, d_lp.ptr),
               "fa_ctc_log_softmax_device")
    lp_all = OC.log_softmax(flat, temperature, 0.0, blank)
    want_lp, bar = D.log_softmax(flat, temperature, 0.0, blank)
    assert (np.abs(lp_all.astype(np.float64) - want_lp) <= bar).all()
    off = np.concatenate([[0], np.cumsum(lengths)]).astype(np.int64)
    dec = dec_mod.CtcDecoder({v: p for v, p in enumerate(pieces) if p is not None}, V, blank)
    try:
        d_tok = _lib.DeviceBuffer(4 * rows)
        st, lens, scores, total = dec.beam_search_device(d_lp, off, d_tok, rows, None, 64, 0.3, 0.5, 40)
        assert st == 0
        ids = dec_mod._split(d_tok.download(rows, np.int32), lens)
    finally:
        dec.close()
    assert d_lp.download(rows * V, np.float32).tobytes() == lp_all.reshape(-1).tobytes()
    clips = [lp_all[off[i]:off[i + 1]] for i in range(len(lengths))]
    for c, got, s in zip(clips, ids, scores):
        want = O.beam_search(c, pieces, None, 64, 0.3, 0.5, blank, 40)
        assert got == want[0] and bits(s) == bits(want[1])
    pruned_report(f"logits at temperature {temperature}", clips, V, blank, pieces, None, ids, scores)


def test_ctcws_every_window_on_the_gpu():
    from fluidaudio_b200 import ctc_spotting as S
    n = fixed = 0
    for name, lp, blank in T.ws_clips(2):
        Tn = lp.shape[0]
        win = T.windows(Tn)
        a = [w[0] for w in win]
        b = [w[1] for w in win]
        for tok in T.TERMS:
            score, start, end = S.word_spot_constrained(lp, [tok] * len(win), a, b, blank)
            for i, (x, y) in enumerate(win):
                want = OC.word_spot_constrained(lp, tok, x, y, blank)
                assert (bits(score[i]), int(start[i]), int(end[i])) == (bits(want[0]), want[1], want[2]), (name, tok, x, y)
                fixed += T.check_window(name, lp, tok, blank, x, y, (score[i], int(start[i]), int(end[i])))
                n += 1
    print(f"\nGPU CTC-WS constrained: {n} windows, {fixed} with a unique best alignment (frames compared)")


def test_ctcws_detections_on_the_gpu():
    from fluidaudio_b200 import ctc_spotting as S
    for name, lp, blank in T.ws_clips(3):
        if lp.shape[0] == 0:
            continue
        sp = S.CtcSpotter(lp.shape[1], T.TERMS, blank)
        try:
            counts, det = sp.spot([lp], float("-inf"))
        finally:
            sp.close()
        _, want = OC.spot([lp], T.TERMS, float("-inf"), blank)
        got = [(int(d["term"]), int(bits(d["score"])), int(d["start_frame"]), int(d["end_frame"])) for d in det]
        assert got == [(k, int(bits(s)), a, e) for _, k, s, a, e in want], name
        for k, tok in enumerate(T.TERMS):
            T.check_detections(name, lp, tok, blank, [(d["score"], d["start_frame"], d["end_frame"]) for d in det
                                                      if int(d["term"]) == k])
