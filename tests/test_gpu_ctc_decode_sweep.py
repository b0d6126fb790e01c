"""CTC decoding on the H100 (``fa_ctc_greedy``, ``fa_ctc_beam_search``): ids and lengths exact and score bits equal to
the oracle (``oracle/oracle_ctc_decode.cpp``) across clip counts, frame counts, vocabulary sizes, beam widths and
candidate counts, with and without a synthetic bigram LM, through both variants; plus a short capacity, the NaN / +inf
refusal, launch counts and the reference's decoder tests through the GPU."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import ctc_decode_cases as cases  # noqa: E402
from oracle import oracle_ctc_decode as O  # noqa: E402

pytestmark = pytest.mark.gpu


def bits(x):
    return np.float32(x).view(np.uint32)


@pytest.fixture(scope="module")
def D(gpu_lib):
    from fluidaudio_b200 import ctc_decoding
    return ctc_decoding


def _lm_pair(D, rng, **kw):
    uni, bi = cases.synthetic_lm(rng, **kw)
    lm = D.ARPALanguageModel()
    lm.unigrams = {w: D.ARPALanguageModel.Entry(*e) for w, e in uni.items()}
    lm.bigrams = {c: {w: D.ARPALanguageModel.Entry(p, np.float32(0)) for w, p in r.items()} for c, r in bi.items()}
    return lm, O.LmArrays(uni, bi)


def _greedy_device(D, clips, V, blank):
    from fluidaudio_b200 import _lib
    lp, off = D._clips(clips, V)
    B = len(clips)
    d_lp, d_tok = _lib.DeviceBuffer(max(4, lp.nbytes)), _lib.DeviceBuffer(4 * max(1, int(off[-1])))
    d_lp.upload(lp)
    lengths, total = np.zeros(max(B, 1), np.int64), C.c_int64()
    _lib.check(_lib.load().fa_ctc_greedy_device(d_lp.ptr, _lib.ptr(off), B, V, blank, _lib.ptr(lengths), d_tok.ptr,
                                                max(1, int(off[-1])), C.byref(total)), "fa_ctc_greedy_device")
    tok = d_tok.download(max(1, int(off[-1])), np.int32)
    return D._split(tok, lengths[:B])


@pytest.mark.parametrize("V", [2, 33, 1025])
@pytest.mark.parametrize("n_clips", [1, 3, 257])
def test_greedy_equals_the_oracle(D, V, n_clips):
    rng = np.random.default_rng(V * 1000 + n_clips)
    lens = [0, 1, 20000] if n_clips == 3 else ([5000] if n_clips == 1 else list(rng.integers(0, 200, size=n_clips)))
    kinds = ["normal", "ties", "constant", "neginf"]
    clips = [cases.rows(rng, int(T), V, kinds[i % 4]) for i, T in enumerate(lens)]
    for c in clips[: max(1, n_clips // 2)]:
        if len(c):
            c[rng.integers(len(c), size=max(1, len(c) // 10)), 0] = np.nan                   # NaN in column 0 wins
            c[rng.integers(len(c), size=max(1, len(c) // 10)), rng.integers(V)] = np.nan     # elsewhere it never does
    for blank in (V - 1, V + 3):
        want = [O.greedy(c, blank) for c in clips]
        assert D.greedy_ids(clips, V, blank) == want
        assert _greedy_device(D, clips, V, blank) == want


def _check_beam(D, clips, V, blank, voc, lm_pair, B, K, w=0.3, bonus=0.0):
    lm, arrays = lm_pair if lm_pair else (None, None)
    dec = D.CtcDecoder(voc, V, blank)
    try:
        ids, scores, _ = dec.beam_search(clips, lm, B, w, bonus, K)
    finally:
        dec.close()
    for c, got, s in zip(clips, ids, scores):
        want, ws = O.beam_search(c, cases.pieces(voc, V), arrays, B, w, bonus, blank, K)
        assert got == want and bits(s) == bits(ws), (B, K, len(c))


@pytest.mark.parametrize("B", [1, 2, 10, 100, 128])
@pytest.mark.parametrize("K", [1, 5, 40, 64, 1000])
def test_beam_without_lm_equals_the_oracle(D, B, K):
    rng = np.random.default_rng(B * 131 + K)
    V = 65 if K != 1000 else 33
    voc = cases.vocabulary(rng, V)
    clips = [cases.rows(rng, int(T), V, kind) for T, kind in
             zip([0, 1, 40, 73, 25], ["normal", "ties", "normal", "neginf", "constant"])]
    _check_beam(D, clips, V, V - 1, voc, None, B, K)


@pytest.mark.parametrize("B,K", [(1, 1), (10, 5), (100, 40), (128, 64)])
def test_beam_with_lm_equals_the_oracle(D, B, K):
    rng = np.random.default_rng(7 + B)
    V = 1025
    voc = cases.vocabulary(rng, V)
    pair = _lm_pair(D, rng, words=20000, bigrams=100000, max_len=5)
    clips = [cases.rows(rng, int(T), V, kind) for T, kind in zip([60, 1, 0, 45], ["normal", "ties", "normal", "neginf"])]
    _check_beam(D, clips, V, V - 1, voc, pair, B, K)
    _check_beam(D, clips[:1], V, V + 5, voc, pair, B, K, w=0.0, bonus=1.5)


def test_many_clips_and_a_long_clip(D):
    rng = np.random.default_rng(11)
    V = 33
    voc = cases.vocabulary(rng, V)
    pair = _lm_pair(D, rng, words=300, bigrams=1500)
    clips = [cases.rows(rng, int(T), V, "ties") for T in rng.integers(0, 30, size=257)]
    _check_beam(D, clips, V, 32, voc, pair, 10, 5)
    _check_beam(D, [cases.rows(rng, 20000, V, "normal")], V, 32, voc, pair, 4, 3)


def test_device_variant_and_a_short_capacity(D):
    from fluidaudio_b200 import _lib
    rng = np.random.default_rng(12)
    V = 33
    voc = cases.vocabulary(rng, V)
    lm, arrays = _lm_pair(D, rng, words=300, bigrams=1500)
    clips = [cases.rows(rng, T, V, "normal") for T in (50, 0, 31)]
    want = [O.beam_search(c, cases.pieces(voc, V), arrays, 16, 0.3, 0.5, 32, 8) for c in clips]
    lp, off = D._clips(clips, V)
    d_lp, d_tok = _lib.DeviceBuffer(lp.nbytes), _lib.DeviceBuffer(4 * 200)
    d_lp.upload(lp)
    dec = D.CtcDecoder(voc, V, 32)
    st, lengths, scores, total = dec.beam_search_device(d_lp, off, d_tok, 200, lm, 16, 0.3, 0.5, 8)
    assert st == 0 and total == sum(len(w[0]) for w in want)
    got = D._split(d_tok.download(200, np.int32), lengths)
    assert got == [w[0] for w in want] and [bits(s) for s in scores] == [bits(w[1]) for w in want]
    st, lengths2, scores2, total2 = dec.beam_search_device(d_lp, off, d_tok, total - 1, lm, 16, 0.3, 0.5, 8)
    assert st == 3 and total2 == total and list(lengths2) == list(lengths)
    assert [bits(s) for s in scores2] == [bits(s) for s in scores]
    dec.close()


def test_beam_width_zero_gives_no_ids_and_minus_inf(D):
    """beam_width 0 with frames: the first prune keeps nothing, in both variants"""
    from fluidaudio_b200 import _lib
    rng = np.random.default_rng(15)
    V = 33
    voc = cases.vocabulary(rng, V)
    lm, arrays = _lm_pair(D, rng, words=300, bigrams=1500)
    clips = [cases.rows(rng, T, V, kind) for T, kind in ((1, "normal"), (40, "ties"), (0, "normal"), (7, "neginf"))]
    for K in (1, 5, 32):
        _check_beam(D, clips, V, 32, voc, (lm, arrays), 0, K)
        _check_beam(D, clips, V, 32, voc, None, 0, K)
    dec = D.CtcDecoder(voc, V, 32)
    lp, off = D._clips(clips, V)
    d_lp, d_tok = _lib.DeviceBuffer(lp.nbytes), _lib.DeviceBuffer(64)
    d_lp.upload(lp)
    st, lengths, scores, total = dec.beam_search_device(d_lp, off, d_tok, 16, lm, 0, 0.3, 0.0, 5)
    assert st == 0 and total == 0 and list(lengths) == [0] * 4
    assert list(scores) == [-np.inf, -np.inf, 0.0, -np.inf]
    dec.close()


def test_nan_and_inf_are_refused_with_the_outputs_untouched(D):
    from fluidaudio_b200 import _lib
    rng = np.random.default_rng(13)
    V = 17
    dec = D.CtcDecoder(cases.vocabulary(rng, V), V, 16)
    for bad in (np.nan, np.inf):
        clips = [cases.rows(rng, 20, V), cases.rows(rng, 9, V)]
        clips[1][4, 3] = bad
        lp, off = D._clips(clips, V)
        lengths, scores, tok, total = np.full(2, -7, np.int64), np.full(2, 9.0, np.float32), np.full(40, -3, np.int32), \
            C.c_int64(-5)
        cfg = dec.config()
        st = _lib.load().fa_ctc_beam_search(dec._h, None, _lib.ptr(lp), _lib.ptr(off), 2, C.byref(cfg),
                                            _lib.ptr(lengths), _lib.ptr(scores), _lib.ptr(tok), 40, C.byref(total))
        assert st == 1 and b"clip 1" in _lib.load().fa_last_error()
        assert (lengths == -7).all() and (scores == 9.0).all() and (tok == -3).all() and total.value == -5
    dec.close()


def test_launch_counts(D):
    from fluidaudio_b200 import _lib
    rng = np.random.default_rng(14)
    V = 33
    clips = [cases.rows(rng, T, V) for T in (30, 12)]
    dec = D.CtcDecoder(cases.vocabulary(rng, V), V, 32)
    before = _lib.kernel_launch_count()
    dec.beam_search(clips, None, 8, 0.3, 0.0, 5)
    assert _lib.kernel_launch_count() - before == 3
    before = _lib.kernel_launch_count()
    D.greedy_ids(clips, V, 32)
    assert _lib.kernel_launch_count() - before == 3
    dec.close()


# ---- the reference's decoder tests, through the GPU -----------------------------------------------------------------
VOCAB = {0: "▁hello", 1: "▁world", 2: "▁the", 3: "s", 4: "ing"}


def frames(hot, V=6, blank=5, high=-0.05, low=-5.0):
    m = np.full((len(hot), V), low, np.float32)
    for t, h in enumerate(hot):
        m[t, h] = high
    return m


def test_reference_greedy_cases(D):
    assert D.ctc_greedy_decode(frames([0, 5, 1]), VOCAB, 5) == "hello world"
    assert D.ctc_greedy_decode(frames([0, 0, 0, 1]), VOCAB, 5) == "hello world"
    assert D.ctc_greedy_decode(frames([2, 5, 2]), VOCAB, 5) == "the the"
    assert D.ctc_greedy_decode(frames([5, 5, 5]), VOCAB, 5) == ""
    assert D.ctc_greedy_decode(np.zeros((0, 6), np.float32), VOCAB, 5) == ""


def test_reference_beam_cases(D):
    lp = frames([0, 5, 1, 1, 5, 2, 3])
    assert D.ctc_beam_search(lp, VOCAB, blank_id=5) == D.ctc_greedy_decode(lp, VOCAB, 5)
    assert D.ctc_beam_search(frames([5, 5, 5]), VOCAB, blank_id=5) == ""
    assert D.ctc_beam_search(np.zeros((0, 6), np.float32), VOCAB, blank_id=5) == ""
    assert D.ctc_beam_search(frames([0]), VOCAB, blank_id=5) == "hello"
