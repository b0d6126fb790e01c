"""CTC decoding on the CPU: the reference's decoder and ARPA tests on the oracle (``oracle/oracle_ctc_decode.cpp``) and
the Python loader (``fluidaudio_b200.ctc_decoding``, ARPA fixtures written here, the ``\\r\\n`` one included), the
reference's tab-split parse of a KenLM-style bigram line, Swift's number syntax, and the oracle's beam search on seeded
cases that reach the rules the GPU sweep relies on (a pruned prefix re-created while its child survives, ties, LM
terms with bigram hits, backoff and unknown words, a blank outside the vocabulary, beam widths 0 to 2)."""
import math
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import ctc_decode_cases as cases  # noqa: E402
import ctc_decode_restated as R  # noqa: E402
from fluidaudio_b200 import ctc_decoding as D  # noqa: E402
from oracle import oracle_ctc_decode as O  # noqa: E402

VOCAB = {0: "▁hello", 1: "▁world", 2: "▁the", 3: "s", 4: "ing"}
PIECES = [VOCAB.get(v) for v in range(6)]


def bits(x):
    return np.float32(x).view(np.uint32)


def frames(hot, V=6, high=-0.05, low=-5.0):
    m = np.full((len(hot), V), low, np.float32)
    for t, h in enumerate(hot):
        m[t, h] = high
    return m


# ---- logAddExp and decodeCtcTokenIds ------------------------------------------------------------------------------
def test_log_add_exp_equal_values():
    assert abs(O.log_add_exp(0.0, 0.0) - math.log(2.0)) < 1e-6


def test_log_add_exp_with_neg_infinity():
    assert O.log_add_exp(-np.inf, -3.0) == np.float32(-3.0) and O.log_add_exp(-2.0, -np.inf) == np.float32(-2.0)


def test_log_add_exp_both_neg_infinity():
    assert O.log_add_exp(-np.inf, -np.inf) == -np.inf


def test_log_add_exp_large_difference():
    assert abs(O.log_add_exp(0.0, -100.0)) < 1e-6


def test_log_add_exp_is_commutative():
    rng = np.random.default_rng(0)
    for a, b in rng.normal(0, 20, size=(200, 2)).astype(np.float32):
        assert bits(O.log_add_exp(a, b)) == bits(O.log_add_exp(b, a))


def test_decode_token_ids():
    assert D.decode_ctc_token_ids([0, 1], VOCAB) == "hello world"
    assert D.decode_ctc_token_ids([], VOCAB) == ""
    assert D.decode_ctc_token_ids([0, 99, 1], VOCAB) == "hello world"
    assert D.decode_ctc_token_ids([2, 3, 4], VOCAB) == "thesing"
    # .whitespaces is Zs and tab: a newline at either end stays
    assert D.decode_ctc_token_ids([0], {0: "\u2581a\n"}) == "a\n"
    assert D.decode_ctc_token_ids([0], {0: "\t\u00a0a\u3000"}) == "a"


# ---- greedy ------------------------------------------------------------------------------------------------------
def test_greedy_reference_cases():
    assert D.decode_ctc_token_ids(O.greedy(frames([0, 5, 1]), 5), VOCAB) == "hello world"
    assert O.greedy(frames([0, 0, 0, 1]), 5) == [0, 1]
    assert O.greedy(frames([2, 5, 2]), 5) == [2, 2]
    assert O.greedy(frames([5, 5, 5]), 5) == []
    assert O.greedy(np.zeros((0, 6), np.float32), 5) == []


def test_greedy_nan_rule():
    x = frames([1, 2, 3])
    x[0, 0] = np.nan   # column 0 as NaN wins
    x[1, 4] = np.nan   # elsewhere never
    assert O.greedy(x, 5) == [0, 2, 3]


# ---- beam search -------------------------------------------------------------------------------------------------
def test_beam_reference_cases():
    lp = frames([0, 5, 1, 1, 5, 2, 3])
    assert O.beam_search(lp, PIECES, blank_id=5)[0] == O.greedy(lp, 5)
    assert O.beam_search(frames([5, 5, 5]), PIECES, blank_id=5)[0] == []
    assert O.beam_search(np.zeros((0, 6), np.float32), PIECES, blank_id=5) == ([], np.float32(0.0))
    assert O.beam_search(frames([0]), PIECES, blank_id=5)[0] == [0]
    assert O.beam_search(frames([0, 1]), PIECES, beam_width=0, blank_id=5) == ([], np.float32(-np.inf))


def test_ctc_beam_total_acoustic_and_lm():
    """testCtcBeamTotalAcoustic / testCtcBeamTotalIncludesLM / testCtcBeamLastToken(Empty), on the restatement's beam"""
    b = R.Beam((1, 2), -1.0, -2.0, 0.0, [], None)
    assert b.total_acoustic == R.log_add_exp(-1.0, -2.0) == O.log_add_exp(-1.0, -2.0)
    b.lm_score = np.float32(-0.5)
    assert b.total == np.float32(R.log_add_exp(-1.0, -2.0) - np.float32(0.5))
    assert b.prefix[-1] == 2 and not R.Beam((), 0.0, -np.inf, 0.0, [], None).prefix


def test_multiarray_layout_matches_the_frames():
    """testGreedyDecodeMLMultiArray / testBeamSearchMLMultiArrayMatchesGreedy: a [1, T, V] buffer read row by row"""
    lp = frames([0, 5, 1, 1, 5, 2])
    flat = lp.reshape(1, *lp.shape).ravel().reshape(lp.shape)
    assert O.greedy(flat, 5) == O.greedy(lp, 5) == [0, 1, 2]
    assert O.beam_search(flat, PIECES, blank_id=5)[0] == O.greedy(lp, 5)


def test_beam_lm_changes_the_result():
    """testBeamSearchWithLMInfluencesResult: two near-equal readings, the LM's bigram picks one"""
    voc = {0: "▁patient", 1: "▁has", 2: "▁diabetes", 3: "▁die", 4: "▁beetus"}
    lp = np.full((5, 6), -8.0, np.float32)
    lp[0, 0] = lp[1, 1] = -0.01
    lp[2, 2], lp[2, 3] = -0.9, -0.8
    lp[3, 5] = lp[4, 5] = -0.01
    lm = O.LmArrays({"patient": (np.float32(-1.5), np.float32(-0.3)), "has": (np.float32(-1.8), np.float32(-0.2)),
                     "diabetes": (np.float32(-2.2), np.float32(-0.1)), "die": (np.float32(-4.0), np.float32(-0.5))},
                    {"has": {"diabetes": np.float32(-0.5)}})
    pieces = [voc.get(v) for v in range(6)]
    assert O.beam_search(lp, pieces, None, 10, blank_id=5)[0] == [0, 1, 3]
    assert O.beam_search(lp, pieces, lm, 10, lm_weight=1.0, blank_id=5)[0] == [0, 1, 2]


def test_a_pruned_prefix_is_recreated_while_its_child_survives():
    """the case that parent pointers alone would get wrong: the seeded search reaches it"""
    found = 0
    for seed in range(40):
        rng = np.random.default_rng(seed)
        V = 6
        lp = cases.rows(rng, 12, V, "ties")
        found += O.beam_search(lp, [None] * V, None, 2, blank_id=V - 1, token_candidates=3, stats=True)[2]
    assert found > 0


def test_ties_resolve_by_first_insertion():
    """hand-worked: every token column ties.  B = 1 keeps the first-inserted best, the extension by the lowest index;
    B = 2 keeps the blank extension and that one, and the final pick is the first of two equal totals: the empty
    prefix"""
    lp = np.array([[-1.0, -1.0, -1.0, -2.0]], np.float32)
    rl = R.beam_search(lp, {}, None, 1, blank_id=3)
    assert O.beam_search(lp, [None] * 4, None, 1, blank_id=3) == rl == ([0], np.float32(-1.0))
    lp[0, 3] = -1.0
    assert O.beam_search(lp, [None] * 4, None, 2, blank_id=3)[0] == R.beam_search(lp, {}, None, 2, blank_id=3)[0] == []


def _cases():
    """seeded small searches that reach every rule: tie-heavy, constant and -inf rows; a blank outside [0, V); K up to
    and past V - 1; B in {0, 1, 2, 7}; T in {0, 1, ...}; an LM with bigram hits, backoff, unknown words, `▁`-only,
    empty and missing pieces; lm_weight 0 with a word bonus"""
    for seed in range(8):
        rng = np.random.default_rng(200 + seed)
        V = int(rng.integers(3, 10))
        voc = cases.vocabulary(rng, V, letters="abc", missing=0.15)
        uni, bi = cases.synthetic_lm(rng, words=25, bigrams=80, letters="abc", max_len=3)
        lms = [None, (uni, bi)]
        for kind in ("ties", "constant", "neginf", "normal"):
            T = int(rng.integers(0, 14)) if kind != "normal" else 1
            lp = cases.rows(rng, T, V, kind)
            for B in (0, 1, 2, 7):
                K = int(rng.choice([1, 3, V - 1, V + 4]))
                blank = int(rng.choice([V - 1, 0, V + 2]))
                lm = lms[(seed + B) % 2]
                w, bonus = (0.0, 0.7) if seed % 3 == 0 else (0.3, 0.0)
                yield f"{seed}-{kind}-{B}", lp, voc, lm, B, K, blank, w, bonus


def _oracle(lp, voc, lm, B, K, blank, w, bonus):
    arrays = O.LmArrays(*lm) if lm else None
    return O.beam_search(lp, cases.pieces(voc, lp.shape[1]), arrays, B, w, bonus, blank, K)


def test_oracle_equals_the_restatement():
    n = 0
    for name, lp, voc, lm, B, K, blank, w, bonus in _cases():
        want = R.beam_search(lp, voc, R.LM(*lm) if lm else None, B, w, bonus, blank, K)
        got = _oracle(lp, voc, lm, B, K, blank, w, bonus)
        assert got[0] == want[0] and bits(got[1]) == bits(want[1]), name
        assert O.greedy(lp, blank) == R.greedy(lp, blank), name
        n += 1
    assert n == 128


def test_the_restatement_reaches_a_recreated_prefix():
    found = 0
    for seed in range(40):
        rng = np.random.default_rng(seed)
        lp = cases.rows(rng, 12, 6, "ties")
        st = {}
        R.beam_search(lp, {}, None, 2, blank_id=5, token_candidates=3, stats=st)
        found += st["recreated"]
        assert st["recreated"] == O.beam_search(lp, [None] * 6, None, 2, blank_id=5, token_candidates=3, stats=True)[2]
    assert found > 0


@pytest.fixture(scope="module")
def emul(tmp_path_factory):
    import ctypes as C
    import subprocess
    out = str(tmp_path_factory.mktemp("ctc_decode") / "libctc_decode_emul.so")
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-fPIC", "-shared", "-o", out,
                           os.path.join(os.path.dirname(os.path.abspath(__file__)), "emul", "ctc_decode_emul.cpp")])
    L = C.CDLL(out)
    vp, i32, i64, f32 = C.c_void_p, C.c_int32, C.c_int64, C.c_float
    L.ctc_decode_emul_greedy.argtypes = [vp, i32, i32, i32, vp]
    L.ctc_decode_emul_greedy.restype = i32
    lm = [i32, vp, vp, vp, vp, vp, i64, vp, vp, vp]
    L.ctc_decode_emul_beam.argtypes = [vp, i32, i32, i32, vp, vp, i32] + lm + [i32, i32, f32, f32, vp, i64,
                                                                             C.POINTER(f32)]
    L.ctc_decode_emul_beam.restype = i64
    return L


def _emul_beam(L, lp, voc, lm, B, K, blank, w, bonus):
    import ctypes as C
    T, V = lp.shape
    buf, off = O.blob([voc.get(v, "") for v in range(V)])
    arrays = O.LmArrays(*lm) if lm else O.LmArrays({}, {})
    out = np.zeros(max(1, T), np.int32)
    score = C.c_float()
    n = L.ctc_decode_emul_beam(lp.ctypes.data, T, V, blank, buf.ctypes.data, off.ctypes.data, int(lm is not None),
                               *arrays.args(), B, K, w, bonus, out.ctypes.data, out.size, C.byref(score))
    assert n >= 0
    return [int(x) for x in out[:n]], np.float32(score.value)


def test_emulation_equals_the_oracle(emul):
    for name, lp, voc, lm, B, K, blank, w, bonus in _cases():
        got = _emul_beam(emul, lp, voc, lm, B, K, blank, w, bonus)
        want = _oracle(lp, voc, lm, B, K, blank, w, bonus)
        assert got[0] == want[0] and bits(got[1]) == bits(want[1]), name
        ids = np.zeros(max(1, lp.shape[0]), np.int32)
        n = emul.ctc_decode_emul_greedy(lp.ctypes.data, lp.shape[0], lp.shape[1], blank, ids.ctypes.data)
        assert list(ids[:n]) == O.greedy(lp, blank), name


def test_emulation_equals_the_oracle_with_a_larger_lm(emul):
    rng = np.random.default_rng(31)
    V = 65
    voc = cases.vocabulary(rng, V)
    lm = cases.synthetic_lm(rng, words=2000, bigrams=8000, max_len=4)
    for T, B, K in ((40, 16, 8), (25, 100, 40), (12, 128, 64)):
        lp = cases.rows(rng, T, V, "normal")
        got = _emul_beam(emul, lp, voc, lm, B, K, V - 1, 0.3, 0.1)
        want = _oracle(lp, voc, lm, B, K, V - 1, 0.3, 0.1)
        assert got[0] == want[0] and bits(got[1]) == bits(want[1]), (T, B, K)


def test_greedy_nan_rule_in_the_emulation(emul):
    x = frames([1, 2, 3, 3])
    x[0, 0] = np.nan
    x[1, 4] = np.nan
    ids = np.zeros(4, np.int32)
    n = emul.ctc_decode_emul_greedy(x.ctypes.data, 4, 6, 5, ids.ctypes.data)
    assert list(ids[:n]) == O.greedy(x, 5) == R.greedy(x, 5) == [0, 2, 3]


# ---- ARPA ---------------------------------------------------------------------------------------------------------
SAMPLE = ("\\data\\\nngram 1=4\nngram 2=2\n\n\\1-grams:\n-1.0\tthe\t-0.5\n-1.2\tcat\t-0.3\n-1.5\tsat\t0.0\n"
          "-2.0\t<unk>\t0.0\n\n\\2-grams:\n-0.5\tthe\tcat\n-0.8\tcat\tsat\n\n\\end\\\n")


def _write(tmp_path, text, name="lm.arpa"):
    p = tmp_path / name
    p.write_bytes(text.encode("utf-8") if isinstance(text, str) else text)
    return str(p)


def test_load_arpa(tmp_path):
    lm = D.ARPALanguageModel.load(_write(tmp_path, SAMPLE))
    assert len(lm.unigrams) == 4 and len(lm.bigrams) == 2
    e = lm.unigrams["the"]
    assert e.log_prob == np.float32(np.float32(-1.0) * D.ARPALanguageModel.LOG10_TO_NAT)
    assert e.backoff == np.float32(np.float32(-0.5) * D.ARPALanguageModel.LOG10_TO_NAT)
    assert "cat" in lm.bigrams["the"]


def test_load_missing_and_empty(tmp_path):
    with pytest.raises(OSError):
        D.ARPALanguageModel.load(str(tmp_path / "none.arpa"))
    lm = D.ARPALanguageModel.load(_write(tmp_path, ""))
    assert lm.unigrams == {} and lm.bigrams == {}


def test_score_rules(tmp_path):
    lm = D.ARPALanguageModel.load(_write(tmp_path, SAMPLE))
    n = D.ARPALanguageModel.LOG10_TO_NAT
    assert lm.score("cat", "the") == lm.bigrams["the"]["cat"].log_prob
    assert lm.score("sat", "the") == np.float32(lm.unigrams["the"].backoff + lm.unigrams["sat"].log_prob)
    assert lm.score("cat", None) == lm.unigrams["cat"].log_prob
    assert lm.score("zebra", None) == D.ARPALanguageModel.UNK_LOG_PROB
    assert lm.score("zebra", "the") == np.float32(np.float32(-0.5) * n + D.ARPALanguageModel.UNK_LOG_PROB)
    arrays = O.LmArrays({w: (e.log_prob, e.backoff) for w, e in lm.unigrams.items()},
                        {c: {w: e.log_prob for w, e in r.items()} for c, r in lm.bigrams.items()})
    for word, prev in (("cat", "the"), ("sat", "the"), ("cat", None), ("zebra", None), ("zebra", "the"),
                       ("sat", "zebra")):
        assert bits(O.lm_score(arrays, word, prev)) == bits(lm.score(word, prev))


def test_windows_line_endings(tmp_path):
    text = "\\data\\\r\nngram 1=2\r\n\r\n\\1-grams:\r\n-1.0\thello\t0.0\r\n-1.0\tworld\t0.0\r\n\r\n\\end\\\r\n"
    lm = D.ARPALanguageModel.load(_write(tmp_path, text))
    assert set(lm.unigrams) == {"hello", "world"}


def test_kenlm_style_bigram_line_splits_on_tabs_as_the_reference(tmp_path):
    text = "\\2-grams:\n-0.3\tthe cat\t-0.1\n\\end\\\n"
    lm = D.ARPALanguageModel.load(_write(tmp_path, text))
    assert list(lm.bigrams) == ["the cat"] and list(lm.bigrams["the cat"]) == ["-0.1"]


def test_invalid_utf8_ends_the_read_and_duplicates_overwrite(tmp_path):
    text = b"\\1-grams:\n-1.0\ta\n-2.0\ta\n\xff\xfe\n-1.0\tb\n"
    lm = D.ARPALanguageModel.load(_write(tmp_path, text))
    assert list(lm.unigrams) == ["a"] and lm.unigrams["a"].log_prob == np.float32(np.float32(-2.0) *
                                                                                 D.ARPALanguageModel.LOG10_TO_NAT)


@pytest.mark.parametrize("text,value", [("-1.5", -1.5), ("1e-3", 1e-3), ("0x1p-2", 0.25), ("+2", 2.0), (" 1", None),
                                        ("1 ", None), ("1_0", None), ("", None), ("abc", None), ("1.5\x00x", 1.5)])
def test_swift_float_syntax(text, value):
    got = D.swift_float(text)
    assert (got is None) if value is None else got == np.float32(value)
