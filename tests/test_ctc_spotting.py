"""CTC keyword spotting on the CPU: the reference's CtcDPAlgorithmTests on the oracle (``oracle/oracle_ctc.cpp``), the
oracle held to a pure-Python restatement (``tests/ctc_restated.py``), and the host build of the kernels' arithmetic
(``fluidaudio_b200/csrc/ctc/ctc_core.cuh`` through ``tests/emul/ctc_emul.cpp``) held to the oracle bit for bit, on
seeded cases that reach every rule of the dynamic program (``tests/ctc_cases.py``)."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import ctc_cases  # noqa: E402
import ctc_restated as R  # noqa: E402
from oracle import oracle_ctc as O  # noqa: E402

W = O.WILDCARD
NEG_MAX = -np.finfo(np.float32).max


def bits(x):
    return np.float32(x).view(np.uint32)


# ---- the reference's CtcDPAlgorithmTests, on the oracle ------------------------------------------------------------
def make_log_probs(frames, vocab, hot, high=-0.1, cold=-10.0):
    m = np.full((frames, vocab), cold, np.float32)
    for f, t in hot:
        if f < frames and t < vocab:
            m[f, t] = high
    return m


def make_frame(vocab, hot, high, blank_id, blank, cold):
    row = np.full(vocab, cold, np.float32)
    if blank_id < vocab:
        row[blank_id] = blank
    if hot is not None and hot < vocab:
        row[hot] = high
    return row


def test_non_wildcard_count_all_regular():
    assert O.non_wildcard_count([0, 1, 2]) == 3


def test_non_wildcard_count_mixed():
    assert O.non_wildcard_count([0, W, 1]) == 2


def test_non_wildcard_count_all_wildcards():
    assert O.non_wildcard_count([W, W, W]) == 0


def test_non_wildcard_count_empty():
    assert O.non_wildcard_count([]) == 0


def test_constrained_window_basic():
    lp = make_log_probs(20, 5, [(5, 0), (6, 1)])
    score, start, end = O.word_spot_constrained(lp, [0, 1], 3, 12)
    assert score > -1.0 and start >= 3 and end <= 12


def test_constrained_window_misses_keyword():
    lp = make_log_probs(20, 5, [(15, 0), (16, 1)])
    assert O.word_spot_constrained(lp, [0, 1], 0, 10)[0] < -5.0


def test_constrained_window_clamped():
    lp = make_log_probs(5, 3, [(2, 0)])
    assert O.word_spot_constrained(lp, [0], -5, 100)[0] > -np.inf


def test_constrained_window_too_small():
    lp = make_log_probs(20, 5, [])
    assert O.word_spot_constrained(lp, [0, 1, 2], 5, 7)[0] == -np.inf


def test_constrained_empty_window():
    lp = make_log_probs(10, 5, [])
    assert O.word_spot_constrained(lp, [0], 5, 5)[0] == -np.inf


def test_multiple_empty_keyword():
    assert O.word_spot_multiple(make_log_probs(5, 3, []), []) == []


def test_multiple_empty_log_probs():
    assert O.word_spot_multiple(np.zeros((0, 3), np.float32), [0]) == []


def test_multiple_below_min_score():
    assert O.word_spot_multiple(make_log_probs(5, 3, []), [0], min_score=-5.0) == []


def test_multiple_single_occurrence():
    res = O.word_spot_multiple(make_log_probs(10, 5, [(2, 0)], high=-0.1), [0], min_score=-1.0)
    assert len(res) >= 1 and res[0][0] > -1.0


def test_dp_table_score_monotonicity():
    lp = make_log_probs(3, 3, [(0, 0), (1, 1), (2, 2)], high=-0.05)
    assert abs(O.word_spot_constrained(lp, [0, 1, 2], 0, 3)[0] - (-0.05)) <= 0.01


def test_blank_emission_cost_is_accumulated():
    b, V = 3, 4
    rows = [make_frame(V, h, -0.1, b, -0.5, -10.0) for h in (0, None, None, None, 1)]
    assert abs(O.word_spot_constrained(np.array(rows), [0, 1], 0, 5, blank_id=b)[0] - (-0.85)) <= 0.01


def test_repeated_tokens_require_intervening_blank():
    b, V = 2, 3
    no_blank = np.array([make_frame(V, 0, -0.1, b, -0.5, -10.0) for _ in range(2)])
    with_blank = np.array([make_frame(V, h, -0.1, b, -0.5, -10.0) for h in (0, None, 0)])
    a = O.word_spot_constrained(no_blank, [0, 0], 0, 2, blank_id=b)[0]
    c = O.word_spot_constrained(with_blank, [0, 0], 0, 3, blank_id=b)[0]
    assert c > a + 1.0


def test_wildcard_still_free_cost():
    b, V = 3, 4
    rows = [make_frame(V, 0, -0.1, b, -10.0, -10.0), make_frame(V, None, -0.1, b, -0.1, -10.0),
            make_frame(V, 2, -0.1, b, -10.0, -10.0)]
    assert abs(O.word_spot_constrained(np.array(rows), [0, W, 2], 0, 3, blank_id=b)[0] - (-0.1)) <= 0.05


# ---- the host build of ctc_core.cuh ---------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def emul(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("ctc") / "libctc_emul.so")
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-fPIC", "-shared", "-o", out,
                           os.path.join(ROOT, "tests", "emul", "ctc_emul.cpp")])
    L = C.CDLL(out)
    vp, i32, i64, f32 = C.c_void_p, C.c_int32, C.c_int64, C.c_float
    L.ctc_emul_log_softmax.argtypes = [vp, i32, i32, i32, f32, f32, i32, vp]
    L.ctc_emul_merge_overlap.argtypes = [vp, vp, i64, vp]
    L.ctc_emul_multiple.argtypes = [vp, i32, i32, vp, i32, f32, i32, vp, vp, vp, i32]
    L.ctc_emul_multiple.restype = i32
    L.ctc_emul_constrained.argtypes = [vp, i32, i32, vp, i32, i64, i64, i32, vp, vp, vp]
    L.ctc_emul_threshold.argtypes = [i32, f32, i32]
    L.ctc_emul_threshold.restype = f32
    return L


def emul_multiple(L, lp, toks, thr, blank):
    lp = np.ascontiguousarray(lp, np.float32)
    tok = np.asarray(toks, np.int32)
    T, V = lp.shape
    cap = T // 2 + 2
    s, a, e = np.empty(cap, np.float32), np.empty(cap, np.int32), np.empty(cap, np.int32)
    n = L.ctc_emul_multiple(lp.ctypes.data, T, V, tok.ctypes.data, len(tok), thr, blank, s.ctypes.data, a.ctypes.data,
                            e.ctypes.data, cap)
    return [(np.float32(s[i]), int(a[i]), int(e[i])) for i in range(n)]


def emul_constrained(L, lp, toks, ss, se, blank):
    lp = np.ascontiguousarray(lp, np.float32)
    tok = np.asarray(toks, np.int32)
    s, a, b = C.c_float(), C.c_int64(), C.c_int64()
    L.ctc_emul_constrained(lp.ctypes.data, lp.shape[0], lp.shape[1], tok.ctypes.data, len(tok), ss, se, blank,
                           C.byref(s), C.byref(a), C.byref(b))
    return np.float32(s.value), a.value, b.value


def same(a, b):
    return len(a) == len(b) and all(bits(x[0]) == bits(y[0]) and tuple(x[1:]) == tuple(y[1:]) for x, y in zip(a, b))


CASES = ctc_cases.cases(0)


@pytest.mark.parametrize("case", range(0, len(CASES), 3))   # every third case: the restatement is slow
def test_oracle_equals_restatement(case):
    name, lp, toks, blank = CASES[case]
    rng = np.random.default_rng(case)
    for ms in ctc_cases.MIN_SCORES:
        thr = O.threshold(ms, len(toks))
        assert bits(thr) == bits(R.threshold(ms, len(toks)))
        assert same(O.word_spot_multiple(lp, toks, thr, blank), R.word_spot_multiple(lp, toks, thr, blank)), (name, ms)
    for ss, se in ctc_cases.windows(rng, len(lp), 2):
        assert same([O.word_spot_constrained(lp, toks, ss, se, blank)],
                    [R.word_spot_constrained(lp, toks, ss, se, blank)]), (name, ss, se)


@pytest.mark.parametrize("case", range(len(CASES)))
def test_emulation_equals_oracle(emul, case):
    name, lp, toks, blank = CASES[case]
    rng = np.random.default_rng(case)
    for ms in ctc_cases.MIN_SCORES:
        thr = O.threshold(ms, len(toks))
        assert bits(emul.ctc_emul_threshold(int(ms is not None), 0.0 if ms is None else ms, len(toks))) == bits(thr)
        if len(lp) == 0:
            continue
        assert same(emul_multiple(emul, lp, toks, thr, blank), O.word_spot_multiple(lp, toks, thr, blank)), (name, ms)
    if len(lp) == 0:
        return
    for ss, se in ctc_cases.windows(rng, len(lp)):
        assert same([emul_constrained(emul, lp, toks, ss, se, blank)],
                    [O.word_spot_constrained(lp, toks, ss, se, blank)]), (name, ss, se)


def test_cases_reach_every_rule():
    """the fallback and -FLT_MAX scores in the output"""
    fallback = flt_max = 0
    for name, lp, toks, blank in CASES:
        for ms in (float("-inf"), -3e38):
            for s, a, e in O.word_spot_multiple(lp, toks, ms, blank):
                flt_max += s <= NEG_MAX / 2
        found = O.word_spot_multiple(lp, toks, float("-inf"), blank)
        fallback += len(found) == 1 and found[0][1:] == (0, 0) and found[0][0] == np.float32(NEG_MAX)
    assert fallback and flt_max


@pytest.mark.parametrize("V", [1, 5, 129])
@pytest.mark.parametrize("temperature", [1.0, 0.7, 1.3])
@pytest.mark.parametrize("bias,blank", [(0.0, 1024), (0.5, 2), (0.5, 1024)])
def test_log_softmax(emul, V, temperature, bias, blank):
    rng = np.random.default_rng(V)
    x = (rng.normal(0, 4, size=(9, V))).astype(np.float32)
    x[0, 0] = -np.inf
    want = O.log_softmax(x, temperature, bias, blank)
    assert want.tobytes() == R.log_softmax(x, temperature, bias, blank).tobytes()
    for vm, src in ((False, x), (True, np.ascontiguousarray(x.T))):
        got = np.empty_like(want)
        emul.ctc_emul_log_softmax(src.ctypes.data, 9, V, int(vm), temperature, bias, blank, got.ctypes.data)
        assert got.tobytes() == want.tobytes()
        assert O.log_softmax(src, temperature, bias, blank, vocab_major=vm).tobytes() == want.tobytes()


@pytest.mark.parametrize("overlap", [0, 1, 3, 25])
def test_merge_chunks(emul, overlap):
    rng = np.random.default_rng(overlap)
    V = 6
    chunks = [ctc_cases.log_probs(rng, n, V, "neginf") for n in (5, 0, 2, 7, 1, 4)]
    chunks[3][:2] = -np.inf
    want = O.merge_chunks(chunks, overlap)
    assert want.tobytes() == R.merge_chunks(chunks, overlap).tobytes()
    a, b = chunks[0], chunks[3][:5]
    got = np.empty_like(a)
    emul.ctc_emul_merge_overlap(a.ctypes.data, b.ctypes.data, a.size, got.ctypes.data)
    assert got.tobytes() == np.array([R.merge_overlap_frame(x, y) for x, y in zip(a, b)], np.float32).tobytes()
