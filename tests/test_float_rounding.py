"""The float32 exp, log and log1p that five families promise to round like their oracles, checked on every float32 input.

fa_float.cuh's f_exp / f_log / f_log1p (host build: tests/emul/fa_float_emul.cpp), oracle/oracle_float.h (through
tests/emul/oracle_float_emul.cpp) and tests/float_exact.py must each return the correctly rounded float32 of the exact
function.  The reference is built here, independently of the library's table: glibc's float64 result rounded to
float32, replaced by mpmath's correctly rounded value wherever that float64 result lies within 3 float64 ulps of a
float32 rounding boundary (tests/emul/float_reference.cpp scans all 2^32 inputs on every core).

The planted cases then drive each family's own arithmetic (the oracle, the Python restatement and the host build of
the kernels' code) onto inputs where glibc's (float)f((double)x) rounds wrong, or where a 1-ulp float64 error can, and
require all three to agree with each other and with the correctly rounded value.  The exhaustive checks take about
6 minutes on 8 cores, most of it in the long double oracle.
"""
import ctypes
import math
import os
import re
import subprocess

import numpy as np
import pytest

import float_exact as FE

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F = np.float32
CAP = 64   # mismatches reported per check


def bits(x):
    return np.ascontiguousarray(x, np.float32).view(np.uint32)


def from_bits(b):
    return np.uint32(b).view(np.float32)


def hexf(x):
    return float(np.float32(x)).hex()


@pytest.fixture(scope="module")
def reference(tmp_path_factory):
    """The reference library and, per function, its fragile inputs with their correctly rounded values."""
    L = FE.reference_library(tmp_path_factory.mktemp("float_reference"))
    return L, [FE.fragile_table(L, fn) for fn in range(3)]


def _compile(tmp_path_factory, src, symbol):
    out = str(tmp_path_factory.mktemp("float_impl") / (src.replace(".cpp", ".so")))
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-fPIC", "-shared", "-o", out,
                           os.path.join(ROOT, "tests", "emul", src)])
    L = ctypes.CDLL(out)
    getattr(L, symbol).argtypes = [ctypes.c_int, ctypes.c_uint64, ctypes.c_uint64, ctypes.c_void_p]
    getattr(L, symbol).restype = None
    return L, getattr(L, symbol)


@pytest.fixture(scope="module")
def fa_float(tmp_path_factory):
    return _compile(tmp_path_factory, "fa_float_emul.cpp", "fa_float_emul_eval")


@pytest.fixture(scope="module")
def oracle_float(tmp_path_factory):
    return _compile(tmp_path_factory, "oracle_float_emul.cpp", "oracle_float_eval")


def _exhaustive(reference, impl, fn):
    L, tables = reference
    xs, vals = tables[fn]
    bad = np.zeros((CAP, 3), np.uint32)
    n = L.fr_check(fn, ctypes.cast(impl, ctypes.c_void_p), xs.ctypes.data, vals.ctypes.data, len(xs), bad.ctypes.data,
                   CAP)
    report = "\n".join(f"{FE.NAMES[fn]}({hexf(from_bits(x))}) = {hexf(from_bits(g))}, expected {hexf(from_bits(w))}"
                       for x, g, w in bad[:min(n, CAP)])
    assert n == 0, f"{n} mismatches over all 2^32 inputs:\n{report}"


@pytest.mark.parametrize("fn", [FE.EXP, FE.LOG, FE.LOG1P], ids=FE.NAMES)
def test_fa_float_host_exhaustive(reference, fa_float, fn):
    _exhaustive(reference, fa_float[1], fn)


@pytest.mark.parametrize("fn", [FE.EXP, FE.LOG, FE.LOG1P], ids=FE.NAMES)
def test_oracle_float_exhaustive(reference, oracle_float, fn):
    _exhaustive(reference, oracle_float[1], fn)


# ---- the Python helper and the library's table -----------------------------------------------------------------------
SPECIALS = [0.0, -0.0, 1.0, -1.0, np.inf, -np.inf, np.nan, 2.0 ** -149, -(2.0 ** -149), 2.0 ** -126, 88.72283,
            88.72284, -87.33655, -103.27893, -103.97208, -104.0, float(np.finfo(np.float32).max),
            -float(np.finfo(np.float32).max), 0.5, -0.5, 2.0, 1e-30, -1e-30]


def _reference_at(reference, fn, xs):
    L, tables = reference
    fin, fval = tables[fn]
    xs = np.ascontiguousarray(xs, np.uint32)
    out = np.zeros(len(xs), np.uint32)
    L.fr_reference(fn, 0, len(xs), xs.ctypes.data, fin.ctypes.data, fval.ctypes.data, len(fin), out.ctypes.data)
    return out


@pytest.mark.parametrize("fn", [FE.EXP, FE.LOG, FE.LOG1P], ids=FE.NAMES)
def test_python_helper(reference, fn):
    rng = np.random.default_rng(17 + fn)
    xs = np.concatenate([np.concatenate([t[0] for t in reference[1]]), np.array(SPECIALS, np.float32).view(np.uint32),
                         rng.integers(0, 2 ** 32, size=10 ** 6, dtype=np.uint64).astype(np.uint32)])
    want = _reference_at(reference, fn, xs)
    got = np.array([FE.f32(fn, x) for x in xs.view(np.float32)], np.float32).view(np.uint32)
    nan = np.isnan(got.view(np.float32)) & np.isnan(want.view(np.float32))
    bad = np.flatnonzero((got != want) & ~nan)
    assert bad.size == 0, [(hexf(from_bits(xs[i])), hexf(from_bits(got[i])), hexf(from_bits(want[i]))) for i in bad[:CAP]]


def _library_table():
    """fa_float_table.h as {fn: (inputs, values)}"""
    text = open(os.path.join(ROOT, "fluidaudio_b200", "csrc", "fa_float_table.h")).read()
    out = {}
    for fn, name in enumerate(FE.NAMES):
        block = text.split(f"#define FA_CR_{name.upper()}_TABLE")[1].split("\n\n")[0]
        pairs = re.findall(r"\{0x([0-9a-f]{8})u, 0x([0-9a-f]{8})u\}", block)
        out[fn] = (np.array([int(a, 16) for a, _ in pairs], np.uint32), np.array([int(b, 16) for _, b in pairs], np.uint32))
        assert f"k{name.capitalize()}Count = {len(pairs)};" in text
    return out


@pytest.mark.parametrize("fn", [FE.EXP, FE.LOG, FE.LOG1P], ids=FE.NAMES)
def test_library_table_is_every_fragile_input_with_its_correct_value(reference, fn):
    xs, vals = _library_table()[fn]
    want_x, want_v = reference[1][fn]
    assert np.all(np.diff(xs.astype(np.int64)) > 0), "the table must be sorted by input bits for the binary search"
    assert np.array_equal(xs, want_x) and np.array_equal(vals, want_v)
    for x, v in zip(xs.view(np.float32), vals.view(np.float32)):
        assert FE.fragile(FE._libm(fn, x)) and FE.correctly_rounded(fn, x) == v


def test_glibc_rounds_the_known_inputs_wrong():
    """The inputs at which (float)f((double)x) with glibc is not the correctly rounded float32 (glibc 2.39): the reason
    the library and the oracles no longer use that policy."""
    wrong = {FE.LOG: "0x1.827a74p-7 0x1.2f1fd6p+3 0x1.bacb4ap+25 0x1.b121a6p+76 0x1.6351d8p+95",
             FE.LOG1P: "0x1.800006p-21 0x1.200036p-17 0x1.fb035ap-2 0x1.0f1fd6p+3 0x1.b121a6p+76 0x1.6351d8p+95 "
                       "-0x1.7ffffap-21 -0x1.1fffcap-17 -0x1.1d9188p-9"}
    for fn, xs in wrong.items():
        for x in map(float.fromhex, xs.split()):
            assert FE.fragile(FE._libm(fn, F(x)))
            assert FE._f32(FE._libm(fn, F(x))) != FE.f32(fn, F(x)), (FE.NAMES[fn], float(x).hex())


# ---- planted cases: each family's arithmetic driven onto a hard input ------------------------------------------------
# Each case runs the family's oracle, its Python restatement and the host build of the kernels' code on one input that
# puts a helper's argument exactly on a hard input, and requires the three to agree bit for bit.  Where glibc's
# (float)f((double)x) rounds that input wrong, the case also requires the restatement to differ from what it computes
# under that old policy: the family's result depends on the correct rounding.
HARD_EXP = F(float.fromhex("-0x1.d2259ap+3"))   # fragile: glibc rounds it right, a 1-ulp libm may not
HARD_LOG = F(float.fromhex("0x1.2f1fd6p+3"))    # glibc rounds log wrong here


def _old(fn):
    return lambda x: FE._f32(FE._libm(fn, F(x)))


@pytest.fixture
def old_policy(monkeypatch):
    """Within a test: a restatement's exp / log / log1p as glibc's (float)f((double)x), the policy before the correctly
    rounded definition.  apply(module, exp="its exp's name", ...)."""
    def apply(module, **names):
        for kind, attr in names.items():
            monkeypatch.setattr(module, attr, _old(FE.NAMES.index(kind)))
    return apply


def _emul(tmp_path_factory, src, name):
    out = str(tmp_path_factory.mktemp(name) / f"lib{name}.so")
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-fPIC", "-shared", "-o", out,
                           os.path.join(ROOT, "tests", "emul", src)])
    return ctypes.CDLL(out)


def _sum_row(target, fn_exp=FE.exp):
    """A float32 logit row [0] * 9 + [y] whose float32 exp sum, in index order after subtracting the max 0, is exactly
    target (in (9, 10))."""
    y = F(math.log(float(target) - 9))
    for _ in range(4096):
        s = F(0)
        for v in [F(0)] * 9 + [y]:
            s = F(s + fn_exp(v))
        if s == target:
            return np.array([0] * 9 + [y], np.float32)
        y = np.nextafter(y, F(np.inf) if s < target else F(-np.inf), dtype=np.float32)
    raise AssertionError("no row found")


def test_planted_ctc_spotting(tmp_path_factory, old_policy):
    from oracle import oracle_ctc as O
    import ctc_restated as R
    L = _emul(tmp_path_factory, "ctc_emul.cpp", "ctc_emul")
    L.ctc_emul_log_softmax.argtypes = [ctypes.c_void_p] + [ctypes.c_int32] * 3 + [ctypes.c_float] * 2 + \
        [ctypes.c_int32, ctypes.c_void_p]
    rows = np.stack([_sum_row(HARD_LOG),                                   # lse = log(HARD_LOG)
                     np.array([0, HARD_EXP] + [-30] * 8, np.float32)])      # exp(HARD_EXP)
    want = O.log_softmax(rows)
    got = np.zeros_like(rows)
    L.ctc_emul_log_softmax(rows.ctypes.data, rows.shape[0], rows.shape[1], 0, 1.0, 0.0, 1024, got.ctypes.data)
    restated = np.array(R.log_softmax(rows), np.float32)
    assert np.array_equal(bits(want), bits(got)) and np.array_equal(bits(want), bits(restated))
    assert want[0, 0] == -FE.log(HARD_LOG)
    old_policy(R, exp="fexp", log="flog")
    assert not np.array_equal(bits(np.array(R.log_softmax(rows[:1]), np.float32)), bits(want[:1]))


def test_planted_ctc_decoding():
    from oracle import oracle_ctc_decode as O
    import ctc_decode_restated as R
    a, b = F(0), HARD_EXP   # m = 0: log(1 + exp(HARD_EXP))
    want = O.log_add_exp(a, b)
    assert F(want).tobytes() == F(R.log_add_exp(a, b)).tobytes() == F(FE.log(F(1 + FE.exp(HARD_EXP)))).tobytes()


def test_planted_styletts2(tmp_path_factory):
    from oracle import oracle_styletts2 as O
    import styletts2_restated as R
    L = _emul(tmp_path_factory, "styletts2_emul.cpp", "styletts2_emul")
    L.styletts2_emul_durations.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_void_p]
    logits = np.array([[-HARD_EXP] * 3 + [0.5] * 4, [-HARD_EXP] * 7], np.float32)   # expf(-x) at the hard input
    got = np.zeros(2, np.int32)
    L.styletts2_emul_durations(logits.ctypes.data, 2, 7, got.ctypes.data)
    assert list(O.round_durations(logits)) == R.round_durations(logits) == list(got)


@pytest.mark.parametrize("p", ["0x1.1d9188p-9", "0x1.7ffffap-21", "0x1.1fffcap-17", "0x1.827a74p-7"])
def test_planted_sortformer(tmp_path_factory, old_policy, p):
    """Compression scores of a default-config session whose predictions hold p: log1p(-p) on a hard input, or for
    0x1.827a74p-7, with pred_score_threshold lowered to 0.01, log(p) on one."""
    from fluidaudio_b200 import synth
    from fluidaudio_b200.sortformer import SortformerConfig
    from oracle import oracle_sortformer as SF
    import sortformer_swift as R
    p = F(float.fromhex(p))
    cfg = SortformerConfig.preset("default")
    # below 2^-12 a 1-ulp change of log1p(-p) is under 2^-20 ulps of any score, so those plants check agreement only
    reaches_score = p > F(2.0 ** -12)
    if p == F(float.fromhex("0x1.827a74p-7")):
        cfg.pred_score_threshold = 0.01
        row = np.array([p, 0.75, 0.125, p], np.float32)
    elif not reaches_score:
        row = np.array([p, 0.75, 0.125, p], np.float32)
    else:
        # the other speakers' predictions a, from 0.001 up, until the 1-ulp difference of log1p(-p) survives the
        # score's sums: they keep the sum of log1p(-p) terms small enough that its grid can resolve it
        a = F(0.001)
        while True:
            row = np.array([a, a, a, p], np.float32)
            new, old = _scores_both_policies(R, row, F(cfg.pred_score_threshold))
            if new != old:
                break
            a = np.nextafter(a, F(1), dtype=np.float32)
            assert a < F(0.0011)
    c, _ = cfg.resolved()
    s, rng = SF.Session(vars(cfg)), np.random.default_rng(5)
    comp = None
    while comp is None:
        n, lc = s.lengths(), 1 if s.chunks else 0
        emb, preds = synth.sortformer_chunk(rng, "turns", n.spkcache_length, n.fifo_length, 6, lc, 7)
        preds[:] = row
        assert s.update(emb, preds, lc, 7)[0] == 0
        comp = s.last_compression()
    L = _emul(tmp_path_factory, "sortformer_emul.cpp", "sortformer_emul")
    L.sortformer_emul_compress.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_float,
                                           ctypes.c_float, ctypes.c_int, ctypes.c_int, ctypes.c_int] + \
        [ctypes.c_void_p] * 5
    res = [np.zeros((comp.frames, 4), np.float32) for _ in range(4)]
    per = c.spkcache_len // 4 - c.spkcache_sil_frames_per_spk
    k = lambda r: int(F(per) * F(r))
    pr = np.ascontiguousarray(comp.preds)
    L.sortformer_emul_compress(pr.ctypes.data, comp.frames, c.spkcache_len, c.spkcache_sil_frames_per_spk,
                               c.pred_score_threshold, c.scores_boost_latest, k(c.strong_boost_rate),
                               k(c.weak_boost_rate), k(c.min_pos_scores_rate), *[r.ctypes.data for r in res],
                               np.zeros(c.spkcache_len, np.int32).ctypes.data)
    planted = np.flatnonzero((comp.preds == row).all(axis=1))
    assert planted.size > 0
    restated = np.array([R.frame_scores(comp.preds[i], c.pred_score_threshold) for i in planted], np.float32)
    assert np.array_equal(bits(comp.scores), bits(res[0]))
    assert np.array_equal(bits(comp.scores[planted]), bits(restated))
    if not reaches_score:
        return
    old_policy(R, log="vlog", log1p="vlog1p")
    old = np.array([R.frame_scores(comp.preds[i], c.pred_score_threshold) for i in planted], np.float32)
    assert not np.array_equal(bits(old), bits(restated))


def _scores_both_policies(R, row, thr):
    """sortformer_swift.frame_scores of one row as bytes, correctly rounded and under the old policy"""
    new = np.array(R.frame_scores(row, thr), np.float32).tobytes()
    saved = R.vlog, R.vlog1p
    R.vlog, R.vlog1p = _old(FE.LOG), _old(FE.LOG1P)
    try:
        old = np.array(R.frame_scores(row, thr), np.float32).tobytes()
    finally:
        R.vlog, R.vlog1p = saved
    return new, old


def _prepare_restated(x):
    """decode_frame's log-probabilities of one frame (OfflineSegmentationProcessor.swift:337-346) over float32 scalars"""
    m = x[0]
    for v in x[1:]:
        m = v if m < v else m
    s = F(0)
    for v in x:
        s = F(s + FE.exp(F(v + -m)))
    neg_lse = -F(FE.log(s) + m)
    return np.array([F(v + neg_lse) for v in x], np.float32)


def test_planted_prepare(tmp_path_factory):
    from oracle import oracle_prepare as P
    L = _emul(tmp_path_factory, "prepare_emul.cpp", "prepare_emul")
    L.prepare_emul_decode.restype = ctypes.c_longlong
    L.prepare_emul_decode.argtypes = [ctypes.c_void_p, ctypes.c_longlong, ctypes.c_int, ctypes.c_float,
                                      ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p]
    # The exp sum of 8 classes lies in [1, 8], where no log input is hard: the plant is exp(HARD_EXP), once as a
    # shifted logit and once as the empty class's probability exp(x[0] - lse) (lse = 0 when exp(...) sums to 1
    # within float32: the rest are -inf-like).
    x = np.array([[0, HARD_EXP, -200, -200, -200, -200, -200, -200],
                  [HARD_EXP, 0, -200, -200, -200, -200, -200, -200]], np.float32)
    want = P.seg_decode(x[None]).log_probs[0]
    got, w, hist = np.zeros_like(x), np.zeros((2, 3), np.float32), np.zeros(8, np.int64)
    L.prepare_emul_decode(x.ctypes.data, 2, 8, 0.5, got.ctypes.data, w.ctypes.data, hist.ctypes.data)
    restated = np.stack([_prepare_restated(r) for r in x])
    assert np.array_equal(bits(want), bits(got)) and np.array_equal(bits(want), bits(restated))
