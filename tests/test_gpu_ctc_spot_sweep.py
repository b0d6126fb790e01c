"""CTC keyword spotting on the H100 against the oracle (``oracle/oracle_ctc.cpp``), bit for bit.

The log-softmax and the chunk merge equal the oracle's bits in both layouts.  The spotter's counts, every detection's
frames and score bits, and their order equal the oracle run on the same log-probs the GPU got, so the dynamic program
is checked apart from libm.  The sweep covers 1, 3 and 17 clips, clips of 0 to 20 000 frames, up to 300 terms of 1 to
127 tokens (128 refused), wildcards, repeats, out-of-range ids, constant matrices, thresholds from nil to -inf, the
device variant, a too-small capacity and the launch count; then thousands of constrained queries, the reference's
CtcDPAlgorithmTests through the GPU, and one clip at a user's size (45 000 x 1025, 100 terms).
"""
import ctypes as C
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import ctc_cases  # noqa: E402
from fluidaudio_b200 import _lib  # noqa: E402
from fluidaudio_b200 import ctc_spotting as S  # noqa: E402
from oracle import oracle_ctc as O  # noqa: E402

pytestmark = pytest.mark.gpu
W = S.WILDCARD


@pytest.fixture(scope="module", autouse=True)
def device():
    if _lib.device_count() < 1:
        pytest.skip("needs an H100")
    _lib.set_device(0)


def bits(x):
    return np.asarray(x, np.float32).view(np.uint32)


def terms_of(rng, K, V, max_n=8):
    out = []
    for k in range(K):
        n = int(rng.integers(1, max_n + 1))
        t = rng.integers(0, V, size=n).astype(np.int64)
        r = rng.uniform()
        if r < 0.1:
            t[rng.integers(0, n)] = W
        elif r < 0.15:
            t[:] = W
        elif r < 0.25 and n > 1:
            t[1] = t[0]
        elif r < 0.3:
            t[-1] = V + 3 if rng.uniform() < 0.5 else -7
        out.append([int(x) for x in t])
    return out


def check_spot(clips, terms, V, blank, min_score, device_too=True):
    want_counts, want = O.spot(clips, terms, min_score, blank)
    sp = S.CtcSpotter(V, terms, blank)
    try:
        before = _lib.kernel_launch_count()
        counts, det = sp.spot(clips, min_score)
        launches = _lib.kernel_launch_count() - before
        assert np.array_equal(counts, want_counts)
        assert len(det) == len(want)
        got = [(int(d["clip"]), int(d["term"]), int(bits(d["score"])), int(d["start_frame"]), int(d["end_frame"]))
               for d in det]
        assert got == [(b, k, int(bits(s)), a, e) for b, k, s, a, e in want]
        pairs = len(clips) * len(terms)
        first_capacity = max(1, sum(map(len, clips)) // 8)   # CtcSpotter.spot's first guess, then a retry
        n = len(want)
        assert launches == (0 if pairs == 0 else (1 + (n > 0) if n <= first_capacity else 3))
        if device_too and pairs:
            off = np.concatenate([[0], np.cumsum([len(c) for c in clips])]).astype(np.int64)
            flat = np.ascontiguousarray(np.concatenate(clips), np.float32)
            d_lp = _lib.DeviceBuffer(max(4, flat.nbytes))
            d_lp.upload(flat)
            cap = max(1, len(want))
            d_det = _lib.DeviceBuffer(cap * _lib.CTC_DETECTION.itemsize)
            st, dc, total = sp.spot_device(d_lp, off, d_det, cap, min_score)
            assert st == 0 and total == len(want) and np.array_equal(dc, counts)
            _lib.synchronize()
            assert d_det.download(cap, _lib.CTC_DETECTION)[:total].tobytes() == det.tobytes()
    finally:
        sp.close()
    return len(want)


@pytest.mark.parametrize("V", [5, 129, 1025])
@pytest.mark.parametrize("temperature", [1.0, 0.7, 1.3])
@pytest.mark.parametrize("bias", [0.0, 0.5])
def test_log_softmax_bit_exact(V, temperature, bias):
    rng = np.random.default_rng(V)
    x = rng.normal(0, 5, size=(301, V)).astype(np.float32)
    for blank in (V - 1, V + 1000):
        want = O.log_softmax(x, temperature, bias, blank)
        assert S.apply_log_softmax(x, blank, temperature, bias).tobytes() == want.tobytes()
        got = S.apply_log_softmax(np.ascontiguousarray(x.T), blank, temperature, bias, vocab_major=True)
        assert got.tobytes() == want.tobytes()


def test_log_softmax_device_variant():
    rng = np.random.default_rng(3)
    x = rng.normal(0, 3, size=(1000, 1025)).astype(np.float32)
    d_in, d_out = _lib.DeviceBuffer(x.nbytes), _lib.DeviceBuffer(x.nbytes)
    d_in.upload(x)
    before = _lib.kernel_launch_count()
    _lib.check(_lib.load().fa_ctc_log_softmax_device(d_in.ptr, 1000, 1025, 0, 0.9, 0.25, 1024, d_out.ptr),
               "fa_ctc_log_softmax_device")
    assert _lib.kernel_launch_count() - before == 1
    _lib.synchronize()
    assert d_out.download(x.shape, np.float32).tobytes() == O.log_softmax(x, 0.9, 0.25, 1024).tobytes()


@pytest.mark.parametrize("overlap", [0, 1, 25, 400])
def test_merge_chunks_bit_exact(overlap):
    rng = np.random.default_rng(overlap)
    V = 129
    chunks = [ctc_cases.log_probs(rng, n, V, "neginf") for n in (187, 0, 30, 187, 3, 120)]
    chunks[3][:4] = -np.inf
    chunks[4][:] = -np.inf
    want = O.merge_chunks(chunks, overlap)
    before = _lib.kernel_launch_count()
    got = S.merge_chunks(chunks, overlap=overlap)
    assert _lib.kernel_launch_count() - before == 1
    assert got.shape == want.shape and got.tobytes() == want.tobytes()


def test_merge_chunks_overlap_from_frame_duration():
    assert S.overlap_frames(0.08) == 25 and S.overlap_frames(0.04) == 50


SWEEP = [
    # (clips' frames, terms, vocab, blank, max tokens, min_score, kind)
    ([20000], 300, 1025, 1024, 8, None, "random"),
    ([0, 1023, 1024, 1025], 60, 129, 128, 6, -3.0, "random"),
    ([int(t) for t in np.random.default_rng(17).integers(0, 700, size=17)], 40, 5, 1024, 5, -3e38, "random"),
    ([300, 2], 50, 7, 6, 4, float("-inf"), "constant"),
    ([500, 501, 499], 80, 33, 0, 8, 0.5, "coarse"),
    ([800], 120, 9, 8, 6, None, "neginf"),
]


@pytest.mark.parametrize("case", range(len(SWEEP)))
def test_spot_sweep(case):
    frames, K, V, blank, max_n, ms, kind = SWEEP[case]
    rng = np.random.default_rng(case)
    clips = [ctc_cases.log_probs(rng, T, V, kind) for T in frames]
    assert check_spot(clips, terms_of(rng, K, V, max_n), V, blank, ms) >= 0


@pytest.mark.parametrize("ms", [None, -40.0, float("-inf")])
def test_spot_long_terms(ms):
    rng = np.random.default_rng(5)
    V = 11
    terms = [[int(x) for x in rng.integers(0, V, size=n)] for n in (1, 2, 31, 32, 63, 64, 100, 126, 127)]
    terms[3][5] = W
    clips = [ctc_cases.log_probs(rng, T, V) for T in (126, 127, 128, 400)]
    check_spot(clips, terms, V, V - 1, ms)
    with pytest.raises(_lib.FluidAudioError) as e:
        S.CtcSpotter(V, terms + [[1] * 128], V - 1)
    assert e.value.status == 8


def test_spot_case_rules():
    """every seeded case of the CPU tests, one clip per case, one term per case"""
    for i, (name, lp, toks, blank) in enumerate(ctc_cases.cases(1)):
        if i % 7:
            continue
        for ms in ctc_cases.MIN_SCORES:
            check_spot([lp, lp[: len(lp) // 2]], [toks, toks[:1]], lp.shape[1], blank, ms, device_too=False)


def test_too_small_capacity_leaves_detections_untouched():
    rng = np.random.default_rng(9)
    V = 17
    clips = [ctc_cases.log_probs(rng, 200, V) for _ in range(3)]
    terms = terms_of(rng, 10, V)
    want_counts, want = O.spot(clips, terms, -3e38, V - 1)
    assert len(want) > 4
    sp = S.CtcSpotter(V, terms, V - 1)
    flat = np.ascontiguousarray(np.concatenate(clips))
    off = np.array([0, 200, 400, 600], np.int64)
    det = np.zeros(len(want) - 1, _lib.CTC_DETECTION)
    det["score"] = 7.0
    before = _lib.kernel_launch_count()
    st, counts, total = sp._call(_lib.load().fa_ctc_spot, _lib.ptr(flat), off, -3e38, _lib.ptr(det), len(det))
    assert _lib.kernel_launch_count() - before == 1
    assert st == 3 and total == len(want) and np.array_equal(counts, want_counts)
    assert (det["score"] == 7.0).all() and (det["clip"] == 0).all()
    sp.close()


def test_constrained_queries_bit_exact():
    rng = np.random.default_rng(11)
    V, T, Q = 65, 2000, 3000
    lp = ctc_cases.log_probs(rng, T, V)
    queries = terms_of(rng, Q, V, 10)
    queries[0] = []
    ss = rng.integers(-50, T + 50, size=Q)
    se = ss + rng.integers(-5, 200, size=Q)
    ss[1], se[1] = -2 ** 40, 2 ** 40
    ss[2], se[2] = 2 ** 40, 2 ** 41
    before = _lib.kernel_launch_count()
    score, start, end = S.word_spot_constrained(lp, queries, ss, se, blank_id=V - 1)
    assert _lib.kernel_launch_count() - before == 1
    for q in range(Q):
        ws, wa, we = O.word_spot_constrained(lp, queries[q], int(ss[q]), int(se[q]), V - 1)
        assert (bits(score[q]), start[q], end[q]) == (bits(ws), wa, we), q
    # the device variant
    tok = np.ascontiguousarray(np.concatenate([np.asarray(t, np.int32) for t in queries if t]), np.int32)
    off = np.concatenate([[0], np.cumsum([len(t) for t in queries])]).astype(np.int64)
    d_lp, d_s, d_a, d_e = (_lib.DeviceBuffer(lp.nbytes), _lib.DeviceBuffer(4 * Q), _lib.DeviceBuffer(8 * Q),
                           _lib.DeviceBuffer(8 * Q))
    d_lp.upload(lp)
    ss64, se64 = np.ascontiguousarray(ss, np.int64), np.ascontiguousarray(se, np.int64)
    _lib.check(_lib.load().fa_ctc_spot_constrained_device(d_lp.ptr, T, V, V - 1, Q, _lib.ptr(tok), _lib.ptr(off),
                                                          _lib.ptr(ss64), _lib.ptr(se64), d_s.ptr, d_a.ptr, d_e.ptr),
               "fa_ctc_spot_constrained_device")
    _lib.synchronize()
    assert d_s.download(Q, np.float32).tobytes() == score.tobytes()
    assert np.array_equal(d_a.download(Q, np.int64), start) and np.array_equal(d_e.download(Q, np.int64), end)


def _mlp(frames, vocab, hot, high=-0.1, cold=-10.0):
    m = np.full((frames, vocab), cold, np.float32)
    for f, t in hot:
        m[f, t] = high
    return m


def _frame(V, hot, high, b, blank, cold):
    row = np.full(V, cold, np.float32)
    if b < V:
        row[b] = blank
    if hot is not None:
        row[hot] = high
    return row


def test_reference_kats_through_the_gpu():
    one = lambda lp, toks, a, b, blank=1024: S.word_spot_constrained(lp, [toks], a, b, blank)  # noqa: E731
    s, a, e = one(_mlp(20, 5, [(5, 0), (6, 1)]), [0, 1], 3, 12)
    assert s[0] > -1.0 and a[0] >= 3 and e[0] <= 12
    assert one(_mlp(20, 5, [(15, 0), (16, 1)]), [0, 1], 0, 10)[0][0] < -5.0
    assert one(_mlp(5, 3, [(2, 0)]), [0], -5, 100)[0][0] > -np.inf
    assert one(_mlp(20, 5, []), [0, 1, 2], 5, 7)[0][0] == -np.inf
    assert one(_mlp(10, 5, []), [0], 5, 5)[0][0] == -np.inf
    assert abs(one(_mlp(3, 3, [(0, 0), (1, 1), (2, 2)], -0.05), [0, 1, 2], 0, 3)[0][0] + 0.05) <= 0.01
    rows = np.array([_frame(4, h, -0.1, 3, -0.5, -10.0) for h in (0, None, None, None, 1)])
    assert abs(one(rows, [0, 1], 0, 5, 3)[0][0] + 0.85) <= 0.01
    nb = np.array([_frame(3, 0, -0.1, 2, -0.5, -10.0)] * 2)
    wb = np.array([_frame(3, h, -0.1, 2, -0.5, -10.0) for h in (0, None, 0)])
    assert one(wb, [0, 0], 0, 3, 2)[0][0] > one(nb, [0, 0], 0, 2, 2)[0][0] + 1.0
    rows = np.array([_frame(4, 0, -0.1, 3, -10.0, -10.0), _frame(4, None, -0.1, 3, -0.1, -10.0),
                     _frame(4, 2, -0.1, 3, -10.0, -10.0)])
    assert abs(one(rows, [0, W, 2], 0, 3, 3)[0][0] + 0.1) <= 0.05

    def multiple(lp, toks, ms):
        sp = S.CtcSpotter(lp.shape[1], [toks], 1024)
        counts, det = sp.spot([lp], None if ms is None else ms + max(0, len(toks) - 3))
        sp.close()
        return det
    assert len(multiple(_mlp(5, 3, []), [0], -5.0)) == 0
    det = multiple(_mlp(10, 5, [(2, 0)]), [0], -1.0)
    assert len(det) >= 1 and det[0]["score"] > -1.0
    counts, det = S.CtcSpotter(3, [[]], 1024).spot([_mlp(5, 3, [])], None)
    assert counts.sum() == 0
    counts, det = S.CtcSpotter(3, [[0]], 1024).spot([np.zeros((0, 3), np.float32)], None)
    assert counts.sum() == 0


def test_keyword_spotter_facade():
    rng = np.random.default_rng(2)
    V = 33
    lp = ctc_cases.log_probs(rng, 400, V)
    vocab = [S.CustomVocabularyTerm("ab", [1, 2]), S.CustomVocabularyTerm("hello", [3, 4, 5], [6, 7]),
             S.CustomVocabularyTerm("world", [8, 9, 10, 11, 12]), S.CustomVocabularyTerm("empty", [])]
    got = S.CtcKeywordSpotter(blank_id=V - 1).spot_keywords_from_log_probs(lp, 0.08, vocab, min_score=-4.0)
    want = []
    for term, ids in ((vocab[1], [6, 7]), (vocab[2], [8, 9, 10, 11, 12])):
        want += [(term.text, s, a, e) for s, a, e in O.word_spot_multiple(lp, ids, O.threshold(-4.0, len(ids)), V - 1)]
    assert [(d.term.text, np.float32(d.score), d.start_frame, d.end_frame) for d in got] == want
    assert all(d.start_time == d.start_frame * 0.08 and d.total_frames == 400 for d in got)


def test_user_size_clip():
    """an hour at 80 ms frames: 45 000 x 1025 log-probs and 100 terms"""
    rng = np.random.default_rng(45)
    V = 1025
    logits = rng.normal(0, 3, size=(45000, V)).astype(np.float32)
    lp = S.apply_log_softmax(logits, 1024)
    assert lp.tobytes() == O.log_softmax(logits, 1.0, 0.0, 1024).tobytes()
    assert check_spot([lp], terms_of(rng, 100, V, 8), V, 1024, None, device_too=False) > 0
